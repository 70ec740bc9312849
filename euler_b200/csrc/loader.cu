// Euler 2.0 on-disk format -> host CSR -> eu_graph_create.
//
// Format (SURVEY.md Appendix B; writer euler/tools/{util,node,graph_meta}.py, reader
// euler/core/graph/node.cc:414-526, euler/core/graph/graph_builder.cc:230-332,
// euler/common/bytes_io.h:28-81): little-endian; list<T> = u32 n + n items; str = u32 len + bytes.
//   <dir>/euler.meta : str name, str version, u64 nodes, u64 edges, i32 partitions,
//                      u32 nf x {str name, i32 kind, i32 idx, i64 dim}, u32 ef x {...},
//                      u32 nnt x {str name, u32 id}, u32 net x {str name, u32 id}
//   <dir>/Node/<prefix>_<p>.dat : records  u32 len + { u64 id, i32 type, f32 weight,
//        out block, in block, list<i32> u64 ends, list<u64>, list<i32> f32 ends, list<f32>,
//        list<i32> bin ends, str bin };  block = list<i32> group ids, list<f32> group weights,
//        list<i32> group ends, list<u64> neighbor ids, list<f32> cumulative weights
// A shard loads <prefix>_<p>.dat iff the name splits into exactly 3 tokens on '_' '.', the last is
// "dat" and p % shard_number == shard_index (euler/core/graph/graph.cc:90-98).
#include <dirent.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <unordered_map>
#include <string>
#include <vector>

#include "internal.h"

namespace eu {

struct Reader {
  const unsigned char* p;
  const unsigned char* end;
  bool ok = true;
  template <typename T>
  T get() {
    T v{};
    if (p + sizeof(T) > end) { ok = false; return v; }
    memcpy(&v, p, sizeof(T));
    p += sizeof(T);
    return v;
  }
  template <typename T>
  void list(std::vector<T>* out) {
    uint32_t n = get<uint32_t>();
    if (!ok || p + (size_t)n * sizeof(T) > end) { ok = false; return; }
    out->resize(n);
    if (n) memcpy(out->data(), p, (size_t)n * sizeof(T));
    p += (size_t)n * sizeof(T);
  }
  std::string str() {
    uint32_t n = get<uint32_t>();
    if (!ok || p + n > end) { ok = false; return std::string(); }
    std::string s((const char*)p, n);
    p += n;
    return s;
  }
};

static bool read_file(const std::string& path, std::vector<unsigned char>* buf) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) return false;
  fseek(f, 0, SEEK_END);
  long sz = ftell(f);
  fseek(f, 0, SEEK_SET);
  buf->resize(sz > 0 ? sz : 0);
  size_t got = sz > 0 ? fread(buf->data(), 1, sz, f) : 0;
  fclose(f);
  return got == (size_t)(sz > 0 ? sz : 0);
}

static std::vector<std::string> split_any(const std::string& s, const char* seps) {
  std::vector<std::string> out;
  std::string cur;
  for (char ch : s) {
    if (strchr(seps, ch)) { if (!cur.empty()) out.push_back(cur); cur.clear(); }
    else cur.push_back(ch);
  }
  if (!cur.empty()) out.push_back(cur);
  return out;
}

// euler::hash64 (euler/common/hash.cc:76-128, hash.h:41-52) = the first word of MurmurHash3_x64_128 (Appleby, public
// domain algorithm) with seed 0 -- the hash of the reference's edge_map_ (EdgeIDHashFunc, euler/common/data_types.h:48-56:
// the 20 bytes src | dst | type).  Needed only to replay that map's iteration order for the global edge sampler.
static inline uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
static uint64_t murmur3_x64_128_h1(const unsigned char* data, int size) {
  const uint64_t c1 = 0x87c37b91114253d5ULL, c2 = 0x4cf5ad432745937fULL;
  uint64_t h1 = 0, h2 = 0, k1, k2;
  const int nblocks = size >> 4;
  for (int i = 0; i < nblocks; ++i) {
    memcpy(&k1, data + 16 * i, 8); memcpy(&k2, data + 16 * i + 8, 8);
    k1 *= c1; k1 = rotl64(k1, 31); k1 *= c2; h1 ^= k1;
    h1 = rotl64(h1, 27); h1 += h2; h1 = h1 * 5 + 0x52dce729;
    k2 *= c2; k2 = rotl64(k2, 33); k2 *= c1; h2 ^= k2;
    h2 = rotl64(h2, 31); h2 += h1; h2 = h2 * 5 + 0x38495ab5;
  }
  const unsigned char* tail = data + 16 * nblocks;
  k1 = 0; k2 = 0;
  switch (size & 15) {
    case 15: k2 ^= (uint64_t)tail[14] << 48;  // fallthrough
    case 14: k2 ^= (uint64_t)tail[13] << 40;  // fallthrough
    case 13: k2 ^= (uint64_t)tail[12] << 32;  // fallthrough
    case 12: k2 ^= (uint64_t)tail[11] << 24;  // fallthrough
    case 11: k2 ^= (uint64_t)tail[10] << 16;  // fallthrough
    case 10: k2 ^= (uint64_t)tail[9] << 8;    // fallthrough
    case 9: k2 ^= (uint64_t)tail[8];
      k2 *= c2; k2 = rotl64(k2, 33); k2 *= c1; h2 ^= k2;  // fallthrough
    case 8: k1 ^= (uint64_t)tail[7] << 56;    // fallthrough
    case 7: k1 ^= (uint64_t)tail[6] << 48;    // fallthrough
    case 6: k1 ^= (uint64_t)tail[5] << 40;    // fallthrough
    case 5: k1 ^= (uint64_t)tail[4] << 32;    // fallthrough
    case 4: k1 ^= (uint64_t)tail[3] << 24;    // fallthrough
    case 3: k1 ^= (uint64_t)tail[2] << 16;    // fallthrough
    case 2: k1 ^= (uint64_t)tail[1] << 8;     // fallthrough
    case 1: k1 ^= (uint64_t)tail[0];
      k1 *= c1; k1 = rotl64(k1, 31); k1 *= c2; h1 ^= k1;
  }
  h1 ^= (uint64_t)size; h2 ^= (uint64_t)size;
  h1 += h2; h2 += h1;
  auto fmix = [](uint64_t k) { k ^= k >> 33; k *= 0xff51afd7ed558ccdULL; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ULL; k ^= k >> 33; return k; };
  h1 = fmix(h1); h2 = fmix(h2);
  h1 += h2;
  return h1;
}

struct EdgeKey { uint64_t s, d; int32_t t; };
struct EdgeKeyHash {
  size_t operator()(const EdgeKey& k) const {
    unsigned char tmp[20];
    memcpy(tmp, &k.s, 8); memcpy(tmp + 8, &k.d, 8); memcpy(tmp + 16, &k.t, 4);
    return (size_t)murmur3_x64_128_h1(tmp, 20);
  }
};
struct EdgeKeyEq { bool operator()(const EdgeKey& a, const EdgeKey& b) const { return a.s == b.s && a.d == b.d && a.t == b.t; } };

// Edge/<prefix>_<p>.dat of this shard (records: u64 src, u64 dst, i32 type, f32 weight + the three feature blocks,
// euler/tools/edge.py:47-64; reader euler/core/graph/edge.cc) -> eu_graph_set_edges.  A missing Edge directory = no edges.
static int load_edge_files(eu_graph* g, const std::string& dir, int shard_index, int shard_number,
                           const std::map<int32_t, std::pair<std::string, int64_t>>& dense, const std::map<int32_t, std::string>& sparse,
                           const std::map<int32_t, std::string>& binary) {
  std::vector<std::string> files, readdir_files;
  DIR* dd = opendir((dir + "/Edge").c_str());
  if (!dd) return EU_OK;
  while (dirent* e = readdir(dd)) {
    std::string fn(e->d_name);
    auto tok = split_any(fn, "_.");
    if (tok.size() == 3 && tok[2] == "dat" && atoi(tok[1].c_str()) % shard_number == shard_index) files.push_back(fn);
  }
  closedir(dd);
  readdir_files = files;
  std::sort(files.begin(), files.end());
  const int32_t n_slots = dense.empty() ? 0 : dense.rbegin()->first + 1;
  if (n_slots > EU_MAX_FEAT_SLOTS) { set_error("%d dense edge features unsupported", n_slots); return EU_ERR_UNSUPPORTED; }
  std::vector<int32_t> slot_dims(n_slots, 0), slot_off(n_slots, 0);
  int32_t width = 0;
  for (int32_t s = 0; s < n_slots; ++s) { slot_dims[s] = dense.count(s) ? (int32_t)dense.at(s).second : 0; slot_off[s] = width; width += slot_dims[s]; }
  const int32_t US = sparse.empty() ? 0 : sparse.rbegin()->first + 1, BS = binary.empty() ? 0 : binary.rbegin()->first + 1;
  std::vector<uint64_t> src, dst, u64_all, u64v;
  std::vector<int32_t> type, ue, fe, be;
  std::vector<float> w, feat, fv;
  std::vector<int64_t> u64_ptr(1, 0), bin_ptr(1, 0);
  std::vector<uint8_t> bin_all;
  std::string binv;
  std::map<std::string, std::pair<int64_t, int64_t>> file_rows;
  std::vector<unsigned char> buf;
  for (const auto& fn : files) {
    if (!read_file(dir + "/Edge/" + fn, &buf)) { set_error("cannot read Edge/%s", fn.c_str()); return EU_ERR_IO; }
    Reader f{buf.data(), buf.data() + buf.size()};
    file_rows[fn].first = (int64_t)src.size();
    while (f.p < f.end) {
      uint32_t len = f.get<uint32_t>();
      if (!f.ok || f.p + len > f.end) { set_error("truncated record in Edge/%s", fn.c_str()); return EU_ERR_IO; }
      Reader r{f.p, f.p + len};
      f.p += len;
      src.push_back(r.get<uint64_t>()); dst.push_back(r.get<uint64_t>()); type.push_back(r.get<int32_t>()); w.push_back(r.get<float>());
      r.list(&ue); r.list(&u64v);
      r.list(&fe); r.list(&fv);
      r.list(&be); binv = r.str();
      if (!r.ok) { set_error("malformed edge record in Edge/%s", fn.c_str()); return EU_ERR_IO; }
      const size_t fbase = feat.size();
      feat.resize(fbase + width, 0.f);
      for (int32_t s = 0; s < n_slots && s < (int32_t)fe.size(); ++s) {
        const int32_t b = s == 0 ? 0 : fe[s - 1], e = fe[s];
        if (b < 0 || e > (int32_t)fv.size() || e < b) { set_error("bad f32 edge feature ends in Edge/%s", fn.c_str()); return EU_ERR_IO; }
        const int32_t l2 = std::min(e - b, slot_dims[s]);
        if (l2 > 0) memcpy(&feat[fbase + slot_off[s]], &fv[b], sizeof(float) * l2);
      }
      for (int32_t s = 0; s < US; ++s) {
        if (s < (int32_t)ue.size()) {
          const int32_t b = s == 0 ? 0 : ue[s - 1], e = ue[s];
          if (b < 0 || e < b || e > (int32_t)u64v.size()) { set_error("bad uint64 edge feature ends in Edge/%s", fn.c_str()); return EU_ERR_IO; }
          u64_all.insert(u64_all.end(), u64v.begin() + b, u64v.begin() + e);
        }
        u64_ptr.push_back((int64_t)u64_all.size());
      }
      for (int32_t s = 0; s < BS; ++s) {
        if (s < (int32_t)be.size()) {
          const int32_t b = s == 0 ? 0 : be[s - 1], e = be[s];
          if (b < 0 || e < b || e > (int32_t)binv.size()) { set_error("bad binary edge feature ends in Edge/%s", fn.c_str()); return EU_ERR_IO; }
          bin_all.insert(bin_all.end(), binv.begin() + b, binv.begin() + e);
        }
        bin_ptr.push_back((int64_t)bin_all.size());
      }
    }
    file_rows[fn].second = (int64_t)src.size();
  }
  // iteration order of edge_map_ (std::unordered_map<EdgeID, Edge*, EdgeIDHashFunc, EdgeIDEqualKey>, graph.h) after
  // GraphBuilder::AddToGraph inserted the records file by file in readdir order (graph_builder.cc:160-166, graph.cc:197-203)
  std::vector<int64_t> order;
  {
    std::unordered_map<EdgeKey, int64_t, EdgeKeyHash, EdgeKeyEq> emap;
    for (const auto& fn : readdir_files) {
      const auto& rr = file_rows[fn];
      for (int64_t r = rr.first; r < rr.second; ++r) emap.insert({EdgeKey{src[r], dst[r], type[r]}, r});
    }
    order.reserve(emap.size());
    for (const auto& kv : emap) order.push_back(kv.second);
    if (order.size() != src.size()) {   // duplicate records: not in the map, appended so that every row has a sampler slot
      std::vector<char> seen(src.size(), 0);
      for (int64_t r : order) seen[r] = 1;
      for (int64_t r = 0; r < (int64_t)src.size(); ++r) if (!seen[r]) order.push_back(r);
    }
  }
  eu_edge_desc d{};
  uint64_t u64_dummy = 0; uint8_t bin_dummy = 0;
  d.n_edges = (int64_t)src.size();
  d.src = src.data(); d.dst = dst.data(); d.type = type.data(); d.w = w.data();
  d.feat_dim = width; d.feat = width > 0 ? feat.data() : nullptr;
  d.n_feat_slots = width > 0 ? n_slots : 0; d.feat_slot_dims = slot_dims.data();
  if (US > 0) { d.n_u64_slots = US; d.u64_ptr = u64_ptr.data(); d.u64_val = u64_all.empty() ? &u64_dummy : u64_all.data(); }
  if (BS > 0) { d.n_bin_slots = BS; d.bin_ptr = bin_ptr.data(); d.bin_val = bin_all.empty() ? &bin_dummy : bin_all.data(); }
  d.sampler_order = order.data();
  int rc = eu_graph_set_edges(g, &d);
  if (rc) return rc;
  auto strip = [](std::string nm, const char* pre) { const size_t l = strlen(pre); if (nm.compare(0, l, pre) == 0) nm = nm.substr(l); return nm; };
  g->edge_dense_names.assign(d.n_feat_slots, "");
  for (auto& kv : dense) if (kv.first < d.n_feat_slots) g->edge_dense_names[kv.first] = strip(kv.second.first, "dense_");
  g->edge_sparse_names.assign(US, "");
  for (auto& kv : sparse) g->edge_sparse_names[kv.first] = strip(kv.second, "sparse_");
  g->edge_binary_names.assign(BS, "");
  for (auto& kv : binary) g->edge_binary_names[kv.first] = strip(kv.second, "binary_");
  return EU_OK;
}

}  // namespace eu

using namespace eu;

// what eu_graph_load_inspect reports (host-only: the parse and the sampler-order replay, no device)
struct LoadInspect {
  int64_t n_nodes = 0, n_edges = 0;
  int32_t n_edge_types = 0, n_node_types = 0;
  std::vector<int64_t> order_ids;
  std::vector<int32_t> order_types;
  bool has_labels = false;              // the graph has the binary slot graph_label
  std::vector<std::string> labels;      // then Graph::GetGraphLabel's list
};

static int load_impl(const char* data_path, int shard_index, int shard_number, int device, int load_edges,
                     const eu_feat_storage* storage, eu_graph** out, LoadInspect* inspect) {
  if (!data_path || (!out && !inspect) || shard_number <= 0 || shard_index < 0 || shard_index >= shard_number) {
    set_error("eu_graph_load: bad argument (shard %d of %d)", shard_index, shard_number);
    return EU_ERR_INVALID;
  }
  const std::string dir(data_path);
  // ---- meta
  std::vector<unsigned char> buf;
  if (!read_file(dir + "/euler.meta", &buf)) { set_error("cannot read %s/euler.meta", data_path); return EU_ERR_IO; }
  Reader m{buf.data(), buf.data() + buf.size()};
  m.str(); m.str();
  m.get<uint64_t>(); m.get<uint64_t>();
  int32_t partitions = m.get<int32_t>();
  std::map<int32_t, std::pair<std::string, int64_t>> dense;  // idx -> (name, dim)
  std::map<int32_t, std::string> sparse, binary;               // idx -> name (kind 0 / kind 2)
  uint32_t nf = m.get<uint32_t>();
  for (uint32_t i = 0; i < nf && m.ok; ++i) {
    std::string name = m.str();
    int32_t kind = m.get<int32_t>(), idx = m.get<int32_t>();
    int64_t dim = m.get<int64_t>();
    if (kind == 1) dense[idx] = std::make_pair(name, dim);
    else if (kind == 0) sparse[idx] = name;
    else if (kind == 2) binary[idx] = name;
  }
  std::map<int32_t, std::pair<std::string, int64_t>> e_dense;
  std::map<int32_t, std::string> e_sparse, e_binary;
  uint32_t ef = m.get<uint32_t>();
  for (uint32_t i = 0; i < ef && m.ok; ++i) {
    std::string name = m.str();
    int32_t kind = m.get<int32_t>(), idx = m.get<int32_t>();
    int64_t dim = m.get<int64_t>();
    if (kind == 1) e_dense[idx] = std::make_pair(name, dim);
    else if (kind == 0) e_sparse[idx] = name;
    else if (kind == 2) e_binary[idx] = name;
  }
  std::map<uint32_t, std::string> ntypes, etypes;
  uint32_t nnt = m.get<uint32_t>();
  for (uint32_t i = 0; i < nnt && m.ok; ++i) { std::string s = m.str(); ntypes[m.get<uint32_t>()] = s; }
  uint32_t net = m.get<uint32_t>();
  for (uint32_t i = 0; i < net && m.ok; ++i) { std::string s = m.str(); etypes[m.get<uint32_t>()] = s; }
  if (!m.ok || partitions <= 0) { set_error("malformed euler.meta in %s", data_path); return EU_ERR_IO; }
  const int32_t T = (int32_t)net, NT = (int32_t)nnt;
  if (T < 1 || T > EU_MAX_ETYPES) { set_error("%d edge types unsupported", T); return EU_ERR_UNSUPPORTED; }
  const int32_t n_slots = dense.empty() ? 0 : dense.rbegin()->first + 1;
  if (n_slots > EU_MAX_FEAT_SLOTS) { set_error("%d dense features unsupported", n_slots); return EU_ERR_UNSUPPORTED; }
  std::vector<int32_t> slot_dims(n_slots, 0), slot_off(n_slots, 0);
  int32_t width = 0;
  for (int32_t s = 0; s < n_slots; ++s) {
    slot_dims[s] = dense.count(s) ? (int32_t)dense[s].second : 0;
    slot_off[s] = width;
    width += slot_dims[s];
  }
  // ---- node files of this shard, in name order (rows are laid out in this order); the order readdir returned them in is
  // kept as well: it is the reference's insert order into node_map_ (see the sampler order below)
  std::vector<std::string> files, readdir_files;
  {
    DIR* d = opendir((dir + "/Node").c_str());
    if (!d) { set_error("no such directory %s/Node", data_path); return EU_ERR_IO; }
    while (dirent* e = readdir(d)) {
      std::string fn(e->d_name);
      auto tok = split_any(fn, "_.");
      if (tok.size() == 3 && tok[2] == "dat" && atoi(tok[1].c_str()) % shard_number == shard_index) files.push_back(fn);
    }
    closedir(d);
    readdir_files = files;
    std::sort(files.begin(), files.end());
  }
  std::map<std::string, std::pair<int64_t, int64_t>> file_rows;   // file -> [first row, end row)
  std::vector<uint64_t> ids, nbr;
  std::vector<int32_t> ntype;
  std::vector<float> nw, cum, gcum, feat;
  std::vector<int64_t> gptr(1, 0);
  std::vector<int32_t> gi, ge, fe, ue, be;
  std::vector<float> gw, cw, fv;
  std::vector<uint64_t> nb, u64v;
  const int32_t US = sparse.empty() ? 0 : sparse.rbegin()->first + 1;   // uint64 / binary feature slots (meta idx range)
  const int32_t BS = binary.empty() ? 0 : binary.rbegin()->first + 1;
  std::vector<int64_t> u64_ptr(1, 0), bin_ptr(1, 0);
  std::vector<uint64_t> u64_all;
  std::vector<uint8_t> bin_all;
  std::string binv;
  for (const auto& fn : files) {
    if (!read_file(dir + "/Node/" + fn, &buf)) { set_error("cannot read %s", fn.c_str()); return EU_ERR_IO; }
    Reader f{buf.data(), buf.data() + buf.size()};
    file_rows[fn].first = (int64_t)ids.size();
    while (f.p < f.end) {
      uint32_t len = f.get<uint32_t>();
      if (!f.ok || f.p + len > f.end) { set_error("truncated record in %s", fn.c_str()); return EU_ERR_IO; }
      Reader r{f.p, f.p + len};
      f.p += len;
      ids.push_back(r.get<uint64_t>());
      ntype.push_back(r.get<int32_t>());
      nw.push_back(r.get<float>());
      r.list(&gi); r.list(&gw); r.list(&ge); r.list(&nb); r.list(&cw);
      if (!r.ok || gi.size() != gw.size() || gi.size() != ge.size() || nb.size() != cw.size() || (int32_t)gi.size() > T) {
        set_error("malformed node record (id %llu) in %s", (unsigned long long)ids.back(), fn.c_str());
        return EU_ERR_IO;
      }
      for (size_t k = 0; k < gi.size(); ++k)
        if (gi[k] != (int32_t)k) { set_error("edge group ids are not 0..T-1 for node %llu", (unsigned long long)ids.back()); return EU_ERR_UNSUPPORTED; }
      // edge_group_collection.Init(group ids, group weights): running f32 sum (compact_weighted_collection.h:82-97).
      // Nodes that carry fewer than T groups are padded with empty groups (see DESIGN.md).
      const int64_t base = (int64_t)nbr.size();
      float run = 0.f;
      int32_t last_end = 0;
      for (int32_t t = 0; t < T; ++t) {
        if (t < (int32_t)gi.size()) { run += gw[t]; last_end = ge[t]; }
        gcum.push_back(run);
        gptr.push_back(base + last_end);
      }
      if (last_end != (int32_t)nb.size()) { set_error("group ends do not cover the neighbor list of node %llu", (unsigned long long)ids.back()); return EU_ERR_IO; }
      nbr.insert(nbr.end(), nb.begin(), nb.end());
      cum.insert(cum.end(), cw.begin(), cw.end());
      // in-neighbor block: not on this path (sample_neighbor / walks use out edges only)
      r.list(&gi); r.list(&gw); r.list(&ge); r.list(&nb); r.list(&cw);
      r.list(&ue); r.list(&u64v);
      r.list(&fe); r.list(&fv);
      r.list(&be); binv = r.str();
      if (!r.ok) { set_error("malformed feature block (id %llu)", (unsigned long long)ids.back()); return EU_ERR_IO; }
      // ragged uint64 / binary features: slot s = [ends[s-1], ends[s]) of the node's value array (node.cc:353-364); slots the
      // node does not carry are empty
      for (int32_t s2 = 0; s2 < US; ++s2) {
        if (s2 < (int32_t)ue.size()) {
          const int32_t b = s2 == 0 ? 0 : ue[s2 - 1], e = ue[s2];
          if (b < 0 || e < b || e > (int32_t)u64v.size()) { set_error("bad uint64 feature ends (id %llu)", (unsigned long long)ids.back()); return EU_ERR_IO; }
          u64_all.insert(u64_all.end(), u64v.begin() + b, u64v.begin() + e);
        }
        u64_ptr.push_back((int64_t)u64_all.size());
      }
      for (int32_t s2 = 0; s2 < BS; ++s2) {
        if (s2 < (int32_t)be.size()) {
          const int32_t b = s2 == 0 ? 0 : be[s2 - 1], e = be[s2];
          if (b < 0 || e < b || e > (int32_t)binv.size()) { set_error("bad binary feature ends (id %llu)", (unsigned long long)ids.back()); return EU_ERR_IO; }
          bin_all.insert(bin_all.end(), binv.begin() + b, binv.begin() + e);
        }
        bin_ptr.push_back((int64_t)bin_all.size());
      }
      // dense slots: zero-padded / clipped to the meta dim (get_dense_feature_op.cc:66-75 zero-fills)
      const size_t fbase = feat.size();
      feat.resize(fbase + width, 0.f);
      for (int32_t s = 0; s < n_slots && s < (int32_t)fe.size(); ++s) {
        int32_t b = s == 0 ? 0 : fe[s - 1], e = fe[s];
        int32_t len = std::min(e - b, slot_dims[s]);
        if (b < 0 || e > (int32_t)fv.size() || e < b) { set_error("bad f32 feature ends (id %llu)", (unsigned long long)ids.back()); return EU_ERR_IO; }
        if (len > 0) memcpy(&feat[fbase + slot_off[s]], &fv[b], sizeof(float) * len);
      }
    }
    file_rows[fn].second = (int64_t)ids.size();
  }
  // Global node sampler order = iteration order of the reference's node_map_ (Graph::BuildGlobalSampler, graph.cc:349-354):
  // a std::unordered_map<NodeID, Node*> filled by GraphBuilder::AddToGraph (graph_builder.cc:160-166) task by task, i.e.
  // file by file in ListDirectory (readdir) order (local_file_io.cc:102-119), record by record, with insert() (the first
  // occurrence of an id wins, graph.cc:174-179).  The same container from the same libstdc++, fed the same sequence, iterates
  // in the same order: replay it on the host.
  std::vector<int64_t> order;
  {
    std::unordered_map<uint64_t, int64_t> node_map;
    for (const auto& fn : readdir_files) {
      const auto& rr = file_rows[fn];
      for (int64_t r = rr.first; r < rr.second; ++r) node_map.insert({ids[r], r});
    }
    order.reserve(node_map.size());
    for (const auto& kv : node_map) order.push_back(kv.second);
    // ids stored twice keep the FIRST record in node_map_ but the id -> row table of the device graph resolves to the last:
    // the sampler needs one entry per row, so duplicate rows (absent from the map) are appended; a converter never emits them
    if (order.size() != ids.size()) {
      std::vector<char> seen(ids.size(), 0);
      for (int64_t r : order) seen[r] = 1;
      for (int64_t r = 0; r < (int64_t)ids.size(); ++r) if (!seen[r]) order.push_back(r);
    }
  }
  eu_graph_desc d{};
  d.n_nodes = (int64_t)ids.size();
  d.n_edge_types = T;
  d.n_node_types = NT > 0 ? NT : 1;
  d.ids = ids.data(); d.node_type = ntype.data(); d.node_w = nw.data();
  d.grp_ptr = gptr.data(); d.nbr = nbr.data(); d.cum_w = cum.data(); d.grp_cum = gcum.data();
  d.feat_dim = width; d.feat = width > 0 ? feat.data() : nullptr;
  d.n_feat_slots = width > 0 ? n_slots : 0; d.feat_slot_dims = slot_dims.data();
  d.sampler_order = order.data();
  uint64_t u64_dummy = 0; uint8_t bin_dummy = 0;
  if (US > 0) { d.n_u64_slots = US; d.u64_ptr = u64_ptr.data(); d.u64_val = u64_all.empty() ? &u64_dummy : u64_all.data(); }
  if (BS > 0) { d.n_bin_slots = BS; d.bin_ptr = bin_ptr.data(); d.bin_val = bin_all.empty() ? &bin_dummy : bin_all.data(); }
  if (inspect) {   // everything above is host work: report it and stop before the upload
    inspect->n_nodes = d.n_nodes;
    inspect->n_edges = (int64_t)nbr.size();
    inspect->n_edge_types = d.n_edge_types;
    inspect->n_node_types = d.n_node_types;
    for (int64_t r : order) { inspect->order_ids.push_back((int64_t)ids[r]); inspect->order_types.push_back(ntype[r]); }
    for (auto& kv : binary)   // the device path's rule (graph_build_labels): the slot named graph_label once the prefix is stripped
      if (kv.second == "binary_graph_label" || kv.second == "graph_label") {
        inspect->has_labels = true;
        graph_label_list(order, d.n_nodes, bin_ptr.data(), bin_all.data(), BS, kv.first, &inspect->labels, nullptr);
      }
    return EU_OK;
  }
  int rc = eu_graph_create_storage(&d, device, storage, out);
  if (rc) return rc;
  eu_graph* g = *out;
  g->edge_type_names.assign(T, "");
  for (auto& kv : etypes) if ((int32_t)kv.first < T) g->edge_type_names[kv.first] = kv.second;
  g->node_type_names.assign(d.n_node_types, "");
  for (auto& kv : ntypes) if ((int32_t)kv.first < d.n_node_types) g->node_type_names[kv.first] = kv.second;
  g->dense_feature_names.assign(d.n_feat_slots, "");
  for (auto& kv : dense) {
    std::string nm = kv.second.first;
    if (nm.rfind("dense_", 0) == 0) nm = nm.substr(6);
    if (kv.first < d.n_feat_slots) g->dense_feature_names[kv.first] = nm;
  }
  g->sparse_feature_names.assign(US, "");
  for (auto& kv : sparse) { std::string nm = kv.second; if (nm.rfind("sparse_", 0) == 0) nm = nm.substr(7); g->sparse_feature_names[kv.first] = nm; }
  g->binary_feature_names.assign(BS, "");
  for (auto& kv : binary) { std::string nm = kv.second; if (nm.rfind("binary_", 0) == 0) nm = nm.substr(7); g->binary_feature_names[kv.first] = nm; }
  if (load_edges) {
    rc = load_edge_files(g, dir, shard_index, shard_number, e_dense, e_sparse, e_binary);
    if (rc) { eu_graph_destroy(g); *out = nullptr; return rc; }
  }
  return EU_OK;
}

extern "C" int eu_graph_load_ex(const char* data_path, int shard_index, int shard_number, int device, int load_edges,
                                eu_graph** out) {
  return eu_graph_load_dtype(data_path, shard_index, shard_number, device, load_edges, EU_FEAT_F32, out);
}

extern "C" int eu_graph_load_dtype(const char* data_path, int shard_index, int shard_number, int device, int load_edges,
                                   int32_t feat_dtype, eu_graph** out) {
  if (!out) { set_error("eu_graph_load: bad argument (null out)"); return EU_ERR_INVALID; }
  if (int rc = dtype_check(feat_dtype, "eu_graph_load", "feature")) return rc;
  const eu_feat_storage st{feat_dtype, EU_FEAT_DEVICE, 0};
  return load_impl(data_path, shard_index, shard_number, device, load_edges, &st, out, nullptr);
}

// the descriptor is checked here against every row count (C <= n waits for the files: eu_graph_create_storage checks it)
extern "C" int eu_graph_load_storage(const char* data_path, int shard_index, int shard_number, int device, int load_edges,
                                     const eu_feat_storage* storage, eu_graph** out) {
  if (!out) { set_error("eu_graph_load: bad argument (null out)"); return EU_ERR_INVALID; }
  eu_feat_storage st;
  const int rc = feat_storage_check(storage, storage ? storage->cache_rows : 0, "eu_graph_load", &st);
  if (rc) return rc;
  return load_impl(data_path, shard_index, shard_number, device, load_edges, &st, out, nullptr);
}

extern "C" int eu_graph_load_inspect(const char* data_path, int shard_index, int shard_number, int64_t* n_nodes, int64_t* n_edges,
                                     int32_t* n_edge_types, int32_t* n_node_types, int64_t cap, int64_t* order_ids,
                                     int32_t* order_types) {
  LoadInspect li;
  const int rc = load_impl(data_path, shard_index, shard_number, 0, 0, nullptr, nullptr, &li);
  if (rc) return rc;
  if (n_nodes) *n_nodes = li.n_nodes;
  if (n_edges) *n_edges = li.n_edges;
  if (n_edge_types) *n_edge_types = li.n_edge_types;
  if (n_node_types) *n_node_types = li.n_node_types;
  const int64_t n = std::min<int64_t>(cap, (int64_t)li.order_ids.size());
  for (int64_t i = 0; i < n; ++i) {
    if (order_ids) order_ids[i] = li.order_ids[i];
    if (order_types) order_types[i] = li.order_types[i];
  }
  return EU_OK;
}

extern "C" int eu_graph_labels_inspect(const char* data_path, int64_t cap, int64_t* n_labels, int64_t* n_bytes, int64_t* ptr,
                                       uint8_t* bytes) {
  LoadInspect li;
  const int rc = load_impl(data_path, 0, 1, 0, 0, nullptr, nullptr, &li);
  if (rc) return rc;
  if (!li.has_labels || li.labels.empty()) { set_error("graph label set is empty! (%s has no binary feature graph_label)", data_path); return EU_ERR_STATE; }
  int64_t total = 0;
  if (ptr) ptr[0] = 0;
  for (size_t l = 0; l < li.labels.size(); ++l) {
    const std::string& v = li.labels[l];
    if (bytes && total + (int64_t)v.size() <= cap) memcpy(bytes + total, v.data(), v.size());
    total += (int64_t)v.size();
    if (ptr) ptr[l + 1] = total;
  }
  if (n_labels) *n_labels = (int64_t)li.labels.size();
  if (n_bytes) *n_bytes = total;
  return EU_OK;
}

extern "C" int eu_graph_load(const char* data_path, int shard_index, int shard_number, int device, eu_graph** out) {
  return eu_graph_load_ex(data_path, shard_index, shard_number, device, 1, out);
}
