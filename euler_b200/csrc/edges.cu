// Edge store on the device: global edge sampling and edge features (SURVEY.md section 8f, next-4).
// Reference semantics (file:line relative to /root/reference):
//   Graph::SampleEdge(edge_type, count)      euler/core/graph/graph.cc:277-301   alias draw over the edges of ONE type
//   Graph::SampleEdge(edge_types, count)     :303-331   draws the type from edge_type_collection_, which the reference never
//                                            initialises (no Init call anywhere): its sum weight is 0 and the result is EMPTY;
//                                            the same holds for edge_type == -1 (:284-287).  Reported here as EU_ERR_STATE.
//   Graph::BuildGlobalEdgeSampler            :372-399   per type a FastWeightedCollection in edge_map_ iteration order
//   euler::GetEdgeFloat32Feature & co        euler/core/api/api.cc:148-205 over Edge::Get*Feature (same slot layout as Node)
//   tf_euler SampleEdge / GetEdge*Feature    tf_euler/kernels/sample_edge_op.cc, get_edge_dense_feature_op.cc,
//                                            get_edge_sparse_feature_op.cc, get_edge_binary_feature_op.cc
// Layout: SoA edge arrays, dense features [nE, W] (slots concatenated, zero padded), ragged uint64 / binary features, and an
// open-addressing table (src, dst, type) -> edge row built on the host.
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <string>
#include <vector>

#include "internal.h"

namespace eu {

__device__ __forceinline__ unsigned long long edge_hash(unsigned long long s, unsigned long long d, int32_t t) {
  return mix64(s * 0x9E3779B97F4A7C15ull ^ mix64(d + 0x632BE59BD9B4E019ull * (unsigned long long)(uint32_t)t));
}
static inline unsigned long long edge_hash_host(unsigned long long s, unsigned long long d, int32_t t) {
  return mix64(s * 0x9E3779B97F4A7C15ull ^ mix64(d + 0x632BE59BD9B4E019ull * (unsigned long long)(uint32_t)t));
}

// Graph::GetEdgeByID (graph.h:95-108): edge row or -1
__device__ __forceinline__ int64_t lookup_edge(const DevEdges& e, unsigned long long s, unsigned long long d, long long t) {
  if (e.n == 0 || t < INT32_MIN || t > INT32_MAX) return -1;
  unsigned long long h = edge_hash(s, d, (int32_t)t) & e.hmask;
  while (true) {
    const EdgeSlot sl = e.htab[h];
    if (sl.row < 0) return -1;
    if (sl.src == s && sl.dst == d && sl.type == (int32_t)t) return sl.row;
    h = (h + 1) & e.hmask;
  }
}

__global__ void k_edge_rows(DevEdges e, const long long* __restrict__ edges /* [E,3] */, int64_t E, long long* __restrict__ rows) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= E) return;
  rows[i] = lookup_edge(e, (unsigned long long)edges[i * 3], (unsigned long long)edges[i * 3 + 1], edges[i * 3 + 2]);
}

// out[i, 0:dim] = feat[row(i), soff : soff + min(sdim, dim)], zeros elsewhere / for unknown edges (get_edge_dense_feature_op.cc:60-70)
__global__ void k_edge_feature(DevEdges e, const long long* __restrict__ rows, int64_t E, int32_t dim, int32_t soff, int32_t sdim,
                               float* __restrict__ out) {
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t i = tid / dim;
  if (i >= E) return;
  const int32_t d = (int32_t)(tid - i * dim);
  const long long r = rows[i];
  out[tid] = (r >= 0 && d < sdim) ? e.feat[r * (int64_t)e.feat_dim + soff + d] : 0.f;
}

template <bool SPARSE>
__global__ void k_edge_ragged_len(DevEdges e, const long long* __restrict__ rows, int64_t E, int32_t fid, long long* __restrict__ out_ptr) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i == 0) out_ptr[0] = 0;
  if (i >= E) return;
  const long long r = rows[i];
  const int64_t* ptr = SPARSE ? e.u64_ptr : e.bin_ptr;
  const int32_t S = SPARSE ? e.n_u64_slots : e.n_bin_slots;
  long long len = 0;
  if (r >= 0 && fid >= 0 && fid < S && ptr) len = ptr[r * S + fid + 1] - ptr[r * S + fid];
  if (SPARSE && len == 0) len = 1;   // one default entry, as for nodes
  out_ptr[i + 1] = len;
}

template <bool SPARSE>
__global__ void k_edge_ragged_fill(DevEdges e, const long long* __restrict__ rows, int64_t E, int32_t fid, long long default_value,
                                   const long long* __restrict__ out_ptr, int64_t cap, long long* __restrict__ out_values,
                                   unsigned char* __restrict__ out_bytes) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= E) return;
  const long long r = rows[i];
  const int64_t* ptr = SPARSE ? e.u64_ptr : e.bin_ptr;
  const int32_t S = SPARSE ? e.n_u64_slots : e.n_bin_slots;
  int64_t b = 0, en = 0;
  if (r >= 0 && fid >= 0 && fid < S && ptr) { b = ptr[r * S + fid]; en = ptr[r * S + fid + 1]; }
  const int64_t o = out_ptr[i];
  if (SPARSE && en == b) { if (o < cap) out_values[o] = default_value; return; }
  for (int64_t k = 0; k < en - b; ++k) {
    if (o + k >= cap) break;
    if (SPARSE) out_values[o + k] = (long long)e.u64_val[b + k]; else out_bytes[o + k] = e.bin_val[b + k];
  }
}

// AliasMethod::Next over the edges of one type (alias_method.cc:66-78), 2 uniforms per draw; out[j] = (src, dst, type)
template <bool PHILOX>
__global__ void k_sample_edge(DevEdges e, const int64_t* __restrict__ order, const float* __restrict__ prob, const int32_t* __restrict__ alias,
                              long long n, int32_t count, unsigned long long key, EuRngState* rng, long long* __restrict__ out) {
  const int32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= count) return;
  double u1, u2;
  if (PHILOX) philox_uniform2(0x45444745ull, (uint32_t)j, (uint32_t)rng->calls, key, u1, u2);
  else {
    uint32_t x = modmul(rng->x, modpow_a(4ull * (unsigned long long)j));
    u1 = minstd_uniform(x);
    u2 = minstd_uniform(x);
  }
  long long col = (long long)floor(__dmul_rn((double)n, u1));
  const bool coin = u2 < (double)__ldg(prob + col);
  if (!coin) col = (long long)__ldg(alias + col);
  const int64_t r = order[col];
  out[j * 3] = (long long)e.src[r]; out[j * 3 + 1] = (long long)e.dst[r]; out[j * 3 + 2] = e.type[r];
}

__global__ void k_advance_engine2(EuRngState* rng, unsigned long long uniforms) {
  rng->x = modmul(rng->x, modpow_a(2ull * uniforms));
  rng->draws += uniforms;
  rng->calls += 1;
}

void fwc_build_public(const std::vector<float>& w, std::vector<float>* prob, std::vector<int32_t>* alias, float* sum);

template <typename T>
static int up(eu_graph* g, const T** dst, const T* src, int64_t count) {
  T* p = nullptr;
  int rc = g->alloc(&p, count);
  if (rc) return rc;
  if (count > 0 && src) {
    cudaError_t e = cudaMemcpy(p, src, sizeof(T) * (size_t)count, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) { set_error("cudaMemcpy -> %s", cudaGetErrorString(e)); return EU_ERR_CUDA; }
  }
  *dst = p;
  return EU_OK;
}

static int edge_rows(eu_ctx* c, const int64_t* edges, int64_t E, long long** rows_out, int64_t extra_bytes, char** extra) {
  int rc = ctx_misc(c, 256 + 8 * std::max<int64_t>(E, 1) + extra_bytes + 256);
  if (rc) return rc;
  long long* rows = (long long*)((char*)c->d_misc + 256);
  if (extra) *extra = (char*)c->d_misc + 256 + ((8 * std::max<int64_t>(E, 1) + 255) & ~(int64_t)255);
  if (E > 0) {
    k_edge_rows<<<(unsigned)ceil_div(E, 256), 256, 0, c->stream>>>(c->g->e, (const long long*)edges, E, rows);
    EU_LAUNCHED();
  }
  *rows_out = rows;
  return EU_OK;
}

}  // namespace eu

using namespace eu;

extern "C" {

int eu_graph_set_edges(eu_graph* g, const eu_edge_desc* d) {
  if (!g || !d || d->n_edges < 0 || (d->n_edges > 0 && (!d->src || !d->dst || !d->type))) { set_error("eu_graph_set_edges: bad argument"); return EU_ERR_INVALID; }
  if (g->e.n > 0 || g->edges_set) { set_error("eu_graph_set_edges: edges are already attached"); return EU_ERR_STATE; }
  EU_CUDA(cudaSetDevice(g->device));
  DevEdges& e = g->e;
  const int64_t n = d->n_edges;
  int rc;
  if ((rc = up(g, (const uint64_t**)&e.src, d->src, n))) return rc;
  if ((rc = up(g, (const uint64_t**)&e.dst, d->dst, n))) return rc;
  if ((rc = up(g, &e.type, d->type, n))) return rc;
  std::vector<float> ones;
  if (!d->w) ones.assign((size_t)n, 1.0f);
  if ((rc = up(g, &e.w, d->w ? d->w : ones.data(), n))) return rc;
  e.feat_dim = d->feat ? d->feat_dim : 0;
  if (e.feat_dim > 0) {
    if ((rc = up(g, &e.feat, d->feat, n * (int64_t)e.feat_dim))) return rc;
    e.n_slots = d->n_feat_slots > 0 ? d->n_feat_slots : 1;
    if (e.n_slots > EU_MAX_FEAT_SLOTS) { set_error("eu_graph_set_edges: more than %d dense slots", EU_MAX_FEAT_SLOTS); return EU_ERR_UNSUPPORTED; }
    int32_t off = 0;
    for (int s = 0; s < e.n_slots; ++s) {
      const int32_t dm = d->n_feat_slots > 0 ? d->feat_slot_dims[s] : e.feat_dim;
      e.slot_off[s] = off; e.slot_dim[s] = dm; off += dm;
      g->edge_dense_names.push_back("feat" + std::to_string(s));
    }
    if (off != e.feat_dim) { set_error("eu_graph_set_edges: feat_dim != sum(feat_slot_dims)"); return EU_ERR_INVALID; }
  }
  if (d->n_u64_slots > 0 && d->u64_ptr) {
    e.n_u64_slots = d->n_u64_slots;
    if ((rc = up(g, &e.u64_ptr, d->u64_ptr, n * d->n_u64_slots + 1))) return rc;
    if ((rc = up(g, (const uint64_t**)&e.u64_val, d->u64_val, std::max<int64_t>(d->u64_ptr[n * d->n_u64_slots], 1)))) return rc;
    for (int s = 0; s < d->n_u64_slots; ++s) g->edge_sparse_names.push_back("u64_" + std::to_string(s));
  }
  if (d->n_bin_slots > 0 && d->bin_ptr) {
    e.n_bin_slots = d->n_bin_slots;
    if ((rc = up(g, &e.bin_ptr, d->bin_ptr, n * d->n_bin_slots + 1))) return rc;
    if ((rc = up(g, (const uint8_t**)&e.bin_val, d->bin_val, std::max<int64_t>(d->bin_ptr[n * d->n_bin_slots], 1)))) return rc;
    for (int s = 0; s < d->n_bin_slots; ++s) g->edge_binary_names.push_back("bin_" + std::to_string(s));
  }
  // (src, dst, type) -> row; a later duplicate is ignored like edge_map_.insert (graph.cc:197-203)
  unsigned long long cap = 64;
  while (cap < (unsigned long long)n * 2) cap <<= 1;
  std::vector<EdgeSlot> tab((size_t)cap);
  for (auto& s : tab) { s.src = 0; s.dst = 0; s.type = 0; s.pad = 0; s.row = -1; }
  for (int64_t r = 0; r < n; ++r) {
    unsigned long long h = edge_hash_host(d->src[r], d->dst[r], d->type[r]) & (cap - 1);
    bool dup = false;
    while (tab[h].row >= 0) {
      if (tab[h].src == d->src[r] && tab[h].dst == d->dst[r] && tab[h].type == d->type[r]) { dup = true; break; }
      h = (h + 1) & (cap - 1);
    }
    if (!dup) { tab[h].src = d->src[r]; tab[h].dst = d->dst[r]; tab[h].type = d->type[r]; tab[h].row = r; }
  }
  if ((rc = up(g, &e.htab, tab.data(), (int64_t)cap))) return rc;
  e.hmask = cap - 1;
  // per edge type an alias table over that type's edges, in sampler order (graph.cc:372-399; same float ops as for nodes)
  int32_t T = 0;
  for (int64_t r = 0; r < n; ++r) T = std::max(T, d->type[r] + 1);
  T = std::max(T, g->d.T);
  std::vector<std::vector<int64_t>> rows_t(T);
  std::vector<std::vector<float>> w_t(T);
  std::vector<float> sums(T, 0.f);
  for (int64_t k = 0; k < n; ++k) {
    const int64_t r = d->sampler_order ? d->sampler_order[k] : k;
    const int32_t t = d->type[r];
    if (t < 0) { set_error("eu_graph_set_edges: negative edge type"); return EU_ERR_INVALID; }
    const float w = d->w ? d->w[r] : 1.0f;
    rows_t[t].push_back(r); w_t[t].push_back(w); sums[t] += w;
  }
  g->edge_samplers.resize(T);
  for (int32_t t = 0; t < T; ++t) {
    for (auto& x : w_t[t]) x /= sums[t];
    std::vector<float> prob; std::vector<int32_t> alias;
    eu_graph::EdgeSampler& s = g->edge_samplers[t];
    s.n = (int64_t)rows_t[t].size();
    fwc_build_public(w_t[t], &prob, &alias, &s.fwc_sum);
    if ((rc = up(g, (const int64_t**)&s.order, rows_t[t].data(), s.n))) return rc;
    if ((rc = up(g, (const float**)&s.prob, prob.data(), s.n))) return rc;
    if ((rc = up(g, (const int32_t**)&s.alias, alias.data(), s.n))) return rc;
  }
  e.n = n;
  g->edges_set = true;
  EU_CUDA(cudaDeviceSynchronize());
  return EU_OK;
}

int64_t eu_graph_num_edge_records(const eu_graph* g) { return g ? g->e.n : -1; }

int32_t eu_graph_edge_dense_feature_id(const eu_graph* g, const char* name) {
  if (!g || !name) return -1;
  for (size_t i = 0; i < g->edge_dense_names.size(); ++i) if (g->edge_dense_names[i] == name) return (int32_t)i;
  return -1;
}
int eu_graph_set_edge_dense_feature_name(eu_graph* g, int32_t fid, const char* name) {
  if (!g || !name || fid < 0 || fid >= (int32_t)g->edge_dense_names.size()) {
    set_error("eu_graph_set_edge_dense_feature_name: bad argument (slot %d)", (int)fid);
    return EU_ERR_INVALID;
  }
  g->edge_dense_names[fid] = name;
  return EU_OK;
}
int32_t eu_graph_edge_sparse_feature_id(const eu_graph* g, const char* name) {
  if (!g || !name) return -1;
  for (size_t i = 0; i < g->edge_sparse_names.size(); ++i) if (g->edge_sparse_names[i] == name) return (int32_t)i;
  return -1;
}
int32_t eu_graph_edge_binary_feature_id(const eu_graph* g, const char* name) {
  if (!g || !name) return -1;
  for (size_t i = 0; i < g->edge_binary_names.size(); ++i) if (g->edge_binary_names[i] == name) return (int32_t)i;
  return -1;
}

int eu_sample_edge(eu_ctx* c, int32_t count, const int32_t* types, int32_t n_types, int64_t* out) {
  if (!c || count < 0 || n_types < 1 || !types || (count > 0 && !out)) { set_error("eu_sample_edge: bad argument"); return EU_ERR_INVALID; }
  eu_graph* g = c->g;
  EU_CUDA(cudaSetDevice(g->device));
  if (!g->edges_set) { set_error("eu_sample_edge: no edges loaded (data_type must include edges)"); return EU_ERR_STATE; }
  if (n_types != 1 || types[0] == -1) {
    // graph.cc:284-287,316-324: the type is drawn from edge_type_collection_, which no code path of the reference ever
    // initialises -> GetSumWeight() == 0 -> empty result; there is nothing to be bit-exact with
    set_error("eu_sample_edge: sampling over several edge types returns nothing in the reference (edge_type_collection_ is never "
              "initialised, graph.cc:277-331); pass exactly one edge type");
    return EU_ERR_STATE;
  }
  const int32_t t = types[0];
  if (t < 0 || t >= (int32_t)g->edge_samplers.size()) { set_error("eu_sample_edge: edge type %d out of range", t); return EU_ERR_INVALID; }
  const eu_graph::EdgeSampler& s = g->edge_samplers[t];
  if (s.n == 0 || s.fwc_sum == 0.f) { set_error("eu_sample_edge: edge type %d has no edges", t); return EU_ERR_STATE; }
  if (count == 0) return EU_OK;
  const unsigned blocks = (unsigned)ceil_div(count, 256);
  if (c->rng == EU_RNG_PHILOX) k_sample_edge<true><<<blocks, 256, 0, c->stream>>>(g->e, s.order, s.prob, s.alias, s.n, count, c->seed, c->d_rng, (long long*)out);
  else k_sample_edge<false><<<blocks, 256, 0, c->stream>>>(g->e, s.order, s.prob, s.alias, s.n, count, c->seed, c->d_rng, (long long*)out);
  EU_LAUNCHED();
  k_advance_engine2<<<1, 1, 0, c->stream>>>(c->d_rng, 2ull * (unsigned long long)count);
  EU_LAUNCHED();
  return EU_OK;
}

int eu_get_edge_dense_feature(eu_ctx* c, const int64_t* edges, int64_t E, int32_t fid, int32_t dim, float* out) {
  if (!c || E < 0 || dim < 0 || (E > 0 && (!edges || (dim > 0 && !out)))) { set_error("eu_get_edge_dense_feature: bad argument"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  if (E == 0 || dim == 0) return EU_OK;
  const DevEdges& e = c->g->e;
  long long* rows = nullptr;
  int rc = edge_rows(c, edges, E, &rows, 0, nullptr);
  if (rc) return rc;
  const bool have = fid >= 0 && fid < e.n_slots;
  k_edge_feature<<<(unsigned)ceil_div(E * (int64_t)dim, 256), 256, 0, c->stream>>>(e, rows, E, dim, have ? e.slot_off[fid] : 0, have ? e.slot_dim[fid] : 0, out);
  EU_LAUNCHED();
  return EU_OK;
}

static int edge_ragged(eu_ctx* c, bool sparse, const int64_t* edges, int64_t E, int32_t fid, int64_t default_value, int64_t cap,
                       int64_t* out_ptr, int64_t* out_values, uint8_t* out_bytes, const char* what) {
  if (!c || E < 0 || cap < 0 || !out_ptr || (E > 0 && !edges) || (cap > 0 && !(sparse ? (void*)out_values : (void*)out_bytes))) { set_error("%s: bad argument", what); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  if (E >= ((int64_t)1 << 31)) { set_error("%s: more than 2^31 edges", what); return EU_ERR_UNSUPPORTED; }
  size_t tmp = 0;
  cub::DeviceScan::InclusiveSum((void*)nullptr, tmp, (long long*)nullptr, (long long*)nullptr, (int)(E + 1), c->stream);
  long long* rows = nullptr;
  char* extra = nullptr;
  int rc = edge_rows(c, edges, E, &rows, (int64_t)tmp + 256, &extra);
  if (rc) return rc;
  const DevEdges& e = c->g->e;
  const unsigned blocks = (unsigned)ceil_div(std::max<int64_t>(E, 1), 256);
  if (sparse) k_edge_ragged_len<true><<<blocks, 256, 0, c->stream>>>(e, rows, E, fid, (long long*)out_ptr);
  else k_edge_ragged_len<false><<<blocks, 256, 0, c->stream>>>(e, rows, E, fid, (long long*)out_ptr);
  EU_LAUNCHED();
  EU_CUDA(cub::DeviceScan::InclusiveSum(extra, tmp, (long long*)out_ptr, (long long*)out_ptr, (int)(E + 1), c->stream));
  EU_LAUNCHED();
  if (cap > 0 && E > 0) {
    if (sparse) k_edge_ragged_fill<true><<<blocks, 256, 0, c->stream>>>(e, rows, E, fid, (long long)default_value, (const long long*)out_ptr, cap, (long long*)out_values, nullptr);
    else k_edge_ragged_fill<false><<<blocks, 256, 0, c->stream>>>(e, rows, E, fid, 0, (const long long*)out_ptr, cap, nullptr, out_bytes);
    EU_LAUNCHED();
  }
  return EU_OK;
}

int eu_get_edge_sparse_feature(eu_ctx* c, const int64_t* edges, int64_t E, int32_t fid, int64_t default_value, int64_t cap, int64_t* out_ptr,
                               int64_t* out_values) {
  return edge_ragged(c, true, edges, E, fid, default_value, cap, out_ptr, out_values, nullptr, "eu_get_edge_sparse_feature");
}
int eu_get_edge_binary_feature(eu_ctx* c, const int64_t* edges, int64_t E, int32_t fid, int64_t cap, int64_t* out_ptr, uint8_t* out_bytes) {
  return edge_ragged(c, false, edges, E, fid, 0, cap, out_ptr, nullptr, out_bytes, "eu_get_edge_binary_feature");
}

}  // extern "C"
