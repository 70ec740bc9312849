// Graph-level minibatches: the graph-label table of a graph, sample_graph_label and get_graph_by_label.
//
// Reference semantics (file:line relative to /root/reference):
//   Graph::GetGraphLabel        euler/core/graph/graph.cc:439-457 (an unordered_set over node_map_, one value per node)
//   SampleGraphLabelOp          euler/core/kernels/sample_graph_label_op.cc (floor(ThreadLocalRandom() * L) per draw)
//   GetGraphByLabelOp           euler/core/kernels/get_graph_by_label_op.cc + tf_euler/kernels/get_graph_by_label_op.cc
//                               (row i lists the nodes of graph i; an unknown or empty one gets the single entry (i, 0) = 0)
//
// The nodes of a label come from the reference's hash index on `graph_label`, which the converter builds from the values
// present (euler/tools/json2partindex.py:131-146): the label "" lists no nodes.  Its row order is that of the index file; here
// a graph's node ids are listed in ascending order, a chosen order (only float summation order downstream depends on it).
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <unordered_map>
#include <unordered_set>

#include "segment.cuh"

namespace eu {

void graph_label_list(const std::vector<int64_t>& order, int64_t n, const int64_t* bin_ptr, const uint8_t* bin_val, int32_t S,
                      int32_t fid, std::vector<std::string>* labels, std::vector<int32_t>* row_label) {
  auto value = [&](int64_t r) {   // Node::GetBinaryFeature: the slot's bytes, "" for a node without them
    const int64_t b = bin_ptr[r * S + fid], e = bin_ptr[r * S + fid + 1];
    return std::string((const char*)bin_val + b, (size_t)(e - b));
  };
  // the same container from the same libstdc++, fed the same sequence, iterates in the same order
  std::unordered_set<std::string> set;
  for (int64_t i = 0; i < n; ++i) set.insert(value(order.empty() ? i : order[i]));
  labels->assign(set.begin(), set.end());
  if (!row_label) return;
  std::unordered_map<std::string, int32_t> index;
  for (size_t l = 0; l < labels->size(); ++l) index.emplace((*labels)[l], (int32_t)l);
  const int32_t L = (int32_t)labels->size();
  row_label->resize(n);
  for (int64_t r = 0; r < n; ++r) {
    const std::string v = value(r);
    (*row_label)[r] = v.empty() ? L : index[v];
  }
}

int graph_build_labels(eu_graph* g) {
  if (g->labels_built) return EU_OK;
  const DevGraph& d = g->d;
  int32_t fid = -1;
  for (size_t k = 0; k < g->binary_feature_names.size(); ++k)
    if (g->binary_feature_names[k] == "graph_label") fid = (int32_t)k;
  if (fid < 0 || d.n_bin_slots <= fid || !d.bin_ptr) {
    set_error("graph label set is empty! (the graph has no binary feature slot 'graph_label')");
    return EU_ERR_STATE;
  }
  if (d.n >= ((int64_t)1 << 31)) { set_error("graph labels: 2^31 or more nodes are not supported"); return EU_ERR_UNSUPPORTED; }
  EU_CUDA(cudaSetDevice(g->device));
  const int64_t n = d.n, S = d.n_bin_slots;
  std::vector<int64_t> ptr(n * S + 1);
  EU_CUDA(cudaMemcpy(ptr.data(), d.bin_ptr, sizeof(int64_t) * ptr.size(), cudaMemcpyDeviceToHost));
  std::vector<uint8_t> val((size_t)ptr[n * S]);
  if (!val.empty()) EU_CUDA(cudaMemcpy(val.data(), d.bin_val, val.size(), cudaMemcpyDeviceToHost));
  std::vector<std::string> labels;
  std::vector<int32_t> row_label;
  graph_label_list(g->sampler_order, n, ptr.data(), val.data(), (int32_t)S, fid, &labels, &row_label);
  if (labels.empty()) { set_error("graph label set is empty! (the graph has no nodes)"); return EU_ERR_STATE; }
  const int64_t L = (int64_t)labels.size();
  // rows sorted by (label, node id): a stable sort by label of the rows sorted by id; rows without a label (key L) go last
  int32_t *lab = nullptr, *lab2 = nullptr;
  unsigned long long *ids2 = nullptr;
  void* tmp = nullptr;
  size_t t1 = 0, t2 = 0;
  cub::DeviceRadixSort::SortPairs((void*)nullptr, t1, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                  (const int32_t*)nullptr, (int32_t*)nullptr, (int)n);
  cub::DeviceRadixSort::SortPairs((void*)nullptr, t2, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                  (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)n, 0, radix_bits(L + 1));
  int rc;
  if ((rc = g->alloc(&g->d_label_ptr, L + 1))) return rc;
  if ((rc = g->alloc(&g->d_label_ids, n))) return rc;
  cudaError_t e = cudaSuccess;
  auto ok = [&](cudaError_t x) { if (e == cudaSuccess) e = x; return e == cudaSuccess; };
  if (ok(cudaMalloc(&lab, 4 * (size_t)std::max<int64_t>(n, 1))) && ok(cudaMalloc(&lab2, 4 * (size_t)std::max<int64_t>(n, 1))) &&
      ok(cudaMalloc(&ids2, 8 * (size_t)std::max<int64_t>(n, 1))) && ok(cudaMalloc(&tmp, std::max<size_t>(std::max(t1, t2), 1))) &&
      ok(cudaMemcpy(lab, row_label.data(), 4 * (size_t)n, cudaMemcpyHostToDevice)) &&
      ok(cub::DeviceRadixSort::SortPairs(tmp, t1, d.ids, ids2, lab, lab2, (int)n)) &&
      ok(cub::DeviceRadixSort::SortPairs(tmp, t2, (const uint32_t*)lab2, (uint32_t*)lab, ids2, g->d_label_ids, (int)n, 0,
                                         radix_bits(L + 1)))) {
    k_seg_starts<<<stride_grid(L + 1), 256>>>(lab, n, L, g->d_label_ptr);
    g_launches += 3;
    ok(cudaGetLastError()) && ok(cudaDeviceSynchronize());
  }
  cudaFree(lab); cudaFree(lab2); cudaFree(ids2); cudaFree(tmp);
  if (e != cudaSuccess) { set_error("graph labels: %s", cudaGetErrorString(e)); return EU_ERR_CUDA; }
  g->labels = std::move(labels);
  g->labels_built = true;
  return EU_OK;
}

// one label per draw: idx = floor(u * L), u one ThreadLocalRandom() draw (minstd: draw j of the stream; Philox: the
// counter (tag, j) under the call's salt)
template <bool PHILOX>
__global__ void k_sample_graph_label(int32_t count, int64_t L, unsigned long long key, const EuRngState* __restrict__ rng,
                                     int32_t* __restrict__ out) {
  const int32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= count) return;
  double u, u1;
  if (PHILOX) {
    philox_uniform2(0x47524C42ull, (uint32_t)j, (uint32_t)rng->calls, key, u, u1);
  } else {
    uint32_t x = modmul(rng->x, modpow_a(2ull * (unsigned long long)j));
    u = minstd_uniform(x);
  }
  const int64_t idx = (int64_t)floor(__dmul_rn(u, (double)L));
  // u < 1, but u * L can round up to L for a large L: the reference would index past its label vector; clamp instead
  out[j] = (int32_t)(idx < L ? idx : L - 1);
}

// pass 1: len[i] = the entries of graph i (its nodes, or 1: the (i, 0) = 0 entry of an unknown or empty label); len[B] = 0
__global__ void k_label_lengths(const int32_t* __restrict__ labels, int64_t B, int64_t L, const int32_t* __restrict__ lptr,
                                long long* __restrict__ len) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i <= B; i += (int64_t)gridDim.x * blockDim.x) {
    long long n = 0;
    if (i < B) {
      const int32_t l = __ldg(labels + i);
      n = (l >= 0 && l < L) ? __ldg(lptr + l + 1) - __ldg(lptr + l) : 0;
      if (n == 0) n = 1;
    }
    len[i] = n;
  }
}

// pass 2: a warp per graph i copies its label's node ids to values[ptr[i] ...) and writes indices (i, j); coalesced
__global__ void k_label_fill(const int32_t* __restrict__ labels, int64_t B, int64_t L, const int32_t* __restrict__ lptr,
                             const unsigned long long* __restrict__ lids, const long long* __restrict__ ptr, int64_t cap,
                             long long* __restrict__ indices, long long* __restrict__ values) {
  const int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (i >= B) return;
  const int32_t l = __ldg(labels + i);
  const long long o = __ldg(ptr + i);
  const long long b = (l >= 0 && l < L) ? __ldg(lptr + l) : 0, e = (l >= 0 && l < L) ? __ldg(lptr + l + 1) : 0;
  if (b == e) {
    if (lane == 0 && o < cap) { indices[2 * o] = i; indices[2 * o + 1] = 0; values[o] = 0; }
    return;
  }
  for (long long j = lane; j < e - b && o + j < cap; j += 32) {
    indices[2 * (o + j)] = i;
    indices[2 * (o + j) + 1] = j;
    values[o + j] = (long long)__ldg(lids + b + j);
  }
}

}  // namespace eu

using namespace eu;

extern "C" {

int eu_graph_set_binary_feature_name(eu_graph* g, int32_t fid, const char* name) {
  if (!g || !name || fid < 0 || fid >= (int32_t)g->binary_feature_names.size()) {
    set_error("eu_graph_set_binary_feature_name: bad argument (slot %d)", (int)fid);
    return EU_ERR_INVALID;
  }
  if (g->labels_built) { set_error("eu_graph_set_binary_feature_name: the graph-label table is already built"); return EU_ERR_STATE; }
  g->binary_feature_names[fid] = name;
  return EU_OK;
}

int eu_graph_labels(eu_graph* g, int64_t cap, int64_t* n_labels, int64_t* n_bytes, int64_t* ptr, uint8_t* bytes) {
  if (!g) { set_error("eu_graph_labels: bad argument"); return EU_ERR_INVALID; }
  int rc = graph_build_labels(g);
  if (rc) return rc;
  const std::vector<std::string>& L = g->labels;
  int64_t total = 0;
  if (ptr) ptr[0] = 0;
  for (size_t l = 0; l < L.size(); ++l) {
    if (bytes && total + (int64_t)L[l].size() <= cap) memcpy(bytes + total, L[l].data(), L[l].size());
    total += (int64_t)L[l].size();
    if (ptr) ptr[l + 1] = total;
  }
  if (n_labels) *n_labels = (int64_t)L.size();
  if (n_bytes) *n_bytes = total;
  return EU_OK;
}

int eu_sample_graph_label(eu_ctx* c, int32_t count, int32_t* out) {
  if (!c || count < 0 || (count > 0 && !out)) { set_error("eu_sample_graph_label: bad argument"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  int rc = graph_build_labels(c->g);
  if (rc) return rc;
  if (count == 0) return EU_OK;
  const int64_t L = (int64_t)c->g->labels.size();
  const unsigned blocks = (unsigned)ceil_div(count, 256);
  if (c->rng == EU_RNG_PHILOX) k_sample_graph_label<true><<<blocks, 256, 0, c->stream>>>(count, L, c->seed, c->d_rng, out);
  else k_sample_graph_label<false><<<blocks, 256, 0, c->stream>>>(count, L, c->seed, c->d_rng, out);
  EU_LAUNCHED();
  k_advance_engine<<<1, 1, 0, c->stream>>>(c->d_rng, (unsigned long long)count);
  EU_LAUNCHED();
  return EU_OK;
}

int eu_get_graph_by_label(eu_ctx* c, const int32_t* labels, int64_t B, int64_t cap, int64_t* ptr, int64_t* indices,
                          int64_t* values, int64_t* total, int64_t* max_len) {
  if (!c || B < 0 || cap < 0 || !ptr || (B > 0 && !labels) || (cap > 0 && (!indices || !values))) {
    set_error("eu_get_graph_by_label: bad argument");
    return EU_ERR_INVALID;
  }
  if (B >= ((int64_t)1 << 31)) { set_error("eu_get_graph_by_label: 2^31 or more graphs are not supported"); return EU_ERR_UNSUPPORTED; }
  EU_CUDA(cudaSetDevice(c->g->device));
  int rc = graph_build_labels(c->g);
  if (rc) return rc;
  eu_graph* g = c->g;
  const int64_t L = (int64_t)g->labels.size();
  cudaStream_t s = c->stream;
  if (cap > 0) {   // pass 2 over the offsets of pass 1
    if (B == 0) return EU_OK;
    EuProfScope ps(c, "graph_by_label_fill", B);
    k_label_fill<<<(unsigned)ceil_div(B * 32, 256), 256, 0, s>>>(labels, B, L, g->d_label_ptr, g->d_label_ids,
                                                                  (const long long*)ptr, cap, (long long*)indices, (long long*)values);
    EU_LAUNCHED();
    return EU_OK;
  }
  // pass 1: lengths -> exclusive scan into ptr [B + 1] -> (total, longest) read back in one synchronisation
  size_t scan = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, scan, (const long long*)nullptr, (long long*)nullptr, (int)(B + 1));
  const size_t o_len = 256, o_tmp = o_len + a256(8 * (size_t)(B + 1));
  if ((rc = ctx_misc(c, (int64_t)(o_tmp + scan)))) return rc;
  char* m = (char*)c->d_misc;
  long long* stats = (long long*)m;
  long long* len = (long long*)(m + o_len);
  EU_CUDA(cudaMemsetAsync(stats, 0, 16, s));
  k_label_lengths<<<stride_grid(B + 1), 256, 0, s>>>(labels, B, L, g->d_label_ptr, len);
  EU_LAUNCHED();
  EU_CUDA(cub::DeviceScan::ExclusiveSum(m + o_tmp, scan, len, (long long*)ptr, (int)(B + 1), s));
  EU_LAUNCHED();
  k_ragged_stats<<<stride_grid(B + 1), 256, 0, s>>>((const long long*)ptr, B, stats);
  EU_LAUNCHED();
  long long st[2] = {0, 0};
  EU_CUDA(cudaMemcpyAsync(st, stats, 16, cudaMemcpyDeviceToHost, s));
  EU_CUDA(cudaStreamSynchronize(s));
  if (total) *total = st[0];
  if (max_len) *max_len = st[1];
  return EU_OK;
}

}  // extern "C"
