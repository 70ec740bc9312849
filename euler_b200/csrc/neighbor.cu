// Full-neighbor listing on the HBM-resident CSR (SURVEY.md section 8f, row next-1).
// Reference semantics reproduced (file:line relative to /root/reference):
//   Node::GetFullNeighbor        euler/core/graph/node.cc:176-198  -- per requested edge type, in the order given
//                                (repeats repeat), every edge of that group as (id, weight, type)
//   euler::GetFullNeighbor       euler/core/api/api.cc:208-221     -- per node, missing node -> empty list
//   tf_euler GetFullNeighbor     tf_euler/kernels/get_full_neighbor_op.cc -- CSR-style (ragged) result
// Weights: the reference stores node-global cumulative weights and returns cum[j] - cum[j-1] (f32); same here.
//
// Three kernels, no host sync: per-node lengths -> cub inclusive scan -> one warp per node copies its groups.
#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_sort.cuh>
#include <cub/iterator/counting_input_iterator.cuh>
#include <cub/iterator/transform_input_iterator.cuh>

#include "internal.h"

namespace eu {

__global__ void k_full_len(DevGraph g, const unsigned long long* __restrict__ nodes, int64_t B, ETList et,
                           long long* __restrict__ out_ptr /* [B+1]; [0] = 0, [i+1] = len(i) */) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i == 0) out_ptr[0] = 0;
  if (i >= B) return;
  const int64_t row = lookup_row(g, nodes[i]);
  long long len = 0;
  if (row >= 0) {
    const int64_t* gp = g.grp_ptr + row * g.T;
    for (int32_t k = 0; k < et.K; ++k) {
      const int32_t t = et.v[k];
      if (t >= 0 && t < g.T) len += gp[t + 1] - gp[t];
    }
  }
  out_ptr[i + 1] = len;
}

__global__ void __launch_bounds__(256) k_full_fill(DevGraph g, const unsigned long long* __restrict__ nodes, int64_t B, ETList et,
                                                   const long long* __restrict__ out_ptr, int64_t cap,
                                                   unsigned long long* __restrict__ out_ids, float* __restrict__ out_w,
                                                   int32_t* __restrict__ out_t) {
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; i < B; i += nwarps) {
    const int64_t row = lookup_row(g, nodes[i]);
    if (row < 0) continue;
    const int64_t* gp = g.grp_ptr + row * g.T;
    const int64_t base = gp[0];
    int64_t o = out_ptr[i];
    for (int32_t k = 0; k < et.K; ++k) {
      const int32_t t = et.v[k];
      if (t < 0 || t >= g.T) continue;
      const int64_t b = gp[t], e = gp[t + 1];
      for (int64_t j = b + lane; j < e; j += 32) {
        const int64_t pos = o + (j - b);
        if (pos < cap) {
          out_ids[pos] = g.nbr[j];
          out_w[pos] = __fsub_rn(g.cum_w[j], j == base ? 0.f : g.cum_w[j - 1]);
          out_t[pos] = t;
        }
      }
      o += e - b;
    }
  }
}

// euler::GetNodeType (api.cc:50-61): the node's type, DEFAULT_INT32 (= INT32_MIN, data_types.cc:23) when the node is absent
__global__ void k_node_type(DevGraph g, const unsigned long long* __restrict__ nodes, int64_t B, int32_t* __restrict__ out) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= B) return;
  const int64_t row = lookup_row(g, nodes[i]);
  out[i] = row >= 0 ? g.node_type[row] : (int32_t)0x80000000;
}

__global__ void k_node_weight(DevGraph g, const unsigned long long* __restrict__ nodes, int64_t B, float* __restrict__ out) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= B) return;
  const int64_t row = lookup_row(g, nodes[i]);
  out[i] = row >= 0 ? g.node_w[row] : 0.f;
}

// ---- sorted / top-k listings (tf_euler get_sorted_full_neighbor / get_top_k_neighbor): the full listing above, then a
// STABLE segmented sort per node (cub::DeviceSegmentedSort) and a gather.
struct ClampOffset {   // segment bound clipped to the number of entries that were actually written
  const long long* ptr; long long cap;
  __host__ __device__ long long operator()(long long i) const { const long long v = ptr[i]; return v < cap ? v : cap; }
};

__global__ void k_iota(long long* __restrict__ a, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) a[i] = i;
}

__global__ void k_permute_wt(const long long* __restrict__ idx, const unsigned long long* __restrict__ ids, const float* __restrict__ w,
                             const int32_t* __restrict__ t, int64_t n, unsigned long long* __restrict__ o_ids, float* __restrict__ o_w,
                             int32_t* __restrict__ o_t) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const long long k = idx[i];
    if (o_ids) o_ids[i] = ids[k];
    o_w[i] = w[k];
    o_t[i] = t[k];
  }
}

// [B, k] dense outputs: the first min(k, len) entries of every node's (sorted) listing, the rest default_node / 0.0 / -1
// (tf_euler/kernels/get_top_k_neighbor_op.cc:75-77,105-114)
__global__ void k_topk_pack(const long long* __restrict__ ptr, const long long* __restrict__ idx, const unsigned long long* __restrict__ ids,
                            const float* __restrict__ w, const int32_t* __restrict__ t, int64_t B, int32_t k, long long default_node,
                            long long* __restrict__ o_ids, float* __restrict__ o_w, int32_t* __restrict__ o_t) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= B * (int64_t)k) return;
  const int64_t r = i / k, j = i - r * k;
  const long long b = ptr[r], e = ptr[r + 1];
  if (b + j < e) {
    const long long s = idx[b + j];
    o_ids[i] = (long long)ids[s]; o_w[i] = w[s]; o_t[i] = t[s];
  } else {
    o_ids[i] = default_node; o_w[i] = 0.f; o_t[i] = -1;
  }
}

}  // namespace eu

using namespace eu;

extern "C" int eu_get_node_type(eu_ctx* c, const int64_t* nodes, int64_t B, int32_t* out) {
  if (!c || B < 0 || (B > 0 && (!nodes || !out))) { set_error("eu_get_node_type: bad argument"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  if (B == 0) return EU_OK;
  k_node_type<<<(unsigned)ceil_div(B, 256), 256, 0, c->stream>>>(c->g->d, (const unsigned long long*)nodes, B, out);
  EU_LAUNCHED();
  return EU_OK;
}

// Node::GetWeight (euler/core/graph/node.h:78) of every node, 0.0 for ids that are not in the graph: the device side of
// eu_get_node_weight_host, which has no device entry point of its own
int eu::get_node_weight(eu_ctx* c, const int64_t* nodes, int64_t B, float* out) {
  if (B == 0) return EU_OK;
  k_node_weight<<<(unsigned)ceil_div(B, 256), 256, 0, c->stream>>>(c->g->d, (const unsigned long long*)nodes, B, out);
  EU_LAUNCHED();
  return EU_OK;
}

extern "C" int eu_get_full_neighbor(eu_ctx* c, const int64_t* nodes, int64_t B, const int32_t* etypes, int32_t K,
                                    int64_t cap, int64_t* out_ptr, int64_t* out_ids, float* out_w, int32_t* out_t) {
  if (!c || B < 0 || K < 0 || K > EU_MAX_ETYPES || cap < 0 || !out_ptr || (B > 0 && !nodes) || (K > 0 && !etypes) ||
      (cap > 0 && (!out_ids || !out_w || !out_t))) {
    set_error("eu_get_full_neighbor: bad argument");
    return EU_ERR_INVALID;
  }
  EU_CUDA(cudaSetDevice(c->g->device));
  const DevGraph& d = c->g->d;
  ETList et{};
  et.K = K;
  for (int32_t k = 0; k < K; ++k) et.v[k] = etypes[k];
  cudaStream_t s = c->stream;
  size_t tmp = 0;
  cub::DeviceScan::InclusiveSum((void*)nullptr, tmp, (long long*)nullptr, (long long*)nullptr, (int)(B + 1), s);
  int rc = ctx_misc(c, (int64_t)tmp + 256);
  if (rc) return rc;
  { EuProfScope ps(c, "k_full_len", B);
    k_full_len<<<(unsigned)ceil_div(std::max<int64_t>(B, 1), 256), 256, 0, s>>>(d, (const unsigned long long*)nodes, B, et, (long long*)out_ptr); }
  EU_LAUNCHED();
  EU_CUDA(cub::DeviceScan::InclusiveSum(c->d_misc, tmp, (long long*)out_ptr, (long long*)out_ptr, (int)(B + 1), s));
  EU_LAUNCHED();
  if (cap > 0 && B > 0) {
    EuProfScope ps(c, "k_full_fill", B);
    const unsigned blocks = (unsigned)std::min<int64_t>(ceil_div(B * 32, 256), kSMs * 8);
    k_full_fill<<<blocks, 256, 0, s>>>(d, (const unsigned long long*)nodes, B, et, (const long long*)out_ptr, cap,
                                       (unsigned long long*)out_ids, out_w, out_t);
    EU_LAUNCHED();
  }
  return EU_OK;
}

// tf_euler.get_sorted_full_neighbor (tf_euler/python/euler_ops/neighbor_ops.py:100-119; engine: API_GET_NB_NODE with
// "order_by id asc", euler/core/kernels/get_neighbor_op.cc:128-141; Node::GetSortedFullNeighbor node.cc:210-262): the
// full listing of every node ordered by neighbor id (unsigned) ascending.  Ties (the same neighbor under several edge
// types, multi-edges) keep the listing order: the engine's comparator `a <= b` is not a strict weak order, so its
// std::sort is undefined for equal ids -- stable is the definition here; with distinct ids the results are identical.
// Same calling convention as eu_get_full_neighbor (cap = 0: lengths only); cap must cover the whole listing.
extern "C" int eu_get_sorted_full_neighbor(eu_ctx* c, const int64_t* nodes, int64_t B, const int32_t* etypes, int32_t K,
                                           int64_t cap, int64_t* out_ptr, int64_t* out_ids, float* out_w, int32_t* out_t) {
  int rc = eu_get_full_neighbor(c, nodes, B, etypes, K, cap, out_ptr, out_ids, out_w, out_t);
  if (rc || cap == 0 || B == 0) return rc;
  if (cap >= ((int64_t)1 << 31) || B >= ((int64_t)1 << 31)) { set_error("eu_get_sorted_full_neighbor: more than 2^31 entries"); return EU_ERR_UNSUPPORTED; }
  cudaStream_t s = c->stream;
  ClampOffset f{(const long long*)out_ptr, (long long)cap};
  cub::CountingInputIterator<long long> cnt(0);
  cub::TransformInputIterator<long long, ClampOffset, cub::CountingInputIterator<long long>> seg(cnt, f);
  size_t tmp = 0;
  cub::DeviceSegmentedSort::StableSortPairs((void*)nullptr, tmp, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                            (const long long*)nullptr, (long long*)nullptr, (int)cap, (int)B, seg, seg + 1, s);
  tmp = (tmp + 255) & ~(size_t)255;
  // scratch: keys_out 8n | idx 8n | idx_out 8n | w 4n | t 4n | cub temp   (own allocation: ctx_misc is in use by the listing)
  char* buf = nullptr;
  const size_t n = (size_t)cap;
  EU_CUDA(cudaMalloc(&buf, 32 * n + 1024 + tmp));
  unsigned long long* keys_out = (unsigned long long*)buf;
  long long* idx = (long long*)(buf + 8 * n);
  long long* idx_out = (long long*)(buf + 16 * n);
  float* w2 = (float*)(buf + 24 * n);
  int32_t* t2 = (int32_t*)(buf + 28 * n);
  void* cubtmp = buf + ((32 * n + 255) & ~(size_t)255);
  k_iota<<<kSMs * 4, 256, 0, s>>>(idx, cap);
  g_launches++;
  cudaError_t e = cub::DeviceSegmentedSort::StableSortPairs(cubtmp, tmp, (const unsigned long long*)out_ids, keys_out, (const long long*)idx, idx_out,
                                                            (int)cap, (int)B, seg, seg + 1, s);
  g_launches++;
  if (e == cudaSuccess) {
    k_permute_wt<<<kSMs * 4, 256, 0, s>>>(idx_out, (const unsigned long long*)out_ids, out_w, out_t, cap, nullptr, w2, t2);
    g_launches++;
    // entries past the listing (cap > total) were never sorted: copy back only what the segments cover is not known on the
    // host, so copy everything -- positions outside every segment hold their own (unsorted, unspecified) values either way
    cudaMemcpyAsync(out_ids, keys_out, 8 * n, cudaMemcpyDeviceToDevice, s);
    cudaMemcpyAsync(out_w, w2, 4 * n, cudaMemcpyDeviceToDevice, s);
    cudaMemcpyAsync(out_t, t2, 4 * n, cudaMemcpyDeviceToDevice, s);
    e = cudaStreamSynchronize(s);
  }
  cudaFree(buf);
  if (e != cudaSuccess) { set_error("eu_get_sorted_full_neighbor: %s", cudaGetErrorString(e)); return EU_ERR_CUDA; }
  return EU_OK;
}

// tf_euler.get_top_k_neighbor (neighbor_ops.py:44-46; kernel tf_euler/kernels/get_top_k_neighbor_op.cc:54-121; engine:
// "order_by weight desc, limit k", get_neighbor_op.cc:142-165): per node the k heaviest edges of the requested types,
// heaviest first, as dense [B, k] arrays filled with default_node / 0.0 / -1.  Equal weights keep the listing order (the
// engine's std::sort is unstable; for listings of up to 16 entries -- libstdc++'s insertion-sort range -- and whenever the
// weights differ the results are identical).  Sizes its scratch from the listing length: synchronises the stream once.
extern "C" int eu_get_top_k_neighbor(eu_ctx* c, const int64_t* nodes, int64_t B, const int32_t* etypes, int32_t K, int32_t k,
                                     int64_t default_node, int64_t* out_ids, float* out_w, int32_t* out_t) {
  if (!c || B < 0 || k < 0 || (B > 0 && k > 0 && (!nodes || !out_ids || !out_w || !out_t))) { set_error("eu_get_top_k_neighbor: bad argument"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  if (B == 0 || k == 0) return EU_OK;
  if (B >= ((int64_t)1 << 31)) { set_error("eu_get_top_k_neighbor: more than 2^31 nodes"); return EU_ERR_UNSUPPORTED; }
  cudaStream_t s = c->stream;
  long long* ptr = nullptr;
  EU_CUDA(cudaMalloc(&ptr, 8 * (size_t)(B + 1)));
  int rc = eu_get_full_neighbor(c, nodes, B, etypes, K, 0, (int64_t*)ptr, nullptr, nullptr, nullptr);
  long long total = 0;
  if (!rc && (cudaMemcpyAsync(&total, ptr + B, 8, cudaMemcpyDeviceToHost, s) != cudaSuccess || cudaStreamSynchronize(s) != cudaSuccess)) rc = EU_ERR_CUDA;
  if (!rc && total >= ((long long)1 << 31)) { set_error("eu_get_top_k_neighbor: more than 2^31 entries"); rc = EU_ERR_UNSUPPORTED; }
  char* buf = nullptr;
  if (!rc) {
    const size_t n = (size_t)std::max<long long>(total, 1);
    size_t tmp = 0;
    cub::DeviceSegmentedSort::StableSortPairsDescending((void*)nullptr, tmp, (const float*)nullptr, (float*)nullptr, (const long long*)nullptr,
                                                        (long long*)nullptr, (int)n, (int)B, ptr, ptr + 1, s);
    tmp = (tmp + 255) & ~(size_t)255;
    // ids 8n | w 4n | t 4n | w_sorted 4n (+4n pad) | idx 8n | idx_out 8n | cub temp
    if (cudaMalloc(&buf, 40 * n + 1024 + tmp) != cudaSuccess) { set_error("eu_get_top_k_neighbor: cudaMalloc failed"); rc = EU_ERR_CUDA; }
    if (!rc) {
      unsigned long long* ids = (unsigned long long*)buf;
      float* w = (float*)(buf + 8 * n);
      int32_t* t = (int32_t*)(buf + 12 * n);
      float* ws = (float*)(buf + 16 * n);
      long long* idx = (long long*)(buf + 24 * n);
      long long* idx_out = (long long*)(buf + 32 * n);
      void* cubtmp = buf + ((40 * n + 255) & ~(size_t)255);
      if (total > 0) {
        rc = eu_get_full_neighbor(c, nodes, B, etypes, K, total, (int64_t*)ptr, (int64_t*)ids, w, t);
        if (!rc) {
          k_iota<<<kSMs * 4, 256, 0, s>>>(idx, total);
          g_launches++;
          cudaError_t e = cub::DeviceSegmentedSort::StableSortPairsDescending(cubtmp, tmp, (const float*)w, ws, (const long long*)idx, idx_out,
                                                                              (int)total, (int)B, ptr, ptr + 1, s);
          g_launches++;
          if (e != cudaSuccess) { set_error("eu_get_top_k_neighbor: %s", cudaGetErrorString(e)); rc = EU_ERR_CUDA; }
        }
      }
      if (!rc) {
        k_topk_pack<<<(unsigned)ceil_div(B * (int64_t)k, 256), 256, 0, s>>>(ptr, idx_out, ids, w, t, B, k, (long long)default_node,
                                                                           (long long*)out_ids, out_w, out_t);
        g_launches++;
        if (cudaStreamSynchronize(s) != cudaSuccess) { set_error("eu_get_top_k_neighbor: %s", cudaGetErrorString(cudaGetLastError())); rc = EU_ERR_CUDA; }
      }
    }
  }
  cudaFree(buf); cudaFree(ptr);
  return rc;
}
