// Ragged node features on the HBM-resident graph: uint64 ("sparse") and binary features (SURVEY.md section 8f, next-2).
// Reference semantics (file:line relative to /root/reference):
//   Node::GetUint64Feature / GetBinaryFeature   euler/core/graph/node.cc:330-409   slot s = [idx[s-1], idx[s]) of the node's array
//   tf_euler GetSparseFeature                   tf_euler/kernels/get_sparse_feature_op.cc:52-130  a node without values gets one
//                                               entry {i, 0} = default_value
//   tf_euler GetBinaryFeature                   tf_euler/kernels/get_binary_feature_op.cc          one string per node
// Same shape as the full-neighbor listing: per-node lengths -> cub inclusive scan -> copy; no host sync in the device entry points.
#include <cub/device/device_scan.cuh>

#include <algorithm>

#include "internal.h"

namespace eu {

template <bool SPARSE>
__global__ void k_ragged_len(DevGraph g, const unsigned long long* __restrict__ nodes, int64_t M, int32_t fid,
                             long long* __restrict__ out_ptr) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i == 0) out_ptr[0] = 0;
  if (i >= M) return;
  int64_t b, e;
  const int64_t row = lookup_row(g, nodes[i]);
  if (SPARSE) ragged_slice(g.u64_ptr, g.n_u64_slots, row, fid, &b, &e);
  else ragged_slice(g.bin_ptr, g.n_bin_slots, row, fid, &b, &e);
  long long len = e - b;
  if (SPARSE && len == 0) len = 1;   // one default entry (get_sparse_feature_op.cc:96-99)
  out_ptr[i + 1] = len;
}

template <bool SPARSE>
__global__ void __launch_bounds__(256) k_ragged_fill(DevGraph g, const unsigned long long* __restrict__ nodes, int64_t M, int32_t fid,
                                                     long long default_value, const long long* __restrict__ out_ptr, int64_t cap,
                                                     long long* __restrict__ out_values, unsigned char* __restrict__ out_bytes) {
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; i < M; i += nwarps) {
    int64_t b, e;
    const int64_t row = lookup_row(g, nodes[i]);
    if (SPARSE) ragged_slice(g.u64_ptr, g.n_u64_slots, row, fid, &b, &e);
    else ragged_slice(g.bin_ptr, g.n_bin_slots, row, fid, &b, &e);
    const int64_t o = out_ptr[i];
    if (SPARSE) {
      if (e == b) { if (lane == 0 && o < cap) out_values[o] = default_value; continue; }
      for (int64_t k = lane; k < e - b; k += 32) if (o + k < cap) out_values[o + k] = (long long)g.u64_val[b + k];
    } else {
      for (int64_t k = lane; k < e - b; k += 32) if (o + k < cap) out_bytes[o + k] = g.bin_val[b + k];
    }
  }
}

size_t ragged_scan_bytes(int64_t M) {
  size_t tmp = 0;
  cub::DeviceScan::InclusiveSum((void*)nullptr, tmp, (long long*)nullptr, (long long*)nullptr, (int)(M + 1));
  return tmp;
}

// out_ptr [M + 1] = the entry offsets of the nodes (lengths, then an inclusive scan in the scratch tmp)
template <bool SPARSE>
static int ragged_ptr(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, void* tmp, size_t tmp_bytes, int64_t* out_ptr) {
  cudaStream_t s = c->stream;
  k_ragged_len<SPARSE><<<(unsigned)ceil_div(std::max<int64_t>(M, 1), 256), 256, 0, s>>>(c->g->d, (const unsigned long long*)nodes, M, fid,
                                                                                        (long long*)out_ptr);
  EU_LAUNCHED();
  EU_CUDA(cub::DeviceScan::InclusiveSum(tmp, tmp_bytes, (long long*)out_ptr, (long long*)out_ptr, (int)(M + 1), s));
  EU_LAUNCHED();
  return EU_OK;
}

int sparse_entry_ptr(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, void* tmp, size_t tmp_bytes, int64_t* out_ptr) {
  return ragged_ptr<true>(c, nodes, M, fid, tmp, tmp_bytes, out_ptr);
}

template <bool SPARSE>
static int ragged_get(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int64_t default_value, int64_t cap, int64_t* out_ptr,
                      int64_t* out_values, uint8_t* out_bytes, const char* what) {
  if (!c || M < 0 || cap < 0 || !out_ptr || (M > 0 && !nodes) || (cap > 0 && !(SPARSE ? (void*)out_values : (void*)out_bytes))) {
    set_error("%s: bad argument", what);
    return EU_ERR_INVALID;
  }
  EU_CUDA(cudaSetDevice(c->g->device));
  if (M >= ((int64_t)1 << 31)) { set_error("%s: more than 2^31 nodes", what); return EU_ERR_UNSUPPORTED; }
  const DevGraph& d = c->g->d;
  cudaStream_t s = c->stream;
  const size_t tmp = ragged_scan_bytes(M);
  int rc = ctx_misc(c, (int64_t)tmp + 256);
  if (rc) return rc;
  if ((rc = ragged_ptr<SPARSE>(c, nodes, M, fid, c->d_misc, tmp, out_ptr))) return rc;
  if (cap > 0 && M > 0) {
    const unsigned blocks = (unsigned)std::min<int64_t>(ceil_div(M * 32, 256), kSMs * 8);
    k_ragged_fill<SPARSE><<<blocks, 256, 0, s>>>(d, (const unsigned long long*)nodes, M, fid, (long long)default_value, (const long long*)out_ptr, cap,
                                                 (long long*)out_values, out_bytes);
    EU_LAUNCHED();
  }
  return EU_OK;
}

}  // namespace eu

using namespace eu;

extern "C" {

int eu_get_sparse_feature(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int64_t default_value, int64_t cap, int64_t* out_ptr,
                          int64_t* out_values) {
  return ragged_get<true>(c, nodes, M, fid, default_value, cap, out_ptr, out_values, nullptr, "eu_get_sparse_feature");
}
int eu_get_binary_feature(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int64_t cap, int64_t* out_ptr, uint8_t* out_bytes) {
  return ragged_get<false>(c, nodes, M, fid, 0, cap, out_ptr, nullptr, out_bytes, "eu_get_binary_feature");
}

}  // extern "C"
