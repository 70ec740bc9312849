// Device-side first-occurrence unique (SURVEY.md section 8f, row next-1): the tf.unique of UniqueDataFlow / SageDataFlow
// (tf_euler/python/dataflow/neighbor_dataflow.py:84-109, sage_dataflow.py:35-50) without leaving HBM.
//   tf.unique(x) -> (y, idx): y = the distinct values of x in order of FIRST occurrence, x[i] == y[idx[i]].
// Same machinery as the seed dedup of the sampling path (csrc/sample.cu): an open-addressing table keyed by id that
// keeps the minimum index, then "is this my first occurrence" flags, an exclusive scan, and a scatter.
//   k_uq_insert -> k_uq_first -> cub::ExclusiveSum -> k_uq_emit        (4 launches, no host sync)
#include <cub/device/device_scan.cuh>

#include "internal.h"
#include "uq.cuh"

namespace eu {

__global__ void k_uq_insert(HashSlot* tab, unsigned long long mask, const unsigned long long* __restrict__ ids, int64_t n) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  uq_insert_warp(tab, mask, ids[i], (unsigned long long)i);
}

__global__ void k_uq_first(const HashSlot* tab, unsigned long long mask, const unsigned long long* __restrict__ ids, int64_t n,
                           int32_t* __restrict__ first, int32_t* __restrict__ flag) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int32_t f = (int32_t)uq_first(tab, mask, ids[i]);
  first[i] = f;
  flag[i] = f == (int32_t)i ? 1 : 0;
}

__global__ void k_uq_emit(const unsigned long long* __restrict__ ids, int64_t n, const int32_t* __restrict__ first,
                          const int32_t* __restrict__ flag, const int32_t* __restrict__ pos, unsigned long long* __restrict__ uniq,
                          int32_t* __restrict__ inverse, long long* __restrict__ n_unique) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (flag[i]) uniq[pos[i]] = ids[i];
  inverse[i] = pos[first[i]];
  if (i == n - 1 && n_unique) *n_unique = (long long)pos[i] + flag[i];
}

}  // namespace eu

using namespace eu;

// uniq: device i64[n] (first *n_unique entries valid), inverse: device i32[n], n_unique: device i64[1] (may be NULL)
extern "C" int eu_unique(eu_ctx* c, const int64_t* ids, int64_t n, int64_t* uniq, int32_t* inverse, int64_t* n_unique) {
  if (!c || n < 0 || n >= ((int64_t)1 << 31) || (n > 0 && (!ids || !uniq || !inverse))) { set_error("eu_unique: bad argument"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  cudaStream_t s = c->stream;
  if (n == 0) {
    if (n_unique) EU_CUDA(cudaMemsetAsync(n_unique, 0, sizeof(int64_t), s));
    return EU_OK;
  }
  const int64_t cap = uq_table_cap(n);
  size_t tmp = 0;
  cub::DeviceScan::ExclusiveSum((void*)nullptr, tmp, (int32_t*)nullptr, (int32_t*)nullptr, (int)n, s);
  const int64_t o_tab = 256, o_first = o_tab + 16 * (cap + 1), o_flag = o_first + ((4 * n + 255) & ~(int64_t)255),
                o_pos = o_flag + ((4 * n + 255) & ~(int64_t)255), o_tmp = o_pos + ((4 * n + 255) & ~(int64_t)255);
  int rc = ctx_misc(c, o_tmp + (int64_t)tmp + 256);
  if (rc) return rc;
  char* m = (char*)c->d_misc;
  HashSlot* tab = (HashSlot*)(m + o_tab);
  int32_t *first = (int32_t*)(m + o_first), *flag = (int32_t*)(m + o_flag), *pos = (int32_t*)(m + o_pos);
  const unsigned nb = (unsigned)ceil_div(n, 256);
  { EuProfScope ps(c, "k_uq_clear+insert", n);
    k_uq_clear<<<(unsigned)std::min<int64_t>(ceil_div(cap + 1, 256), kSMs * 8), 256, 0, s>>>(tab, cap + 1);
    EU_LAUNCHED();
    k_uq_insert<<<nb, 256, 0, s>>>(tab, (unsigned long long)cap - 1, (const unsigned long long*)ids, n); }
  EU_LAUNCHED();
  { EuProfScope ps(c, "k_uq_first", n);
    k_uq_first<<<nb, 256, 0, s>>>(tab, (unsigned long long)cap - 1, (const unsigned long long*)ids, n, first, flag); }
  EU_LAUNCHED();
  EU_CUDA(cub::DeviceScan::ExclusiveSum(m + o_tmp, tmp, flag, pos, (int)n, s));
  EU_LAUNCHED();
  { EuProfScope ps(c, "k_uq_emit", n);
    k_uq_emit<<<nb, 256, 0, s>>>((const unsigned long long*)ids, n, first, flag, pos, (unsigned long long*)uniq, inverse, (long long*)n_unique); }
  EU_LAUNCHED();
  return EU_OK;
}
