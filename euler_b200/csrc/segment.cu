// Edge orders and the chunk bookkeeping of fixed-order segment sums (see segment.cuh).
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "segment.cuh"

namespace eu {

__global__ void k_check_sorted(const int32_t* __restrict__ idx, int64_t E, int* unsorted) {
  int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e + 1 < E && __ldg(idx + e) > __ldg(idx + e + 1)) *unsorted = 1;
}

__global__ void k_iota(int32_t* __restrict__ v, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) v[i] = (int32_t)i;
}

size_t order_bytes(int64_t E, int64_t n) {
  size_t t = 0;
  cub::DeviceRadixSort::SortPairs((void*)nullptr, t, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const int32_t*)nullptr,
                                  (int32_t*)nullptr, (int)E, 0, radix_bits(n));
  return 3 * a256(4 * (size_t)E) + a256(t);
}

// buf: keys, permutation (edge of each position), iota, cub temp
int order_by(eu_ctx* c, const int32_t* idx, int64_t E, int64_t n, char* buf, EdgeOrder* o) {
  cudaStream_t s = c->stream;
  int32_t* keys = (int32_t*)buf;
  int32_t* perm = (int32_t*)(buf + a256(4 * (size_t)E));
  int32_t* iota = (int32_t*)(buf + 2 * a256(4 * (size_t)E));
  void* tmp = buf + 3 * a256(4 * (size_t)E);
  size_t t = 0;
  cub::DeviceRadixSort::SortPairs((void*)nullptr, t, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const int32_t*)nullptr,
                                  (int32_t*)nullptr, (int)E, 0, radix_bits(n), s);
  k_iota<<<stride_grid(E), 256, 0, s>>>(iota, E);
  EU_LAUNCHED();
  EU_CUDA(cub::DeviceRadixSort::SortPairs(tmp, t, (const uint32_t*)idx, (uint32_t*)keys, (const int32_t*)iota, perm, (int)E, 0,
                                          radix_bits(n), s));
  EU_LAUNCHED();
  o->key = keys;
  o->perm = perm;
  return EU_OK;
}

// Is idx non-decreasing?  One flag read back to the host (a stream synchronisation).
static int is_sorted(eu_ctx* c, const int32_t* idx, int64_t E, int* flag_dev, bool* sorted) {
  *sorted = true;
  if (E < 2) return EU_OK;
  cudaStream_t s = c->stream;
  EU_CUDA(cudaMemsetAsync(flag_dev, 0, sizeof(int), s));
  k_check_sorted<<<(unsigned)ceil_div(E, 256), 256, 0, s>>>(idx, E, flag_dev);
  EU_LAUNCHED();
  int h = 0;
  EU_CUDA(cudaMemcpyAsync(&h, flag_dev, sizeof(int), cudaMemcpyDeviceToHost, s));
  EU_CUDA(cudaStreamSynchronize(s));
  *sorted = h == 0;
  return EU_OK;
}

int order_targets(eu_ctx* c, const int32_t* dst, int64_t E, int64_t n_dst, size_t head_bytes, size_t tail_bytes,
                  const char* sort_scope, TargetOrder* t) {
  int rc = ctx_misc(c, 256);
  if (rc) return rc;
  bool sorted = true;
  if ((rc = is_sorted(c, dst, E, (int*)c->d_misc, &sorted))) return rc;
  const size_t o_ord = 256 + head_bytes, o_tail = o_ord + (sorted ? 0 : order_bytes(E, n_dst));
  if ((rc = ctx_misc(c, (int64_t)(o_tail + tail_bytes)))) return rc;
  char* m = (char*)c->d_misc;
  t->head = m + 256;
  t->tail = m + o_tail;
  t->ord = EdgeOrder();
  t->ord.key = dst;
  if (sorted) return EU_OK;
  if (!sort_scope) return order_by(c, dst, E, n_dst, m + o_ord, &t->ord);
  EuProfScope ps(c, sort_scope, E);
  return order_by(c, dst, E, n_dst, m + o_ord, &t->ord);
}

__global__ void k_seg_starts(const int32_t* __restrict__ key, int64_t P, int64_t n, int32_t* __restrict__ start) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r <= n; r += (int64_t)gridDim.x * blockDim.x)
    start[r] = (int32_t)key_lower_bound(key, P, r);
}

// nc[s] = the chunks of K items of segment s = [start[s], start[s + 1]), for s < n; nc[n] = 0 (an exclusive scan then gives
// every segment's first chunk and, at n, the number of chunks)
__global__ void k_seg_chunks(const int32_t* __restrict__ start, int64_t n, int K, int32_t* __restrict__ nc) {
  for (int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; s <= n; s += (int64_t)gridDim.x * blockDim.x)
    nc[s] = s < n ? (int32_t)(((int64_t)__ldg(start + s + 1) - __ldg(start + s) + K - 1) / K) : 0;
}

__global__ void k_seg_combine(const int32_t* __restrict__ chunk_off, const float* __restrict__ partial, int64_t P, int F,
                              float* __restrict__ S) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= P * F) return;
  const int64_t p = t / F, f = t - p * F;
  const int64_t c0 = __ldg(chunk_off + p), c1 = __ldg(chunk_off + p + 1);
  if (c1 - c0 == 1) return;
  float acc = 0.f;
  for (int64_t c = c0; c < c1; ++c) acc = __fadd_rn(acc, __ldg(partial + c * F + f));
  S[t] = acc;
}

size_t seg_scan_bytes(int64_t n) {
  size_t t = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, t, (const int32_t*)nullptr, (int32_t*)nullptr, (int)(n + 1));
  return t;
}

int seg_chunk_offsets(eu_ctx* c, const int32_t* start, int64_t n, int K, int32_t* nc, void* tmp, size_t tmp_bytes,
                      int32_t* chunk_off) {
  cudaStream_t s = c->stream;
  k_seg_chunks<<<stride_grid(n + 1), 256, 0, s>>>(start, n, K, nc);
  EU_LAUNCHED();
  EU_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, nc, chunk_off, (int)(n + 1), s));
  EU_LAUNCHED();
  return EU_OK;
}

size_t seg_plan_bytes(int64_t E, int64_t n, int64_t width) {
  return 3 * a256(4 * (size_t)(n + 1)) + a256(seg_scan_bytes(n)) + a256(4 * (size_t)(n + E / kSegChunk) * width);
}

int plan_segments(eu_ctx* c, const EdgeOrder& o, int64_t E, int64_t n, char* buf, SegPlan* S) {
  const size_t n1 = a256(4 * (size_t)(n + 1)), scan = seg_scan_bytes(n);
  S->n = n;
  S->slots = n + E / kSegChunk;
  S->start = (int32_t*)buf;
  int32_t* nc = (int32_t*)(buf + n1);
  S->chunk_off = (int32_t*)(buf + 2 * n1);
  S->partial = (float*)(buf + 3 * n1 + a256(scan));
  k_seg_starts<<<stride_grid(n + 1), 256, 0, c->stream>>>(o.key, E, n, S->start);
  EU_LAUNCHED();
  return seg_chunk_offsets(c, S->start, n, kSegChunk, nc, buf + 3 * n1, scan, S->chunk_off);
}

// head[k] = 1 where position k of the sorted keys starts a distinct key
__global__ void k_distinct_heads(const int32_t* __restrict__ key, int64_t E, int32_t* __restrict__ head) {
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < E; k += (int64_t)gridDim.x * blockDim.x)
    head[k] = k == 0 || __ldg(key + k) != __ldg(key + k - 1);
}

// From sid (the inclusive scan of the heads): each distinct key's first position and value, and start[s] = E for s in [D, E]
__global__ void k_distinct_starts(const int32_t* __restrict__ key, const int32_t* __restrict__ sid, int64_t E,
                                  int32_t* __restrict__ skey, int32_t* __restrict__ start) {
  const int64_t D = __ldg(sid + E - 1);
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t <= E; t += (int64_t)gridDim.x * blockDim.x) {
    if (t < E && (t == 0 || __ldg(key + t) != __ldg(key + t - 1))) {
      const int32_t s = __ldg(sid + t) - 1;
      start[s] = (int32_t)t;
      skey[s] = __ldg(key + t);
    }
    if (t >= D) start[t] = (int32_t)E;
  }
}

// mc[s] = the chunks of segment s when it has several, else 0 (an exclusive scan then gives part_off)
__global__ void k_seg_multi(const int32_t* __restrict__ chunk_off, int64_t n, int32_t* __restrict__ mc) {
  for (int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; s <= n; s += (int64_t)gridDim.x * blockDim.x) {
    const int32_t k = s < n ? __ldg(chunk_off + s + 1) - __ldg(chunk_off + s) : 0;
    mc[s] = k > 1 ? k : 0;
  }
}

static size_t distinct_scan_bytes(int64_t E) {
  size_t t = 0;
  cub::DeviceScan::InclusiveSum(nullptr, t, (const int32_t*)nullptr, (int32_t*)nullptr, (int)E);
  return std::max(t, seg_scan_bytes(E));
}

size_t distinct_plan_bytes(int64_t E, int64_t width) {
  return 6 * a256(4 * (size_t)(E + 1)) + a256(distinct_scan_bytes(E)) + a256(4 * (size_t)(2 * E / kSegChunk + 1) * width);
}

int plan_distinct(eu_ctx* c, const EdgeOrder& o, int64_t E, char* buf, DistinctPlan* P) {
  cudaStream_t s = c->stream;
  const size_t n1 = a256(4 * (size_t)(E + 1)), scan = distinct_scan_bytes(E);
  int32_t* sid = (int32_t*)buf;
  P->E = E;
  P->part_rows = 2 * E / kSegChunk + 1;
  P->nd = sid + E - 1;
  P->key = (int32_t*)(buf + n1);
  P->start = (int32_t*)(buf + 2 * n1);
  int32_t* nc = (int32_t*)(buf + 3 * n1);
  P->chunk_off = (int32_t*)(buf + 4 * n1);
  P->part_off = (int32_t*)(buf + 5 * n1);
  void* tmp = buf + 6 * n1;
  P->partial = (float*)(buf + 6 * n1 + a256(scan));
  k_distinct_heads<<<stride_grid(E), 256, 0, s>>>(o.key, E, sid);
  EU_LAUNCHED();
  size_t t = scan;
  EU_CUDA(cub::DeviceScan::InclusiveSum(tmp, t, sid, sid, (int)E, s));
  EU_LAUNCHED();
  k_distinct_starts<<<stride_grid(E + 1), 256, 0, s>>>(o.key, sid, E, P->key, P->start);
  EU_LAUNCHED();
  int rc = seg_chunk_offsets(c, P->start, E, kSegChunk, nc, tmp, scan, P->chunk_off);
  if (rc) return rc;
  k_seg_multi<<<stride_grid(E + 1), 256, 0, s>>>(P->chunk_off, E, nc);
  EU_LAUNCHED();
  t = scan;
  EU_CUDA(cub::DeviceScan::ExclusiveSum(tmp, t, nc, P->part_off, (int)(E + 1), s));
  EU_LAUNCHED();
  return EU_OK;
}

}  // namespace eu
