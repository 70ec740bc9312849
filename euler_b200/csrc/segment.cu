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

size_t row_plan_bytes(int64_t E, int64_t n_rows, int64_t width) {
  return E ? order_bytes(E, n_rows) + distinct_plan_bytes(E, width) : 0;
}

int plan_rows(eu_ctx* c, char* buf, RowList* L) {
  if (!L->E) return EU_OK;
  int rc = order_by(c, L->key, L->E, L->n_rows, buf, &L->ord);
  if (rc) return rc;
  return plan_distinct(c, L->ord, L->E, buf + order_bytes(L->E, L->n_rows), &L->P);
}

constexpr int kRowSumUnroll = 8;   // entries in flight per lane in the chunk sums

// the destination row of distinct segment p: the table row key[p] (dense) or row p of the COO values (sparse)
__device__ __forceinline__ float* distinct_out_row(float* out, const DistinctPlan& P, int64_t p, int dim, bool by_key) {
  return out + (by_key ? (int64_t)__ldg(P.key + p) : p) * dim;
}

// G lanes per chunk of the distinct-row segments, 4 columns per lane and step: the chunk's entries summed left to right from
// +0, kRowSumUnroll of them in flight; a segment of one chunk writes its output row, the chunks of a longer one their partial
// rows.  GATHER: the entries are RowEntries' gathered kind (a template parameter, so the other kinds carry none of its division).
// A column's adds are fma(w, x, acc) in entry order whatever the lane mapping, and fma(1, x, acc) is __fadd_rn(acc, x).  The
// gathered kind asks for one block per SM: under the default bound ptxas spilled around the scalar path's division subroutine.
// The other kinds keep the default (a minimum of 0 emits none); one block per SM would raise them from 63 / 80 registers to
// 70 / 82, and the float4 form would then fit two blocks per SM instead of three.  T: the storage type of S.target.
template <bool VEC, bool GATHER, typename T>
__global__ void __launch_bounds__(256, GATHER ? 1 : 0) k_row_chunks(RowEntries S, const int32_t* __restrict__ perm, DistinctPlan P,
                                                                    int dim, int G, bool by_key, float* __restrict__ out) {
  const int lg = 31 - __clz(G);
  const int sub = (int)(threadIdx.x & (G - 1));
  const int64_t nch_all = __ldg(P.chunk_off + P.E);
  const int64_t step = ((int64_t)gridDim.x * blockDim.x) >> lg;
  constexpr int U = VEC ? kRowSumUnroll : kRowSumUnroll / 2;   // the scalar path's loads take more registers
  int ignored = 0;
  for (int64_t c = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> lg; c < nch_all; c += step) {
    const int64_t p = key_upper_bound(P.chunk_off, P.E + 1, c) - 1;
    const int64_t c0 = __ldg(P.chunk_off + p), nch = __ldg(P.chunk_off + p + 1) - c0;
    const int64_t b = __ldg(P.start + p) + (c - c0) * kSegChunk;
    const int64_t e = min(b + kSegChunk, (int64_t)__ldg(P.start + p + 1));
    float* o = nch == 1 ? distinct_out_row(out, P, p, dim, by_key) : P.partial + (int64_t)(__ldg(P.part_off + p) + (c - c0)) * dim;
    for (int d = sub * 4; d < dim; d += G * 4) {
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int64_t k0 = b; k0 < e; k0 += U) {
        float4 x[U];
        float w[U];
#pragma unroll
        for (int q = 0; q < U; ++q) {
          if (k0 + q < e) {
            const int64_t en = __ldg(perm + k0 + q);
            if (GATHER || en < S.n_src) {
              const float* row = GATHER ? S.gt + (int64_t)(__ldg(S.node + en) / S.group) * S.ld : S.gt + en * dim;
              x[q] = row_load4<VEC>(row, d, dim);
              w[q] = 1.f;
            } else {
              const int64_t t = en - S.n_src;
              x[q] = row_load4<VEC>(static_cast<const T*>(S.target) + row_of(__ldg(S.src + t / S.J), S.n_rows, &ignored) * dim, d, dim);
              w[q] = __ldg(S.coef + t);
            }
          }
        }
#pragma unroll
        for (int q = 0; q < U; ++q) {
          if (k0 + q < e) {
            if (GATHER && S.pool_den != 0.f) {
              x[q].x = __fdiv_rn(x[q].x, S.pool_den); x[q].y = __fdiv_rn(x[q].y, S.pool_den);
              x[q].z = __fdiv_rn(x[q].z, S.pool_den); x[q].w = __fdiv_rn(x[q].w, S.pool_den);
            }
            acc.x = __fmaf_rn(w[q], x[q].x, acc.x); acc.y = __fmaf_rn(w[q], x[q].y, acc.y);
            acc.z = __fmaf_rn(w[q], x[q].z, acc.z); acc.w = __fmaf_rn(w[q], x[q].w, acc.w);
          }
        }
      }
      if (VEC) {
        *reinterpret_cast<float4*>(o + d) = acc;
      } else {
        o[d] = acc.x;
        if (d + 1 < dim) o[d + 1] = acc.y;
        if (d + 2 < dim) o[d + 2] = acc.z;
        if (d + 3 < dim) o[d + 3] = acc.w;
      }
    }
  }
}

// the output row of each segment of several chunks = its partial rows added in chunk order from +0; rows (sparse, may be
// null) gets the segments' row ids
__global__ void k_row_combine(DistinctPlan P, int dim, bool by_key, float* __restrict__ out, int64_t* __restrict__ rows) {
  const int64_t D = __ldg(P.nd);
  if (rows)
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < D; t += (int64_t)gridDim.x * blockDim.x)
      rows[t] = __ldg(P.key + t);
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < D * dim; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = t / dim, f = t - p * dim;
    const int64_t nch = __ldg(P.chunk_off + p + 1) - __ldg(P.chunk_off + p);
    if (nch == 1) continue;
    const float* part = P.partial + (int64_t)__ldg(P.part_off + p) * dim + f;
    float acc = 0.f;
    for (int64_t j = 0; j < nch; ++j) acc = __fadd_rn(acc, __ldg(part + j * dim));
    distinct_out_row(out, P, p, dim, by_key)[f] = acc;
  }
}

int sum_distinct_rows(eu_ctx* c, const RowEntries& S, const RowList& L, int dim, bool by_key, float* out, int64_t* rows) {
  if (!L.E) return EU_OK;
  cudaStream_t s = c->stream;
  const bool vec = dim % 4 == 0 && (!S.node || S.ld % 4 == 0) && aligned16(out) && (!S.gt || aligned16(S.gt)) &&
                   (!S.target || aligned4_elems(S.target, S.target_dtype));
  const int G = group_lanes(ceil_div(dim, 4));
  const unsigned blocks = stride_grid((L.E + L.E / kSegChunk + 1) * G);   // >= one group per chunk, up to the grid cap
  with_dtype(S.target_dtype, [&](auto t) {
    using T = typename decltype(t)::type;
    auto chunks = vec ? k_row_chunks<true, false, T> : k_row_chunks<false, false, T>;
    if constexpr (std::is_same<T, float>::value)   // a list of the gathered kind is f32
      if (S.node) chunks = vec ? k_row_chunks<true, true, float> : k_row_chunks<false, true, float>;
    chunks<<<blocks, 256, 0, s>>>(S, L.ord.perm, L.P, dim, G, by_key, out);
  });
  EU_LAUNCHED();
  k_row_combine<<<stride_grid(L.E * dim), 256, 0, s>>>(L.P, dim, by_key, out, rows);
  EU_LAUNCHED();
  return EU_OK;
}

int read_back(eu_ctx* c, int32_t* hdr, bool* bad, int n, const int32_t* const* nd, int64_t* counts) {
  cudaStream_t s = c->stream;
  int32_t h[kReadBackMax + 1] = {};
  for (int i = 0; i < n; ++i)
    if (nd[i] && nd[i] != hdr + 1 + i) EU_CUDA(cudaMemcpyAsync(hdr + 1 + i, nd[i], sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
  EU_CUDA(cudaMemcpyAsync(h, hdr, sizeof(int32_t) * (1 + n), cudaMemcpyDeviceToHost, s));
  EU_CUDA(cudaStreamSynchronize(s));
  if (bad) *bad = h[0] != 0;
  for (int i = 0; i < n; ++i) counts[i] = nd[i] ? h[1 + i] : 0;
  return EU_OK;
}

__global__ void __launch_bounds__(kMeanThreads) k_f64_mean(const double* __restrict__ rowloss, int64_t B, int64_t N,
                                                           float* __restrict__ loss) {
  __shared__ double sh[kMeanThreads];
  double acc = 0.0;
  for (int64_t i = threadIdx.x; i < B; i += kMeanThreads) acc += __ldg(rowloss + i);
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int s = kMeanThreads / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) *loss = (float)(sh[0] / (double)N);
}

}  // namespace eu
