// Dense feature fetch and message-passing gather / scatter aggregation (f32 data, i32 indices).
//
// Reference semantics (file:line relative to /root/reference):
//   GetDenseFeature   tf_euler/kernels/get_dense_feature_op.cc:63-121 over euler/core/api/api.cc:63-78
//   MPGather          tf_euler/kernels/gather_op.cc:42-51
//   MPScatterAdd      tf_euler/kernels/scatter_op.cc:44-55   (zero init, serial adds in index order)
//   MPScatterMax      tf_euler/kernels/scatter_op.cc:77-91   (init -1e9, strict >)
//   scatter_mean      tf_euler/python/euler_ops/mp_ops.py:65-69
//
// All are HBM-bound row moves: one (sub-)warp per row, 128-bit loads/stores, no shared memory
// (no reuse).  scatter_* has two paths chosen on the device (no host sync):
//   sorted indices (what SageDataFlow / fixed-fanout blocks produce, sage_dataflow.py:43-46):
//     warp per OUTPUT row, its edges found by binary search, accumulated left to right -> the
//     reference's summation order, bit-exact, no atomics;
//   unsorted indices: vector atomics (red.global.add.v4.f32), order-free, within 1e-5 relative.  The f32 atomic add flushes
//     subnormal inputs and results to zero (PTX atom / red .add.f32), which adds an absolute error below 2 * 2^-126 per
//     update: a sum that is itself subnormal can come back as zero.  max is exact there too, but
//     order-free: among equal zeros +0.0 wins (the reference keeps whichever of +0.0 / -0.0 comes first); -0.0 still beats
//     every negative value.  NaN never wins and values at or below -1e9 leave the initial -1e9, on both paths.
#include <stdlib.h>

#include <cooperative_groups.h>

#include <algorithm>

#include "segment.cuh"

namespace cg = cooperative_groups;

namespace eu {

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

// ---------------------------------------------------------------------------- feature fetch
// out[i, 0:dim] = feat[row(ids[i]), 0:min(feat_dim,dim)], zeros elsewhere / for unknown ids.  T: the table's storage type, P
// its placement, O the output's element type (float, or __nv_bfloat16: each value rounded once at the store).
template <typename T, typename O, bool VEC, int P>
__global__ void __launch_bounds__(256) k_feature(DevGraph g, const unsigned long long* __restrict__ ids,
                                                 int64_t M, int32_t dim, int G, int32_t soff, int32_t sdim,
                                                 O* __restrict__ out) {
  const int sh = 31 - __clz(G);   // G is a power of two
  const int sub = (int)(threadIdx.x & (G - 1));
  const int64_t stride = ((int64_t)gridDim.x * blockDim.x) >> sh;
  // grid-stride over the rows: the launcher may cap the grid (EU_FEATURE_CTAS CTAs per SM) so that this HBM-bound copy leaves
  // SM residency to the issue-bound sampling kernels of the other lanes
  for (int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> sh; i < M; i += stride) {
    const int64_t row = sdim > 0 ? lookup_row(g, ids[i]) : -1;
    const int32_t fd = sdim;  // stored width of this slot
    O* o = out + i * (int64_t)dim;
    const T* f = row >= 0 ? feat_row<T, P>(g, row) + soff : nullptr;
    if (VEC) {
      for (int32_t d = sub * 4; d < dim; d += G * 4) {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (f && d < fd) v = feat_ld4(f + d);  // VEC requires fd % 4 == 0 so a float4 never straddles fd
        rn_st4(o + d, v);
      }
    } else {
      for (int32_t d = sub; d < dim; d += G) o[d] = feat_st<O>((f && d < fd) ? feat_ld(f + d) : 0.f);
    }
  }
}

// ---------------------------------------------------------------------------- gather
template <bool VEC>
__global__ void __launch_bounds__(256) k_gather(const float* __restrict__ params, int64_t D,
                                                const int32_t* __restrict__ idx, int64_t E, int G,
                                                float* __restrict__ out) {
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t i = tid >> (31 - __clz(G));   // G is a power of two
  const int sub = (int)(tid & (G - 1));
  if (i >= E) return;
  const float* src = params + (int64_t)__ldg(idx + i) * D;  // no bounds check, as gather_op.cc:47-51
  float* o = out + i * D;
  if (VEC) {
    for (int64_t d = sub * 4; d < D; d += G * 4) st4(o + d, ldg4(src + d));
  } else {
    for (int64_t d = sub; d < D; d += G) o[d] = __ldg(src + d);
  }
}

// ---------------------------------------------------------------------------- scatter
enum { OP_ADD = 0, OP_MAX = 1, OP_MEAN = 2 };

// sorted path: G lanes per OUTPUT row r; edges [lb(r), lb(r+1)) reduced in index order.
template <int OP, bool VEC>
__global__ void __launch_bounds__(256) k_scatter_sorted(const float* __restrict__ upd, int64_t D,
                                                        const int32_t* __restrict__ idx, int64_t E,
                                                        int64_t size, int G, const int* unsorted,
                                                        float* __restrict__ out) {
  if (*unsorted) return;
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t r = tid >> (31 - __clz(G));   // G is a power of two
  const int sub = (int)(tid & (G - 1));
  if (r >= size) return;
  const int64_t b = key_lower_bound(idx, E, r), e = key_lower_bound(idx, E, r + 1);
  const float init = OP == OP_MAX ? -1e9f : 0.f;
  const float denom = __fadd_rn((float)(e - b), 1e-7f);
  float* o = out + r * D;
  if (VEC) {
    for (int64_t d = sub * 4; d < D; d += G * 4) {
      float4 acc = make_float4(init, init, init, init);
      for (int64_t k = b; k < e; ++k) {
        float4 v = ldg4(upd + k * D + d);
        if (OP == OP_MAX) {
          acc.x = v.x > acc.x ? v.x : acc.x; acc.y = v.y > acc.y ? v.y : acc.y;
          acc.z = v.z > acc.z ? v.z : acc.z; acc.w = v.w > acc.w ? v.w : acc.w;
        } else {
          acc.x = __fadd_rn(acc.x, v.x); acc.y = __fadd_rn(acc.y, v.y);
          acc.z = __fadd_rn(acc.z, v.z); acc.w = __fadd_rn(acc.w, v.w);
        }
      }
      if (OP == OP_MEAN) {
        acc.x = __fdiv_rn(acc.x, denom); acc.y = __fdiv_rn(acc.y, denom);
        acc.z = __fdiv_rn(acc.z, denom); acc.w = __fdiv_rn(acc.w, denom);
      }
      st4(o + d, acc);
    }
  } else {
    for (int64_t d = sub; d < D; d += G) {
      float acc = init;
      for (int64_t k = b; k < e; ++k) {
        float v = __ldg(upd + k * D + d);
        if (OP == OP_MAX) acc = v > acc ? v : acc; else acc = __fadd_rn(acc, v);
      }
      if (OP == OP_MEAN) acc = __fdiv_rn(acc, denom);
      o[d] = acc;
    }
  }
}

// unsorted path ------------------------------------------------------------------------------
__global__ void k_fill_if(float* __restrict__ out, int64_t n, float v, const int* unsorted) {
  if (!*unsorted) return;
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) out[i] = v;
}

__device__ __forceinline__ void atomic_max_f32(float* addr, float v) {
  // total order trick: floats with the sign bit clear compare like signed ints, with it set like reversed unsigned.  The branch
  // is chosen on the sign bit, not on v >= 0 (true for -0.0, whose int bits INT_MIN would then never win): -0.0 beats every
  // negative value and loses to +0.0.
  if (v != v) return;  // NaN never wins `upd > out`
  if (__float_as_int(v) >= 0) atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
  else atomicMin(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}

template <int OP, bool VEC>
__global__ void __launch_bounds__(256) k_scatter_atomic(const float* __restrict__ upd, int64_t D,
                                                        const int32_t* __restrict__ idx, int64_t E, int G,
                                                        const int* unsorted, float* __restrict__ out,
                                                        float* __restrict__ cnt) {
  if (!*unsorted) return;
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t i = tid >> (31 - __clz(G));   // G is a power of two
  const int sub = (int)(tid & (G - 1));
  if (i >= E) return;
  const int64_t r = __ldg(idx + i);
  float* o = out + r * D;
  const float* u = upd + i * D;
  if (OP == OP_MEAN && sub == 0) atomicAdd(cnt + r, 1.0f);
  if (VEC && OP != OP_MAX) {
    for (int64_t d = sub * 4; d < D; d += G * 4) atomicAdd(reinterpret_cast<float4*>(o + d), ldg4(u + d));
  } else {
    const int step = VEC ? 4 : 1;
    for (int64_t d = sub * step; d < D; d += G * step)
      for (int q = 0; q < step; ++q) {
        if (OP == OP_MAX) atomic_max_f32(o + d + q, __ldg(u + d + q));
        else atomicAdd(o + d + q, __ldg(u + d + q));
      }
  }
}

__global__ void k_mean_div(float* __restrict__ out, int64_t D, int64_t size, const float* __restrict__ cnt,
                           const int* unsorted) {
  if (!*unsorted) return;
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < size * D) out[i] = __fdiv_rn(out[i], __fadd_rn(cnt[i / D], 1e-7f));
}

// ---------------------------------------------------------------------------- fused SAGE mean
// out[r,:] = (sum_j feat[row(ids[r*count+j]),:]) / (count + 1e-7), j ascending (== get_dense_feature
// followed by scatter_mean over edge_src = repeat(range(rows), count)).
//
// A fanout repeats segments: a seed sampled `count` times with replacement hands the same node to the next hop many times, and
// the sampler gives every copy of a node the same draws.  Two rows whose `count` ids are equal in the same order have
// bit-identical outputs, so each distinct segment is reduced once, in three passes:
//   k_sage_classify   gives every row a source: itself (a representative), an earlier-claimed row with the same segment, or
//                     none (no id exists: zeros, no feature row is read);
//   k_sage_mean       reduces the representatives only;
//   k_sage_broadcast  copies each representative's output to its duplicates, zero-fills the rows without a neighbor, and frees
//                     the table slots the representatives claimed.
// Segments are found through an open-addressing table of 64-bit slots {upper 32 bits of the segment hash, representative + 1},
// 0 = free.  One CAS claims a slot and publishes its representative together, so no reader sees a claimed slot without its
// row.  A hash match is confirmed id by id: the same ids in another order are another segment (float addition does not
// associate).  The table is all-free between calls (allocated zeroed; every claimed slot is freed by the call that claimed it).
__global__ void __launch_bounds__(256) k_sage_classify(DevGraph g, const unsigned long long* __restrict__ ids, int64_t rows,
                                                       int32_t count, unsigned long long* tab, unsigned long long mask,
                                                       int32_t* __restrict__ src, int32_t* __restrict__ reps,
                                                       uint32_t* __restrict__ rep_slot, unsigned int* n_rep) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  // one thread per row: its `count` id loads are independent, and a capped grid (EU_SAGE_CTAS) keeps many rows in flight
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < rows; r += stride) {
    const unsigned long long* seg = ids + r * count;
    unsigned long long h = 0;
    bool any = false;
#pragma unroll 4
    for (int32_t j = 0; j < count; ++j) {
      const unsigned long long id = __ldg(seg + j);
      any |= lookup_row(g, id) >= 0;
      h = mix64(h + id + 1);   // a chain: the hash depends on the order of the ids
    }
    if (!any) { src[r] = -1; continue; }
    const unsigned long long tag = h & 0xFFFFFFFF00000000ull;
    unsigned long long p = h & mask;
    while (true) {
      unsigned long long sl = *reinterpret_cast<volatile unsigned long long*>(tab + p);   // hub segments recur: look before any CAS
      if (sl == 0ull) {
        sl = atomicCAS(tab + p, 0ull, tag | (unsigned long long)(r + 1));
        if (sl == 0ull) {
          src[r] = (int32_t)r;
          // one counter for the whole launch: the winners that are converged here append with one atomic
          const cg::coalesced_group grp = cg::coalesced_threads();
          unsigned int q = 0;
          if (grp.thread_rank() == 0) q = atomicAdd(n_rep, grp.size());
          q = grp.shfl(q, 0) + grp.thread_rank();
          reps[q] = (int32_t)r;
          rep_slot[q] = (uint32_t)p;
          break;
        }
      }
      if ((sl & 0xFFFFFFFF00000000ull) == tag) {
        const int64_t o = (int64_t)(sl & 0xFFFFFFFFull) - 1;
        const unsigned long long* os = ids + o * count;
        bool same = true;
#pragma unroll 4
        for (int32_t j = 0; j < count; ++j) same &= __ldg(seg + j) == __ldg(os + j);
        if (same) { src[r] = (int32_t)o; break; }
      }
      p = (p + 1) & mask;
    }
  }
}

// One warp per representative (list[0 .. *n_list)), or per row when there is no list; the `count` id->row lookups run in parallel across lanes, then NV float4
// per lane are accumulated.
// NV float4 per lane: rows of up to NV * 128 floats.  FULL: the width is exactly NV * 128 (128 / 256: no column guards, the
// width is a compile-time constant); otherwise any multiple of 4 up to NV * 128 (e.g. 64 of configs[4]) with guarded columns.
// O: the output's element type; the sum and the division are f32 whatever it is, and a bf16 output is rounded once at the store.
template <typename T, typename O, int NV, bool FULL, int P>
__global__ void __launch_bounds__(256) k_sage_mean(DevGraph g, const unsigned long long* __restrict__ ids,
                                                   int64_t rows, const int32_t* __restrict__ list, const unsigned int* __restrict__ n_list,
                                                   int32_t count, bool mean, O* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int32_t fd = FULL ? NV * 128 : g.feat_dim;    // == dim, a multiple of 4, <= NV * 128 (checked by the launcher)
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t n = list ? (int64_t)__ldg(n_list) : rows;
  // grid-stride, one warp per output row (the launcher may cap the grid: EU_SAGE_CTAS CTAs per SM)
  for (int64_t q = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; q < n; q += nwarps) {
  const int64_t r = list ? (int64_t)__ldg(list + q) : q;
  float4 acc[NV];
#pragma unroll
  for (int v = 0; v < NV; ++v) acc[v] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int32_t j0 = 0; j0 < count; j0 += 32) {
    // the id -> row lookups of up to 32 neighbors run in parallel across the lanes (rows < 2^31: launcher)
    int32_t my = -1;
    if (j0 + lane < count) my = (int32_t)lookup_row(g, __ldg(ids + r * count + j0 + lane));
    // Only neighbors that exist are visited, in ascending j.  Skipping an absent one is exact: it would add a
    // row of +0.0 and the accumulator can never be -0.0 (it starts at +0.0 and x + (-0.0) keeps +0.0's sign).
    unsigned valid = __ballot_sync(0xffffffffu, my >= 0);
    while (valid) {  // warp-uniform
      float4 v[4][NV];
      int n = 0;
#pragma unroll
      for (int q = 0; q < 4; ++q) {  // 4 independent row reads in flight
        if (valid) {
          const int j = __ffs(valid) - 1;
          valid &= valid - 1;
          const int32_t row = __shfl_sync(0xffffffffu, my, j);
          const T* p = feat_row<T, P>(g, row, fd, lane * 4);
#pragma unroll
          for (int t = 0; t < NV; ++t) v[q][t] = (FULL || lane * 4 + t * 128 < fd) ? feat_ld4(p + t * 128) : make_float4(0.f, 0.f, 0.f, 0.f);
          n = q + 1;
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (q < n) {
#pragma unroll
          for (int t = 0; t < NV; ++t) {
            acc[t].x = __fadd_rn(acc[t].x, v[q][t].x); acc[t].y = __fadd_rn(acc[t].y, v[q][t].y);
            acc[t].z = __fadd_rn(acc[t].z, v[q][t].z); acc[t].w = __fadd_rn(acc[t].w, v[q][t].w);
          }
        }
      }
    }
  }
  const float denom = __fadd_rn((float)count, 1e-7f);
  O* o = out + r * (int64_t)fd + lane * 4;
#pragma unroll
  for (int t = 0; t < NV; ++t) {
    float4 a = acc[t];
    if (mean) { a.x = __fdiv_rn(a.x, denom); a.y = __fdiv_rn(a.y, denom); a.z = __fdiv_rn(a.z, denom); a.w = __fdiv_rn(a.w, denom); }
    if (FULL || lane * 4 + t * 128 < fd) rn_st4(o + t * 128, a);
  }
  }
}

// generic width fallback: one warp per representative, scalar columns
template <typename T, typename O, int P>
__global__ void __launch_bounds__(256) k_sage_mean_generic(DevGraph g, const unsigned long long* __restrict__ ids,
                                                           int64_t rows, const int32_t* __restrict__ list, const unsigned int* __restrict__ n_list,
                                                           int32_t count, int32_t dim, bool mean, O* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int32_t fd = g.feat_dim;
  const float denom = __fadd_rn((float)count, 1e-7f);
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t n = list ? (int64_t)__ldg(n_list) : rows;
  for (int64_t q = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; q < n; q += nwarps) {
    const int64_t r = list ? (int64_t)__ldg(list + q) : q;
    for (int32_t d = lane; d < dim; d += 32) {
      float acc = 0.f;
      for (int32_t j = 0; j < count; ++j) {
        const int64_t row = lookup_row(g, __ldg(ids + r * count + j));
        acc = __fadd_rn(acc, (row >= 0 && d < fd) ? feat_ld(feat_row<T, P>(g, row, fd, 0) + d) : 0.f);
      }
      out[r * (int64_t)dim + d] = feat_st<O>(mean ? __fdiv_rn(acc, denom) : acc);
    }
  }
}

// G lanes per row (G a power of two): a duplicate gets its representative's output, a row without a neighbor gets +0.0 (what
// the reduction writes for it: it starts at +0.0 and adds nothing); representatives are already done.  Then every slot the
// representatives claimed is freed.  O: the output's element type.  A bf16 representative row goes through feat_ld / rn_st4
// unchanged: it was rounded by the same rounding, which maps a widened bf16 value to its own bits (NaN to the same canonical
// NaN).
template <typename O, bool VEC>
__global__ void __launch_bounds__(256) k_sage_broadcast(const int32_t* __restrict__ src, int64_t rows, int32_t dim, int G,
                                                        const uint32_t* __restrict__ rep_slot, const unsigned int* __restrict__ n_rep,
                                                        unsigned long long* tab, O* out) {
  const int sh = 31 - __clz(G);
  const int sub = (int)(threadIdx.x & (G - 1));
  const int64_t gtid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t nthreads = (int64_t)gridDim.x * blockDim.x;
  for (int64_t r = gtid >> sh; r < rows; r += nthreads >> sh) {
    const int64_t s = __ldg(src + r);
    if (s == r) continue;
    O* o = out + r * (int64_t)dim;
    const O* f = s >= 0 ? out + s * (int64_t)dim : nullptr;   // a representative's row: not written by this kernel
    if (VEC) {
      for (int32_t d = sub * 4; d < dim; d += G * 4) rn_st4(o + d, f ? feat_ld4(f + d) : make_float4(0.f, 0.f, 0.f, 0.f));
    } else {
      for (int32_t d = sub; d < dim; d += G) o[d] = feat_st<O>(f ? feat_ld(f + d) : 0.f);
    }
  }
  const int64_t n = (int64_t)__ldg(n_rep);
  for (int64_t q = gtid; q < n; q += nthreads) tab[__ldg(rep_slot + q)] = 0ull;
}

// CTAs per SM of the HBM-bound row movers (0 = one CTA per 8 rows / as many as the rows need).  A capped, persistent grid keeps
// the copy at HBM speed (a few warps per SM cover the bandwidth-delay product) while the issue-bound sampling kernels of the
// other lanes stay resident beside it.
static inline unsigned capped_grid(int64_t want_blocks, const char* env, int dflt) {
  static int cached_sage = -1, cached_feat = -1;
  int& cached = env[3] == 'S' ? cached_sage : cached_feat;
  if (cached < 0) { const char* e = getenv(env); cached = e ? std::max(0, atoi(e)) : dflt; }
  const int64_t cap = cached > 0 ? (int64_t)kSMs * cached : want_blocks;
  return (unsigned)std::max<int64_t>(1, std::min(want_blocks, cap));
}

template <int OP>
static int scatter(eu_ctx* c, const float* upd, int64_t D, const int32_t* idx, int64_t E, int64_t size,
                   float* out) {
  if (!c || D <= 0 || E < 0 || size < 0 || (E > 0 && (!upd || !idx)) || (size > 0 && !out)) {
    set_error("scatter: bad argument");
    return EU_ERR_INVALID;
  }
  EU_CUDA(cudaSetDevice(c->g->device));
  if (size == 0) return EU_OK;
  int rc = ctx_misc(c, 256 + (OP == OP_MEAN ? (int64_t)sizeof(float) * size : 0));
  if (rc) return rc;
  int* unsorted = (int*)c->d_misc;
  float* cnt = (float*)((char*)c->d_misc + 256);
  cudaStream_t s = c->stream;
  EU_CUDA(cudaMemsetAsync(unsorted, 0, sizeof(int), s));
  if (OP == OP_MEAN) EU_CUDA(cudaMemsetAsync(cnt, 0, sizeof(float) * size, s));
  const bool vec = (D % 4 == 0) && aligned16(upd) && aligned16(out);
  const int G = vec ? group_lanes(D / 4) : (D >= 32 ? 32 : 1);
  const int tb = 256;
  if (E > 1) {
    k_check_sorted<<<(unsigned)ceil_div(E, tb), tb, 0, s>>>(idx, E, unsorted);
    EU_LAUNCHED();
  }
  const unsigned gs = (unsigned)ceil_div(size * G, tb), ge = (unsigned)ceil_div((E > 0 ? E : 1) * G, tb);
  EuProfScope ps(c, "scatter(sorted+fallback)", E);
  if (vec) k_scatter_sorted<OP, true><<<gs, tb, 0, s>>>(upd, D, idx, E, size, G, unsorted, out);
  else k_scatter_sorted<OP, false><<<gs, tb, 0, s>>>(upd, D, idx, E, size, G, unsorted, out);
  EU_LAUNCHED();
  k_fill_if<<<kSMs * 4, tb, 0, s>>>(out, size * D, OP == OP_MAX ? -1e9f : 0.f, unsorted);
  EU_LAUNCHED();
  if (E > 0) {
    if (vec) k_scatter_atomic<OP, true><<<ge, tb, 0, s>>>(upd, D, idx, E, G, unsorted, out, cnt);
    else k_scatter_atomic<OP, false><<<ge, tb, 0, s>>>(upd, D, idx, E, G, unsorted, out, cnt);
    EU_LAUNCHED();
  }
  if (OP == OP_MEAN) {
    k_mean_div<<<(unsigned)ceil_div(size * D, tb), tb, 0, s>>>(out, D, size, cnt, unsorted);
    EU_LAUNCHED();
  }
  return EU_OK;
}

// the fused SAGE reduction over a table of T placed at P into an output of O; v4: the float4 path's conditions hold
// (fanout_aggregate)
template <typename T, typename O, int P>
static int launch_sage_mean(eu_ctx* c, const DevGraph& d, const unsigned long long* ids, int64_t rows, const int32_t* reps,
                            const unsigned int* nrep, int32_t count, int32_t dim, bool mean, bool v4, unsigned blocks, O* out) {
  cudaStream_t s = c->stream;
  if (v4 && dim == 128) k_sage_mean<T, O, 1, true, P><<<blocks, 256, 0, s>>>(d, ids, rows, reps, nrep, count, mean, out);
  else if (v4 && dim == 256) k_sage_mean<T, O, 2, true, P><<<blocks, 256, 0, s>>>(d, ids, rows, reps, nrep, count, mean, out);
  else if (v4 && dim <= 128) k_sage_mean<T, O, 1, false, P><<<blocks, 256, 0, s>>>(d, ids, rows, reps, nrep, count, mean, out);
  else if (v4 && dim <= 256) k_sage_mean<T, O, 2, false, P><<<blocks, 256, 0, s>>>(d, ids, rows, reps, nrep, count, mean, out);
  else if (v4 && dim <= 512) k_sage_mean<T, O, 4, false, P><<<blocks, 256, 0, s>>>(d, ids, rows, reps, nrep, count, mean, out);
  else if (v4) k_sage_mean<T, O, 8, false, P><<<blocks, 256, 0, s>>>(d, ids, rows, reps, nrep, count, mean, out);
  else k_sage_mean_generic<T, O, P><<<blocks, 256, 0, s>>>(d, ids, rows, reps, nrep, count, dim, mean, out);
  EU_LAUNCHED();
  return EU_OK;
}

}  // namespace eu

using namespace eu;

extern "C" {

static int dense_feature(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int32_t dim, int32_t out_dtype, void* out,
                         const char* who) {
  if (!c || M < 0 || dim < 0 || (M > 0 && (!nodes || (dim > 0 && !out)))) { set_error("%s: bad argument", who); return EU_ERR_INVALID; }
  if (int rc = dtype_check(out_dtype, who, "output")) return rc;
  EU_CUDA(cudaSetDevice(c->g->device));
  if (M == 0 || dim == 0) return EU_OK;
  const DevGraph& d = c->g->d;
  int32_t soff, sdim;
  dense_slot(d, fid, &soff, &sdim);
  const bool vec = (dim % 4 == 0) && (d.feat_dim % 4 == 0) && (soff % 4 == 0) && (sdim % 4 == 0) && aligned4_elems(out, out_dtype);
  const int G = vec ? group_lanes(dim / 4) : (dim >= 32 ? 32 : 1);
  const unsigned blocks = capped_grid(ceil_div(M * G, 256), "EU_FEATURE_CTAS", 0);
  EuProfScope ps(c, "k_feature", M);
  with_feat(d, [&](auto t, auto p) {
    with_dtype(out_dtype, [&](auto o) {
      using T = typename decltype(t)::type;
      using O = typename decltype(o)::type;
      constexpr int P = decltype(p)::value;
      auto k = vec ? k_feature<T, O, true, P> : k_feature<T, O, false, P>;
      k<<<blocks, 256, 0, c->stream>>>(d, (const unsigned long long*)nodes, M, dim, G, soff, sdim, (O*)out);
    });
  });
  EU_LAUNCHED();
  return EU_OK;
}

int eu_gather(eu_ctx* c, const float* params, int64_t N, int64_t D, const int32_t* idx, int64_t E, float* out) {
  (void)N;
  if (!c || D <= 0 || E < 0 || (E > 0 && (!params || !idx || !out))) { set_error("eu_gather: bad argument"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  if (E == 0) return EU_OK;
  const bool vec = (D % 4 == 0) && aligned16(params) && aligned16(out);
  const int G = vec ? group_lanes(D / 4) : (D >= 32 ? 32 : 1);
  const unsigned blocks = (unsigned)ceil_div(E * G, 256);
  if (vec) k_gather<true><<<blocks, 256, 0, c->stream>>>(params, D, idx, E, G, out);
  else k_gather<false><<<blocks, 256, 0, c->stream>>>(params, D, idx, E, G, out);
  EU_LAUNCHED();
  return EU_OK;
}

int eu_get_dense_feature(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int32_t dim, float* out) {
  return dense_feature(c, nodes, M, fid, dim, EU_FEAT_F32, out, "eu_get_dense_feature");
}
int eu_get_dense_feature_out_dtype(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int32_t dim, int32_t out_dtype, void* out) {
  return dense_feature(c, nodes, M, fid, dim, out_dtype, out, "eu_get_dense_feature_out_dtype");
}

int eu_scatter_add(eu_ctx* c, const float* u, int64_t D, const int32_t* idx, int64_t E, int64_t size, float* out) {
  return scatter<OP_ADD>(c, u, D, idx, E, size, out);
}
int eu_scatter_max(eu_ctx* c, const float* u, int64_t D, const int32_t* idx, int64_t E, int64_t size, float* out) {
  return scatter<OP_MAX>(c, u, D, idx, E, size, out);
}
int eu_scatter_mean(eu_ctx* c, const float* u, int64_t D, const int32_t* idx, int64_t E, int64_t size, float* out) {
  return scatter<OP_MEAN>(c, u, D, idx, E, size, out);
}

static int fanout_aggregate(eu_ctx* c, const int64_t* nbr_ids, int64_t rows, int32_t count, int32_t dim, bool mean, int32_t out_dtype,
                            void* out, const char* who) {
  if (!c || rows < 0 || count < 0 || dim <= 0 || (rows > 0 && (!nbr_ids || !out))) { set_error("%s: bad argument", who); return EU_ERR_INVALID; }
  if (int rc = dtype_check(out_dtype, who, "output")) return rc;
  EU_CUDA(cudaSetDevice(c->g->device));
  if (rows == 0) return EU_OK;
  cudaStream_t s = c->stream;
  const DevGraph& d = c->g->d;
  const unsigned long long* ids = (const unsigned long long*)nbr_ids;
  // otherwise k_sage_mean reduces every row (reps == null); the dedup scratch holds 32-bit row indices
  const bool dedup = rows >= kRepeatMinRows && rows < ((int64_t)1 << 31);
  int64_t cap = 64;   // table slots of this call: a power of two >= 2 * rows
  while (cap < 2 * rows) cap <<= 1;
  if (dedup) {
    int rc = agg_reserve(c, rows, cap);
    if (rc) return rc;
    EU_CUDA(cudaMemsetAsync(c->d_agg_nrep, 0, sizeof(unsigned int), s));
    EuProfScope ps(c, "k_sage_classify", rows);
    k_sage_classify<<<capped_grid(ceil_div(rows, 256), "EU_SAGE_CTAS", 0), 256, 0, s>>>(d, ids, rows, count, c->d_agg_tab, (unsigned long long)cap - 1,
                                                                                      c->d_agg_src, c->d_agg_rep, c->d_agg_slot, c->d_agg_nrep);
    EU_LAUNCHED();
  }
  const unsigned blocks = capped_grid(ceil_div(rows * 32, 256), "EU_SAGE_CTAS", 0);
  const int32_t* reps = dedup ? c->d_agg_rep : nullptr;
  const unsigned int* nrep = c->d_agg_nrep;
  { EuProfScope ps(c, mean ? "k_sage_mean" : "k_sage_add", rows);
    // float4 path: one slot of the full stored width, a multiple of 4 floats up to 1024 (D = 64 of configs[4], 128, 256, ...),
    // on a table and an output aligned to four elements (16 bytes of f32, 8 of bf16)
    const bool v4 = d.n < ((int64_t)1 << 31) && d.n_slots == 1 && dim == d.feat_dim && (dim & 3) == 0 && dim <= 1024 &&
                    aligned4_elems(out, out_dtype) && aligned4_elems(d.feat, d.feat_dtype);
    const int rc = with_feat(d, [&](auto t, auto p) {
      return with_dtype(out_dtype, [&](auto o) {
        using O = typename decltype(o)::type;
        return launch_sage_mean<typename decltype(t)::type, O, decltype(p)::value>(c, d, ids, rows, reps, nrep, count, dim, mean, v4, blocks,
                                                                                   (O*)out);
      });
    });
    if (rc) return rc; }
  if (!dedup) return EU_OK;
  { EuProfScope ps(c, "k_sage_broadcast", rows);
    const bool vec = (dim & 3) == 0 && aligned4_elems(out, out_dtype);
    const int G = vec ? group_lanes(dim / 4) : (dim >= 32 ? 32 : 1);
    const unsigned bb = capped_grid(ceil_div(rows * G, 256), "EU_SAGE_CTAS", 0);
    with_dtype(out_dtype, [&](auto o) {
      using O = typename decltype(o)::type;
      auto k = vec ? k_sage_broadcast<O, true> : k_sage_broadcast<O, false>;
      k<<<bb, 256, 0, s>>>(c->d_agg_src, rows, dim, G, c->d_agg_slot, nrep, c->d_agg_tab, (O*)out);
    }); }
  EU_LAUNCHED();
  return EU_OK;
}

int eu_sage_mean_aggregate(eu_ctx* c, const int64_t* nbr_ids, int64_t rows, int32_t count, int32_t dim, float* out) {
  return fanout_aggregate(c, nbr_ids, rows, count, dim, true, EU_FEAT_F32, out, "eu_sage_mean_aggregate");
}
int eu_sage_mean_aggregate_out_dtype(eu_ctx* c, const int64_t* nbr_ids, int64_t rows, int32_t count, int32_t dim, int32_t out_dtype,
                                     void* out) {
  return fanout_aggregate(c, nbr_ids, rows, count, dim, true, out_dtype, out, "eu_sage_mean_aggregate_out_dtype");
}
// the scatter_add variant over the same fixed-fanout blocks (aggr='add': GCN / the per-relation sums of configs[4]):
// get_dense_feature + scatter_add over edge_src = repeat(range(rows), count), fused
int eu_sage_add_aggregate(eu_ctx* c, const int64_t* nbr_ids, int64_t rows, int32_t count, int32_t dim, float* out) {
  return fanout_aggregate(c, nbr_ids, rows, count, dim, false, EU_FEAT_F32, out, "eu_sage_mean_aggregate");
}
int eu_sage_add_aggregate_out_dtype(eu_ctx* c, const int64_t* nbr_ids, int64_t rows, int32_t count, int32_t dim, int32_t out_dtype,
                                    void* out) {
  return fanout_aggregate(c, nbr_ids, rows, count, dim, false, out_dtype, out, "eu_sage_add_aggregate_out_dtype");
}

}  // extern "C"
