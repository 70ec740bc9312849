// Peer-memory exchange for the sharded path: the all-to-all of a hop / feature fetch is done by the kernels
// themselves with loads/stores on NVLink peer mappings -- no NCCL call, no host-visible counts, no host sync,
// CUDA-graph capturable.  Replaces euler's ID_SPLIT -> REMOTE(gRPC) -> IDX_MERGE/DATA_MERGE
// (euler/core/kernels/id_split_op.cc:46-99, remote_op.cc:60-146, idx_merge_op.cc:32-78).
//
// Every rank owns one symmetric region (same layout everywhere, cudaIpc-mapped into every peer):
//   header | inbox_ids[N][cap] | inbox_src[N][cap] | out_eng | out_ids | out_w | out_t | out_rows
// One exchange =
//   requester  k_bucket_count/place (shard.cu): stable bucket by owner whose placement pass writes each id (+ the original
//                                row index of the seed) straight into owner o's inbox segment [me]; the last CTA publishes the
//                                counts and raises flagA[me] <- epoch on every owner
//   owner      k_sym_wait_in / k_sym_gather_pad : waits for flagA of every source, finds the batch boundaries, builds the
//                                zero-padded sampleNB input (id 0 = "exists nowhere")
//   owner      hop() / gather  : samples the padded inbox as ONE sampleNB call on its own engine (sources in rank order,
//                                each in batch order: the order pinned in euler_b200/sharded.py) -- or, for features,
//   owner      k_sym_reply_*   : writes every result row DIRECTLY into the requester's output arrays at the seed's
//                                original position (TF packing done here), then flagB[me] <- epoch on the requester
//   requester  k_sym_wait      : waits for flagB of every owner; its outputs are complete, already in request order.
// Flags are monotonic epochs kept on the device; all waits are bounded (hdr->error is set on timeout instead of hanging).
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "internal.h"
#include "sym.cuh"

namespace eu {

// Bounded spin until *flag >= want.  A wait that runs out of time POISONS the exchange instead of letting stale data
// through: it sets error in this rank's header, the wait kernel then stores error into every peer's header, every later
// kernel of a poisoned region returns at once (no replies, no flags), and every spin polls its own error word, so the
// whole group drains within microseconds and eu_sym_error() is nonzero on every rank.  A poisoned eu_sym is dead: destroy it.
__device__ __forceinline__ bool spin_until(const unsigned int* flag, unsigned int want, SymHeader* h, long long limit) {
  const long long t0 = clock64();
  while ((int)(ld_acquire_sys(flag) - want) < 0) {
    __nanosleep(200);
    if (ld_volatile_i32(&h->error)) return false;
    if (clock64() - t0 > limit) { h->error = 1; return false; }
  }
  return true;
}

__device__ __forceinline__ void propagate_error(SymHeader* h, char* const* pb_tab, int N) {
  // called by threads 0..N-1 after a barrier that follows the spins
  if (threadIdx.x < N && ld_volatile_i32(&h->error)) {
    *reinterpret_cast<volatile int*>(&hdr_of(pb_tab[threadIdx.x])->error) = 1;
    __threadfence_system();
  }
}

// ---- owner: wait for every source (one small block spins; nothing else of the GPU is held).  A batched hop also
// needs the batch boundaries inside every source's segment: the bucket is stable and src = g*rows_b + position, so
// batch g of source s is the slice [seg_lo[s][g], seg_lo[s][g+1]) -- N*(nb+1) binary searches, done here.
__global__ void __launch_bounds__(256) k_sym_wait_in(char* base, char* const* pb_tab, SymLayout lay, int N, int nb, int64_t rows_b,
                                                     int expect_total /* every source must have bucketed this many ids; -1 = any */,
                                                     int32_t* __restrict__ seg_lo /* [N][nb+1] or null */,
                                                     int32_t* __restrict__ boff /* [nb][N+1] or null */,
                                                     int32_t* __restrict__ act /* [nb] or null */) {
  SymHeader* h = hdr_of(base);
  if (threadIdx.x < N) {
    const bool ok = spin_until(&h->flagA[threadIdx.x], h->epoch, h, lay.timeout_cycles);
    // the segment stride is fixed at creation, but the batch geometry (nb x rows) must be the same on every rank
    if (ok && expect_total >= 0 && ld_volatile_i32(&h->in_total[threadIdx.x]) != expect_total) h->error = 2;
  }
  __syncthreads();
  propagate_error(h, pb_tab, N);
  if (ld_volatile_i32(&h->error)) {   // poisoned: the hop that follows samples nothing
    if (act) for (int g = threadIdx.x; g < nb; g += blockDim.x) act[g] = 0;
    if (boff) for (int i = threadIdx.x; i < nb * (N + 1); i += blockDim.x) boff[i] = 0;
    if (seg_lo) for (int i = threadIdx.x; i < N * (nb + 1); i += blockDim.x) seg_lo[i] = 0;
    return;
  }
  if (!seg_lo) return;
  __syncthreads();
  const int32_t* src = reinterpret_cast<const int32_t*>(base + lay.off_inbox_src);
  for (int i = threadIdx.x; i < N * (nb + 1); i += blockDim.x) {
    const int s = i / (nb + 1), g = i - s * (nb + 1);
    const int32_t n_s = *reinterpret_cast<volatile int*>(&h->in_cnt[s]);
    const int32_t* seg = src + (int64_t)s * lay.cap;
    const int32_t key = (int32_t)(g * rows_b);
    int32_t lo = 0, hi = n_s;
    while (lo < hi) {
      const int32_t mid = lo + ((hi - lo) >> 1);
      if (__ldcg(seg + mid) < key) lo = mid + 1; else hi = mid;
    }
    seg_lo[i] = lo;
  }
  if (!boff) return;
  __syncthreads();
  // batch g of the owner's sampleNB input = the requests of source 0..N-1 for g, back to back: boff[g][s] = where source
  // s starts, act[g] = how many rows the batch really has (the launch is sized for N * rows_b)
  for (int g = threadIdx.x; g < nb; g += blockDim.x) {
    int32_t run = 0;
    for (int s = 0; s < N; ++s) {
      boff[g * (N + 1) + s] = run;
      run += seg_lo[s * (nb + 1) + g + 1] - seg_lo[s * (nb + 1) + g];
    }
    boff[g * (N + 1) + N] = run;
    act[g] = run;
  }
}

// ---- owner: the sampleNB input of batch g = the requests of source 0..N-1 for that batch, back to back (compact: the
// kernels of hop() learn the real row count of every batch from act[g]; nothing is zero-padded)  ->  pad[g][0 .. act[g])
__device__ __forceinline__ int src_of(const int32_t* __restrict__ bo /* [N+1] */, int N, int32_t p) {
  int s = 0;
  while (s + 1 < N && p >= bo[s + 1]) ++s;
  return s;
}

__global__ void __launch_bounds__(256) k_sym_gather_pad(const char* base, SymLayout lay, int N, int nb, int64_t rows_b,
                                                        const int32_t* __restrict__ seg_lo, const int32_t* __restrict__ boff,
                                                        unsigned long long* __restrict__ pad, HashSlot* tabs, int64_t tab_cap) {
  // per batch g only the bo[N] requests that really arrived; each is also entered into the hop's dedup table (exact-RNG
  // mode: tabs != null), so the owner's sampleNB needs no insert pass of its own
  const unsigned long long* ids = reinterpret_cast<const unsigned long long*>(base + lay.off_inbox_ids);
  const int64_t cap_b = (int64_t)N * rows_b;
  const int32_t stride = (int32_t)(gridDim.x * blockDim.x);
  for (int g = 0; g < nb; ++g) {
    const int32_t* bo = boff + g * (N + 1);
    const int32_t live = bo[N];                                            // == the rows_act[g] hop() is given (k_sym_wait_in)
    const unsigned long long mask = (unsigned long long)dedup_cap_eff(tab_cap, &live, 0) - 1;
    for (int32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < live; p += stride) {
      const int s = src_of(bo, N, p);
      const unsigned long long id = ids[(int64_t)s * lay.cap + seg_lo[s * (nb + 1) + g] + (p - bo[s])];
      pad[(int64_t)g * cap_b + p] = id;
      if (tabs) {
        const unsigned peers = __match_any_sync(__activemask(), id);       // runs of equal ids: the lowest lane carries the minimum index
        if ((threadIdx.x & 31) == __ffs(peers) - 1) dedup_insert_one(tabs + (int64_t)g * (tab_cap + 1), mask, id, p);
      }
    }
  }
}

// ---- owner: sampled rows of the padded inbox -> requester's outputs at the original positions (+ TF packing)
__global__ void __launch_bounds__(256) k_sym_reply_sample(char* const* __restrict__ pb_tab, SymLayout lay, int me, int N, int nb, int64_t rows_b,
                                                          const int32_t* __restrict__ seg_lo, const int32_t* __restrict__ boff,
                                                          int32_t count,
                                                          long long default_node, const long long* __restrict__ r_ids,
                                                          const float* __restrict__ r_w, const int32_t* __restrict__ r_t,
                                                          bool want_packed) {
  char* base = pb_tab[me];
  SymHeader* mine = hdr_of(base);
  const int32_t* src = reinterpret_cast<const int32_t*>(base + lay.off_inbox_src);
  __shared__ bool s_last;
  __shared__ int s_err;
  if (threadIdx.x == 0) s_err = ld_volatile_i32(&mine->error);
  __syncthreads();
  if (s_err) return;   // poisoned exchange: no replies, no flags
  // per batch g only the bo[N] rows the owner really received (its input is compact; the arrays are strided for the worst case)
  const int64_t cap_b = (int64_t)N * rows_b;
  const uint32_t stride = gridDim.x * blockDim.x;
  for (int g = 0; g < nb; ++g) {
    const int32_t* bo = boff + g * (N + 1);
    const uint32_t live = (uint32_t)bo[N] * (uint32_t)count;       // < 2^31: rows and count are bounded by the region's capacity
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < live; t += stride) {
      const int32_t p = (int32_t)(t / (uint32_t)count);
      const int32_t j = (int32_t)(t - (uint32_t)p * (uint32_t)count);
      const int64_t row = (int64_t)g * cap_b + p;
      const int64_t tid = row * count + j;
      const int s = src_of(bo, N, p);
      const int64_t dst = (int64_t)src[(int64_t)s * lay.cap + seg_lo[s * (nb + 1) + g] + (p - bo[s])] * count + j;   // requester's flat slot [g][pos][j]
      const long long id = r_ids[tid];
      const bool keep = r_ids[row * count] != 0;   // tf_euler/kernels/sample_neighbor_op.cc:114-122
      char* pb = pb_tab[s];
      reinterpret_cast<long long*>(pb + lay.off_eng)[dst] = id;
      if (want_packed) {
        reinterpret_cast<long long*>(pb + lay.off_ids)[dst] = keep ? id : default_node;
        reinterpret_cast<float*>(pb + lay.off_w)[dst] = keep ? r_w[tid] : 0.f;
        reinterpret_cast<int32_t*>(pb + lay.off_t)[dst] = keep ? r_t[tid] : -1;
      }
    }
  }
  __syncthreads();   // CTA's stores happen-before thread 0's fence (barrier + cumulativity): one system fence per CTA
  if (threadIdx.x == 0) { __threadfence_system(); s_last = atomicAdd(&mine->done, 1u) == gridDim.x - 1; }
  __syncthreads();
  if (!s_last) return;
  if (threadIdx.x < N) __threadfence_system();   // ticket observed (barrier) -> ordered before the flag stores
  if (threadIdx.x == 0) mine->done = 0;
  if (threadIdx.x < N) st_release_sys(&hdr_of(pb_tab[threadIdx.x])->flagB[me], mine->epoch);
}

// ---- owner: feature rows gathered from the local shard straight into the requester's output (G lanes per row)
__global__ void __launch_bounds__(256) k_sym_reply_feature(DevGraph g, char* const* __restrict__ pb_tab, SymLayout lay, int me, int N,
                                                           int32_t dim, int32_t soff, int32_t sdim, int G) {
  char* base = pb_tab[me];
  SymHeader* mine = hdr_of(base);
  const unsigned long long* ids = reinterpret_cast<const unsigned long long*>(base + lay.off_inbox_ids);
  const int32_t* src = reinterpret_cast<const int32_t*>(base + lay.off_inbox_src);
  __shared__ bool s_last;
  __shared__ int s_err;
  if (threadIdx.x == 0) s_err = ld_volatile_i32(&mine->error);
  __syncthreads();
  if (s_err) return;
  const int sh = 31 - __clz(G);
  const int sub = (int)(threadIdx.x & (G - 1));
  for (int s = 0; s < N; ++s) {   // segment s holds in_cnt[s] requests (the stride lay.cap is fixed at creation)
    const int64_t n_s = mine->in_cnt[s];
    float* obase = reinterpret_cast<float*>(pb_tab[s] + lay.off_rows);
    for (int64_t k = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> sh; k < n_s; k += ((int64_t)gridDim.x * blockDim.x) >> sh) {
      const int64_t row = (int64_t)s * lay.cap + k;
      const int64_t gr = sdim > 0 ? lookup_row(g, ids[row]) : -1;
      const float* f = gr >= 0 ? feat_cols<float>(g) + gr * (int64_t)g.feat_dim + soff : nullptr;
      float* o = obase + (int64_t)src[row] * dim;
      for (int32_t d = sub * 4; d < dim; d += G * 4) {   // dim, sdim, soff multiples of 4 (checked by the launcher)
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (f && d < sdim) v = __ldg(reinterpret_cast<const float4*>(f + d));
        *reinterpret_cast<float4*>(o + d) = v;
      }
    }
  }
  __syncthreads();   // CTA's stores happen-before thread 0's fence (barrier + cumulativity): one system fence per CTA
  if (threadIdx.x == 0) { __threadfence_system(); s_last = atomicAdd(&mine->done, 1u) == gridDim.x - 1; }
  __syncthreads();
  if (!s_last) return;
  if (threadIdx.x < N) __threadfence_system();   // ticket observed (barrier) -> ordered before the flag stores
  if (threadIdx.x == 0) mine->done = 0;
  if (threadIdx.x < N) st_release_sys(&hdr_of(pb_tab[threadIdx.x])->flagB[me], mine->epoch);
}

// ---- requester: wait for every owner's replies
__global__ void k_sym_wait(char* base, char* const* pb_tab, SymLayout lay, int N) {
  SymHeader* h = hdr_of(base);
  if (threadIdx.x < N) spin_until(&h->flagB[threadIdx.x], h->epoch, h, lay.timeout_cycles);
  __syncthreads();
  propagate_error(h, pb_tab, N);
}

// ---- fused sharded SAGE mean.  The requester pushes the neighbor ids of its fixed-fanout block (flat [rows*count],
// src index = flat position, stable bucket => ascending inside every segment); the owner sums the features of ITS ids
// per destination row, j ascending, and stores ONE partial row per (owner, destination) into the requester's `part`
// region; the requester adds the N partials in rank order and divides.  NVLink carries rows*dim floats per owner instead
// of rows*count*dim: the hop-2 features never cross the link (sage_dataflow.py:43-46 + mp_ops.py:65-69 fused with the
// REMOTE get_dense_feature they follow).
__device__ __forceinline__ int32_t warp_lower_bound(const int32_t* __restrict__ a, int32_t n, int32_t key, int lane) {
  int32_t lo = 0, hi = n;
  while (hi - lo > 32) {
    const int32_t len = hi - lo;
    const int32_t p = lo + (int32_t)(((int64_t)(lane + 1) * len) / 33);   // lo < p_0 <= .. <= p_31 < hi
    const int c = __popc(__ballot_sync(0xffffffffu, a[p] < key));          // sorted: a prefix of the probes is below
    const int32_t below = __shfl_sync(0xffffffffu, p, c > 0 ? c - 1 : 0);
    const int32_t above = __shfl_sync(0xffffffffu, p, c < 32 ? c : 31);
    lo = c > 0 ? below + 1 : lo;
    hi = c < 32 ? above : hi;
  }
  const bool b = lo + lane < hi && a[lo + lane] < key;
  return lo + __popc(__ballot_sync(0xffffffffu, b));
}

// One warp serves kSageR consecutive destinations of one source: one segment search, then a walk over their inbox
// entries (id -> row lookups 32 at a time across the lanes, 4 feature rows in flight), flushing a partial row -- zeros
// when this shard owns none of a destination's neighbors -- whenever the destination changes.
static constexpr int kSageRMax = 32;   // destinations per warp: R = 8 or 32 (one 32-bit presence mask per group)
template <int NV>   // feat_dim == dim == NV*128
__global__ void __launch_bounds__(256) k_sym_reply_sage(DevGraph g, char* const* __restrict__ pb_tab, SymLayout lay, int me, int N, int64_t rows,
                                                        int32_t count, int kSageR) {
  char* base = pb_tab[me];
  SymHeader* mine = hdr_of(base);
  const unsigned long long* ids = reinterpret_cast<const unsigned long long*>(base + lay.off_inbox_ids);
  const int32_t* src = reinterpret_cast<const int32_t*>(base + lay.off_inbox_src);
  __shared__ bool s_last;
  __shared__ int s_err;
  if (threadIdx.x == 0) s_err = ld_volatile_i32(&mine->error);
  __syncthreads();
  if (s_err) return;
  const int lane = threadIdx.x & 31;
  constexpr int32_t fd = NV * 128;
  const float* __restrict__ feat = feat_cols<float>(g) + lane * 4;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t gps = (rows + kSageR - 1) / kSageR;   // destination groups per source
  for (int64_t w = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; w < (int64_t)N * gps; w += nwarps) {
    const int s = (int)(w / gps);
    const int64_t d0 = (w - (int64_t)s * gps) * kSageR;
    const int nd = (int)(rows - d0 < kSageR ? rows - d0 : kSageR);
    const int32_t n_s = mine->in_cnt[s];
    const int32_t* seg = src + (int64_t)s * lay.cap;
    const unsigned long long* sid = ids + (int64_t)s * lay.cap;
    const int32_t key_lo = (int32_t)(d0 * count), key_hi = (int32_t)((d0 + nd) * count);
    float* o = reinterpret_cast<float*>(pb_tab[s] + lay.off_rows) + ((int64_t)me * rows + d0) * fd + lane * 4;
    int cur = 0;   // next destination (relative to d0) whose partial row is still open
    bool any = false;        // the open destination has at least one row of this shard
    unsigned present = 0;    // bit d: a partial row was stored for destination d0 + d (empty partials are not sent)
    float4 acc[NV];
#pragma unroll
    for (int v = 0; v < NV; ++v) acc[v] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int32_t e0 = warp_lower_bound(seg, n_s, key_lo, lane);; e0 += 32) {
      const int32_t e = e0 + lane;
      int32_t sv = 0;
      const bool in = e < n_s && (sv = seg[e]) < key_hi;
      int32_t my = -1, md = 0;
      if (in) { my = (int32_t)lookup_row(g, sid[e]); md = (sv - key_lo) / count; }
      const int nin = __popc(__ballot_sync(0xffffffffu, in));
      unsigned valid = __ballot_sync(0xffffffffu, my >= 0);
      while (valid) {   // warp-uniform
        float4 v[4][NV];
        int dq[4];
        int n = 0;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          if (valid) {
            const int j = __ffs(valid) - 1;
            valid &= valid - 1;
            const int32_t row = __shfl_sync(0xffffffffu, my, j);
            dq[q] = __shfl_sync(0xffffffffu, md, j);
            const float* p = feat + (int64_t)row * fd;
#pragma unroll
            for (int t = 0; t < NV; ++t) v[q][t] = __ldg(reinterpret_cast<const float4*>(p + t * 128));
            n = q + 1;
          }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          if (q < n) {
            if (cur < dq[q]) {
              if (any) {
#pragma unroll
                for (int t = 0; t < NV; ++t) { *reinterpret_cast<float4*>(o + (int64_t)cur * fd + t * 128) = acc[t]; acc[t] = make_float4(0.f, 0.f, 0.f, 0.f); }
                present |= 1u << cur;
                any = false;
              }
              cur = dq[q];
            }
            any = true;
#pragma unroll
            for (int t = 0; t < NV; ++t) {
              acc[t].x = __fadd_rn(acc[t].x, v[q][t].x); acc[t].y = __fadd_rn(acc[t].y, v[q][t].y);
              acc[t].z = __fadd_rn(acc[t].z, v[q][t].z); acc[t].w = __fadd_rn(acc[t].w, v[q][t].w);
            }
          }
        }
      }
      if (nin < 32) break;
    }
    if (any) {
#pragma unroll
      for (int t = 0; t < NV; ++t) *reinterpret_cast<float4*>(o + (int64_t)cur * fd + t * 128) = acc[t];
      present |= 1u << cur;
    }
    if (lane == 0) reinterpret_cast<unsigned int*>(pb_tab[s] + lay.off_flags)[(int64_t)me * gps + (w - (int64_t)s * gps)] = present;
  }
  __syncthreads();   // CTA's stores happen-before thread 0's fence (barrier + cumulativity): one system fence per CTA
  if (threadIdx.x == 0) { __threadfence_system(); s_last = atomicAdd(&mine->done, 1u) == gridDim.x - 1; }
  __syncthreads();
  if (!s_last) return;
  if (threadIdx.x < N) __threadfence_system();   // ticket observed (barrier) -> ordered before the flag stores
  if (threadIdx.x == 0) mine->done = 0;
  if (threadIdx.x < N) st_release_sys(&hdr_of(pb_tab[threadIdx.x])->flagB[me], mine->epoch);
}

// any width: lanes over columns, entries serial (slow path, same sums)
__global__ void __launch_bounds__(256) k_sym_reply_sage_generic(DevGraph g, char* const* __restrict__ pb_tab, SymLayout lay, int me, int N, int64_t rows,
                                                                int32_t count, int32_t dim) {
  char* base = pb_tab[me];
  SymHeader* mine = hdr_of(base);
  const unsigned long long* ids = reinterpret_cast<const unsigned long long*>(base + lay.off_inbox_ids);
  const int32_t* src = reinterpret_cast<const int32_t*>(base + lay.off_inbox_src);
  __shared__ bool s_last;
  __shared__ int s_err;
  if (threadIdx.x == 0) s_err = ld_volatile_i32(&mine->error);
  __syncthreads();
  if (s_err) return;
  const int lane = threadIdx.x & 31;
  const int32_t fd = g.feat_dim;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t w = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; w < (int64_t)N * rows; w += nwarps) {
    const int s = (int)(w / rows);
    const int64_t d = w - (int64_t)s * rows;
    const int32_t n_s = mine->in_cnt[s];
    const int32_t* seg = src + (int64_t)s * lay.cap;
    const unsigned long long* sid = ids + (int64_t)s * lay.cap;
    const int32_t key_hi = (int32_t)((d + 1) * count);
    const int32_t e_lo = warp_lower_bound(seg, n_s, (int32_t)(d * count), lane);
    float* o = reinterpret_cast<float*>(pb_tab[s] + lay.off_rows) + ((int64_t)me * rows + d) * dim;
    for (int32_t c0 = 0; c0 < dim; c0 += 32) {
      const int32_t col = c0 + lane;
      float acc = 0.f;
      for (int32_t e = e_lo; e < n_s && seg[e] < key_hi; ++e) {   // warp-uniform
        const int64_t row = lookup_row(g, sid[e]);
        if (row >= 0 && col < fd && col < dim) acc = __fadd_rn(acc, __ldg(feat_cols<float>(g) + row * (int64_t)fd + col));
      }
      if (col < dim) o[col] = acc;
    }
  }
  __syncthreads();   // CTA's stores happen-before thread 0's fence (barrier + cumulativity): one system fence per CTA
  if (threadIdx.x == 0) { __threadfence_system(); s_last = atomicAdd(&mine->done, 1u) == gridDim.x - 1; }
  __syncthreads();
  if (!s_last) return;
  if (threadIdx.x < N) __threadfence_system();   // ticket observed (barrier) -> ordered before the flag stores
  if (threadIdx.x == 0) mine->done = 0;
  if (threadIdx.x < N) st_release_sys(&hdr_of(pb_tab[threadIdx.x])->flagB[me], mine->epoch);
}

__device__ __forceinline__ float vadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float4 vadd(float4 a, float4 b) { return make_float4(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z), __fadd_rn(a.w, b.w)); }
__device__ __forceinline__ float vzero(float) { return 0.f; }
__device__ __forceinline__ float4 vzero(float4) { return make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ float vdiv(float a, float d) { return __fdiv_rn(a, d); }
__device__ __forceinline__ float4 vdiv(float4 a, float d) { return make_float4(__fdiv_rn(a.x, d), __fdiv_rn(a.y, d), __fdiv_rn(a.z, d), __fdiv_rn(a.w, d)); }

// requester: out[d,:] = (part[0][d,:] + part[1][d,:] + ...) / (count + 1e-7), rank order
template <typename V>
__global__ void __launch_bounds__(256) k_sym_sage_reduce(const V* __restrict__ part, const unsigned int* __restrict__ flags, int N,
                                                         int64_t rows, int32_t vdim /* V units per row */, int32_t count, int kSageR,
                                                         V* __restrict__ out) {
  const float denom = __fadd_rn((float)count, 1e-7f);
  const int64_t total = rows * vdim;
  const int64_t gps = (rows + kSageR - 1) / kSageR;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t d = i / vdim;
    V acc = vzero(V());
    for (int o = 0; o < N; ++o)   // absent partial == a row of +0.0: skipping it is exact (acc is never -0.0)
      if ((flags[(int64_t)o * gps + d / kSageR] >> (d % kSageR)) & 1u) acc = vadd(acc, __ldcs(part + (int64_t)o * total + i));
    out[i] = vdiv(acc, denom);
  }
}

static inline unsigned sym_grid(int64_t threads) {   // persistent: at most 8 CTAs of 256 per SM
  static int per_sm = 0;
  if (!per_sm) { const char* e = getenv("EU_SYM_CTAS"); per_sm = e ? std::min(8, std::max(1, atoi(e))) : 8; }
  return (unsigned)std::min<int64_t>(std::max<int64_t>(ceil_div(threads, 256), 1), kSMs * (int64_t)per_sm);
}
// reply kernels are NVLink-store bound: fewer resident CTAs keep the link busy and leave SM slots to the compute
// kernels of the other lanes
static inline unsigned reply_grid(int64_t threads) {
  static int per_sm = 0;
  if (!per_sm) { const char* e = getenv("EU_SYM_REPLY_CTAS"); per_sm = e ? std::max(1, atoi(e)) : 4; }
  return (unsigned)std::min<int64_t>(std::max<int64_t>(ceil_div(threads, 256), 1), kSMs * (int64_t)per_sm);
}

static inline int64_t a256(int64_t x) { return (x + 255) & ~(int64_t)255; }

}  // namespace eu

struct eu_sym {
  eu_ctx* c = nullptr;
  int rank = 0, world = 1;
  eu::SymLayout lay{};
  eu::SymPeers peers{};
  char** d_peers = nullptr;   // device copy of peers.base (what the kernels index)
  char* base = nullptr;
  bool connected = false;
  // local scratch
  int64_t* d_sorted = nullptr; int32_t* d_src = nullptr; int64_t* d_counts = nullptr; int64_t* d_offs = nullptr;
  int64_t* d_rids = nullptr; float* d_rw = nullptr; int32_t* d_rt = nullptr;
  unsigned long long* d_pad = nullptr; int32_t* d_seglo = nullptr; int32_t* d_boff = nullptr; int32_t* d_act = nullptr;
  int64_t scratch_rows = 0, scratch_slots = 0, scratch_pad = 0;
};

using namespace eu;

extern "C" {

int eu_sym_create(eu_ctx* c, int32_t rank, int32_t world, int64_t max_rows, int32_t max_count, int64_t max_feat_rows,
                  int32_t max_dim, eu_sym** out, void* handle_out /* 64 bytes */) {
  if (!c || !out || !handle_out || world < 1 || world > kSymMaxRanks || rank < 0 || rank >= world || max_rows < 0 ||
      max_count < 1 || max_feat_rows < 0 || max_dim < 0) { set_error("eu_sym_create: bad argument"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  eu_sym* s = new eu_sym();
  s->c = c; s->rank = rank; s->world = world;
  SymLayout& L = s->lay;
  L.cap = std::max<int64_t>(std::max(max_rows, max_feat_rows), 1);
  L.max_out = max_rows * max_count;
  L.max_rows_f = max_feat_rows;
  L.max_dim = max_dim;
  {
    // bound of every flag wait: generous (a peer may sit in a cudaMalloc, a GC pause or a data-loader stall), and when it
    // does expire the exchange is poisoned on every rank instead of continuing on stale data (spin_until)
    const char* e = getenv("EU_SYM_TIMEOUT_S");
    const double sec = e && atof(e) > 0 ? atof(e) : 30.0;
    int khz = 1900000;
    cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, c->g->device);
    L.timeout_cycles = (long long)(sec * 1e3 * (double)khz);
  }
  int64_t off = a256(sizeof(SymHeader));
  L.off_inbox_ids = off; off += a256(8 * L.cap * world);
  L.off_inbox_src = off; off += a256(4 * L.cap * world);
  L.off_eng = off; off += a256(8 * L.max_out);
  L.off_ids = off; off += a256(8 * L.max_out);
  L.off_w = off; off += a256(4 * L.max_out);
  L.off_t = off; off += a256(4 * L.max_out);
  L.off_rows = off; off += a256(4 * max_feat_rows * (int64_t)max_dim);
  L.off_flags = off; off += a256((max_feat_rows / 8 + 1) * 4 * (int64_t)world);   // partial-row presence masks of eu_sym_sage_mean
  L.bytes = off;
  cudaError_t e = cudaMalloc(&s->base, (size_t)L.bytes);
  if (e != cudaSuccess) { set_error("cudaMalloc(%lld) -> %s", (long long)L.bytes, cudaGetErrorString(e)); delete s; return EU_ERR_CUDA; }
  cudaMemset(s->base, 0, (size_t)L.bytes);
  cudaIpcMemHandle_t h;
  e = cudaIpcGetMemHandle(&h, s->base);
  if (e != cudaSuccess) { set_error("cudaIpcGetMemHandle -> %s", cudaGetErrorString(e)); cudaFree(s->base); delete s; return EU_ERR_CUDA; }
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "ipc handle size");
  memcpy(handle_out, &h, 64);
  s->peers.base[rank] = s->base;
  EU_CUDA(cudaMalloc(&s->d_peers, sizeof(char*) * kSymMaxRanks));
  EU_CUDA(cudaMemcpy(s->d_peers, s->peers.base, sizeof(char*) * kSymMaxRanks, cudaMemcpyHostToDevice));
  EU_CUDA(cudaDeviceSynchronize());
  *out = s;
  return EU_OK;
}

// handles: world x 64 bytes (all_gather of eu_sym_create's handle_out, rank order)
int eu_sym_connect(eu_sym* s, const void* handles) {
  if (!s || !handles) { set_error("eu_sym_connect: bad argument"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(s->c->g->device));
  for (int r = 0; r < s->world; ++r) {
    if (r == s->rank) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, (const char*)handles + 64 * r, 64);
    void* p = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) { set_error("cudaIpcOpenMemHandle(rank %d) -> %s", r, cudaGetErrorString(e)); return EU_ERR_CUDA; }
    s->peers.base[r] = (char*)p;
  }
  EU_CUDA(cudaMemcpy(s->d_peers, s->peers.base, sizeof(char*) * kSymMaxRanks, cudaMemcpyHostToDevice));
  s->connected = true;
  return EU_OK;
}

int eu_sym_destroy(eu_sym* s) {
  if (!s) return EU_OK;
  cudaSetDevice(s->c->g->device);
  cudaDeviceSynchronize();
  for (int r = 0; r < s->world; ++r)
    if (r != s->rank && s->peers.base[r]) cudaIpcCloseMemHandle(s->peers.base[r]);
  cudaFree(s->base); cudaFree(s->d_peers);
  cudaFree(s->d_sorted); cudaFree(s->d_src); cudaFree(s->d_counts); cudaFree(s->d_offs);
  cudaFree(s->d_rids); cudaFree(s->d_rw); cudaFree(s->d_rt); cudaFree(s->d_pad); cudaFree(s->d_seglo); cudaFree(s->d_boff); cudaFree(s->d_act);
  delete s;
  return EU_OK;
}

// device pointers of this rank's output arrays inside the symmetric region (valid until the next call of the same kind)
int eu_sym_outputs(eu_sym* s, int64_t** eng, int64_t** ids, float** w, int32_t** t, float** rows) {
  if (!s) { set_error("null sym"); return EU_ERR_INVALID; }
  if (eng) *eng = (int64_t*)(s->base + s->lay.off_eng);
  if (ids) *ids = (int64_t*)(s->base + s->lay.off_ids);
  if (w) *w = (float*)(s->base + s->lay.off_w);
  if (t) *t = (int32_t*)(s->base + s->lay.off_t);
  if (rows) *rows = (float*)(s->base + s->lay.off_rows);
  return EU_OK;
}

int eu_sym_error(eu_sym* s, int* err) {
  if (!s || !err) { set_error("eu_sym_error: bad argument"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(s->c->g->device));
  SymHeader h;
  EU_CUDA(cudaMemcpy(&h, s->base, sizeof(h), cudaMemcpyDeviceToHost));
  *err = h.error;
  return EU_OK;
}

static int sym_scratch(eu_sym* s, int64_t rows, int64_t slots, int64_t pad_rows = 0) {
  if (pad_rows > s->scratch_pad) {
    EU_CUDA(cudaStreamSynchronize(s->c->stream));
    cudaFree(s->d_pad);
    EU_CUDA(cudaMalloc(&s->d_pad, 8 * (size_t)pad_rows));
    if (!s->d_seglo) {
      EU_CUDA(cudaMalloc(&s->d_seglo, 4 * (size_t)kSymMaxRanks * 66));
      EU_CUDA(cudaMalloc(&s->d_boff, 4 * (size_t)(kSymMaxRanks + 1) * 64));
      EU_CUDA(cudaMalloc(&s->d_act, 4 * (size_t)64));
    }
    s->scratch_pad = pad_rows;
  }
  if (rows > s->scratch_rows) {
    EU_CUDA(cudaStreamSynchronize(s->c->stream));
    cudaFree(s->d_sorted); cudaFree(s->d_src);
    EU_CUDA(cudaMalloc(&s->d_sorted, 8 * (size_t)rows));
    EU_CUDA(cudaMalloc(&s->d_src, 4 * (size_t)rows));
    if (!s->d_counts) { EU_CUDA(cudaMalloc(&s->d_counts, 8 * 64)); EU_CUDA(cudaMalloc(&s->d_offs, 8 * 65)); }
    s->scratch_rows = rows;
  }
  if (slots > s->scratch_slots) {
    EU_CUDA(cudaStreamSynchronize(s->c->stream));
    cudaFree(s->d_rids); cudaFree(s->d_rw); cudaFree(s->d_rt);
    EU_CUDA(cudaMalloc(&s->d_rids, 8 * (size_t)slots));
    EU_CUDA(cudaMalloc(&s->d_rw, 4 * (size_t)slots));
    EU_CUDA(cudaMalloc(&s->d_rt, 4 * (size_t)slots));
    s->scratch_slots = slots;
  }
  return EU_OK;
}

// One sharded sampleNB hop over nb independent batches.  seeds: this rank's frontiers (device, i64[nb][rows]).  Batch g is
// sampled by every shard's engine g as ONE sampleNB call over the requests of rank 0..N-1 for that batch (own dedup scope,
// own RNG stream) -- nb = 1 is Euler's sharded sampleNB; nb > 1 runs nb of them per exchange so that the ~10 kernels and
// two NVLink round trips of an exchange are paid once per nb batches.  Results land in this rank's symmetric output arrays
// (eu_sym_outputs) as [nb][rows][count]: eng ids (the next frontier) always, TF-packed ids/w/t when want_packed.
int eu_sym_sample_hop_batched(eu_sym* s, const int64_t* seeds, int32_t nb, int64_t rows, const int32_t* etypes, int32_t K,
                              int32_t count, int64_t default_node, int32_t num_partitions, int32_t want_packed) {
  if (!s || !s->connected || nb < 1 || nb > 64 || rows < 0 || count < 0 || (rows > 0 && !seeds)) { set_error("eu_sym_sample_hop: bad argument / not connected"); return EU_ERR_INVALID; }
  eu_ctx* c = s->c;
  EU_CUDA(cudaSetDevice(c->g->device));
  // The inbox segment stride is the creation-time capacity (identical on every rank by construction); every rank must
  // issue the same exchange shape (nb x rows) -- the owners verify it (k_sym_wait_in, error 2) instead of trusting it.
  const SymLayout& L = s->lay;
  const int N = s->world;
  const int64_t total = (int64_t)nb * rows;
  if (total > L.cap || total * count > L.max_out || total >= ((int64_t)1 << 31)) { set_error("eu_sym_sample_hop: %d x %lld rows x %d exceed the symmetric region", nb, (long long)rows, count); return EU_ERR_INVALID; }
  if (nb > c->n_eng) { set_error("eu_sym_sample_hop: %d batches but the ctx has %d engines", nb, c->n_eng); return EU_ERR_INVALID; }
  const int64_t prow = (int64_t)N * total;   // padded sampleNB rows, all batches
  int rc = sym_scratch(s, std::max<int64_t>(total, 1), std::max<int64_t>(prow * count, 1), std::max<int64_t>(prow, 1));
  if (rc) return rc;
  cudaStream_t st = c->stream;
  rc = bucket_push(c, seeds, total, num_partitions, N, s->rank, false, s->d_counts, s->d_offs, s->d_peers, L, "k_bucket_push");
  if (rc) return rc;
  { EuProfScope ps(c, "k_sym_wait_in", total); k_sym_wait_in<<<1, 256, 0, st>>>(s->base, s->d_peers, L, N, nb, rows, (int)total, s->d_seglo, s->d_boff, s->d_act); }
  EU_LAUNCHED();
  // exact-RNG mode: the gather also enters the requests into the hop's dedup table (set 0; hop() wipes it), so the scratch is
  // reserved here, before the table is touched
  const bool will_sample = count > 0 && rows > 0;
  HashSlot* tabs = nullptr;
  int64_t tab_cap = 0;
  if (will_sample && c->rng == EU_RNG_MINSTD) {
    rc = ctx_reserve(c, hop_scratch_rows(nb, (int64_t)N * rows), hop_table_slots(nb, (int64_t)N * rows));
    if (rc) return rc;
    tabs = c->d_dedup;
    tab_cap = hop_table_cap((int64_t)N * rows);
  }
  { EuProfScope ps(c, "k_sym_gather_pad", prow); k_sym_gather_pad<<<sym_grid(total), 256, 0, st>>>(s->base, L, N, nb, rows, s->d_seglo, s->d_boff, s->d_pad, tabs, tab_cap); }
  EU_LAUNCHED();
  // (Tried and dropped: k_prepare / k_sample writing their results straight into the requesters' arrays.  The sampler's 8-byte
  // scattered NVLink stores stalled it -- 37 -> 109 us per step at N=2 -- where this reply pass copies coalesced rows.)
  if (will_sample) {
    rc = hop(c, s->d_pad, (int64_t)N * rows, etypes, K, count, /*default_node=*/0, nullptr, s->d_rids, s->d_rw, s->d_rt, 0, /*pre_inserted=*/tabs != nullptr, false, nb, s->d_act);
    if (rc) return rc;
  }
  { EuProfScope ps(c, "k_sym_reply_sample", prow);
    k_sym_reply_sample<<<reply_grid(prow * count), 256, 0, st>>>(s->d_peers, L, s->rank, N, nb, rows, s->d_seglo, s->d_boff, count, default_node,
                                                               (const long long*)s->d_rids, s->d_rw, s->d_rt, want_packed != 0); }
  EU_LAUNCHED();
  { EuProfScope ps(c, "k_sym_wait", total); k_sym_wait<<<1, 32, 0, st>>>(s->base, s->d_peers, L, N); }
  EU_LAUNCHED();
  return EU_OK;
}

int eu_sym_sample_hop(eu_sym* s, const int64_t* seeds, int64_t rows, const int32_t* etypes, int32_t K, int32_t count,
                      int64_t default_node, int32_t num_partitions, int32_t want_packed) {
  return eu_sym_sample_hop_batched(s, seeds, 1, rows, etypes, K, count, default_node, num_partitions, want_packed);
}

// Sharded dense feature fetch: rows land in this rank's symmetric `rows` output, [rows, dim], request order.
int eu_sym_get_dense_feature(eu_sym* s, const int64_t* ids, int64_t rows, int32_t fid, int32_t dim, int32_t num_partitions) {
  if (!s || !s->connected || rows < 0 || dim <= 0 || (rows > 0 && !ids)) { set_error("eu_sym_get_dense_feature: bad argument / not connected"); return EU_ERR_INVALID; }
  eu_ctx* c = s->c;
  EU_CUDA(cudaSetDevice(c->g->device));
  const SymLayout& L = s->lay;
  const DevGraph& d = c->g->d;
  const int N = s->world;
  if (d.feat_dtype != EU_FEAT_F32) { set_error("eu_sym_get_dense_feature: the sharded feature paths read f32 tables only"); return EU_ERR_UNSUPPORTED; }
  if (d.feat_place != EU_FEAT_DEVICE) { set_error("eu_sym_get_dense_feature: the sharded feature paths read tables held in HBM only"); return EU_ERR_UNSUPPORTED; }
  if (rows > L.cap || rows > L.max_rows_f || dim > L.max_dim) { set_error("eu_sym_get_dense_feature: request exceeds the symmetric region"); return EU_ERR_INVALID; }
  const bool have = fid >= 0 && fid < d.n_slots;
  const int32_t soff = have ? d.slot_off[fid] : 0, sdim = have ? d.slot_dim[fid] : 0;
  if ((dim & 3) || (soff & 3) || (sdim & 3) || (d.feat_dim & 3)) { set_error("eu_sym_get_dense_feature: widths must be multiples of 4 floats"); return EU_ERR_UNSUPPORTED; }
  int rc = sym_scratch(s, std::max<int64_t>(rows, 1), 1);
  if (rc) return rc;
  cudaStream_t st = c->stream;
  rc = bucket_push(c, ids, rows, num_partitions, N, s->rank, false, s->d_counts, s->d_offs, s->d_peers, L, "k_bucket_push(feat)");
  if (rc) return rc;
  { EuProfScope ps(c, "k_sym_wait_in(feat)", rows); k_sym_wait_in<<<1, 32, 0, st>>>(s->base, s->d_peers, L, N, 1, 0, -1, nullptr, nullptr, nullptr); }
  EU_LAUNCHED();
  int G = 1;
  while (G < 32 && G < dim / 4) G <<= 1;
  const int64_t prow = rows;   // on average a shard serves as many rows as it requests
  { EuProfScope ps(c, "k_sym_reply_feature", prow);
    k_sym_reply_feature<<<reply_grid(prow * G), 256, 0, st>>>(d, s->d_peers, L, s->rank, N, dim, soff, sdim, G); }
  EU_LAUNCHED();
  { EuProfScope ps(c, "k_sym_wait(feat)", rows); k_sym_wait<<<1, 32, 0, st>>>(s->base, s->d_peers, L, N); }
  EU_LAUNCHED();
  return EU_OK;
}

// Sharded fused SAGE mean over a fixed-fanout block: out[r,:] = mean_j feat(nbr_ids[r*count+j]) with features fetched
// from the owning shards and summed THERE (see k_sym_reply_sage).  Every rank calls it with the same rows/count/dim.
// Uses the symmetric `rows` region as N partial blocks (clobbers eu_sym_get_dense_feature's output).
int eu_sym_sage_mean(eu_sym* s, const int64_t* nbr_ids, int64_t rows, int32_t count, int32_t dim, int32_t num_partitions, float* out) {
  if (!s || !s->connected || rows < 0 || count < 1 || dim <= 0 || (rows > 0 && (!nbr_ids || !out))) { set_error("eu_sym_sage_mean: bad argument / not connected"); return EU_ERR_INVALID; }
  eu_ctx* c = s->c;
  EU_CUDA(cudaSetDevice(c->g->device));
  const SymLayout& L = s->lay;
  const DevGraph& d = c->g->d;
  const int N = s->world;
  const int64_t nid = rows * count;
  if (d.feat_dtype != EU_FEAT_F32) { set_error("eu_sym_sage_mean: the sharded feature paths read f32 tables only"); return EU_ERR_UNSUPPORTED; }
  if (d.feat_place != EU_FEAT_DEVICE) { set_error("eu_sym_sage_mean: the sharded feature paths read tables held in HBM only"); return EU_ERR_UNSUPPORTED; }
  if (nid > L.cap || nid >= ((int64_t)1 << 31) || (int64_t)N * rows * dim > L.max_rows_f * (int64_t)L.max_dim) {
    set_error("eu_sym_sage_mean: %lld x %d ids / %d partial blocks exceed the symmetric region", (long long)rows, count, N);
    return EU_ERR_INVALID;
  }
  int rc = sym_scratch(s, std::max<int64_t>(nid, 1), 1);
  if (rc) return rc;
  cudaStream_t st = c->stream;
  const bool fast = d.n < ((int64_t)1 << 31) && d.n_slots == 1 && dim == d.feat_dim && (dim == 128 || dim == 256);
  static int sage_r = 0;
  if (!sage_r) { const char* e = getenv("EU_SAGE_R"); sage_r = e && atoi(e) == 8 ? 8 : 32; }
  const int kSageR = sage_r;
  if ((rows / 8 + 1) * (int64_t)N > (L.max_rows_f / 8 + 1) * (int64_t)N) { set_error("eu_sym_sage_mean: presence bits exceed the symmetric region"); return EU_ERR_INVALID; }
  // the generic-width owners store every partial row: the requester marks them all present before its push goes out
  if (!fast) EU_CUDA(cudaMemsetAsync(s->base + L.off_flags, 0xFF, (size_t)(ceil_div(rows, kSageR) * N * 4), st));
  // ids that exist nowhere (0 / default fill) contribute nothing: they are dropped at the bucket, not shipped
  rc = bucket_push(c, nbr_ids, nid, num_partitions, N, s->rank, true, s->d_counts, s->d_offs, s->d_peers, L, "k_bucket_push(sage)");
  if (rc) return rc;
  { EuProfScope ps(c, "k_sym_wait_in(sage)", nid); k_sym_wait_in<<<1, 32, 0, st>>>(s->base, s->d_peers, L, N, 1, 0, (int)nid, nullptr, nullptr, nullptr); }
  EU_LAUNCHED();
  { EuProfScope ps(c, "k_sym_reply_sage", (int64_t)N * rows);
    const unsigned grid = sym_grid((int64_t)N * ceil_div(rows, kSageR) * 32);   // search-latency bound at large N: full occupancy
    if (fast && dim == 128) k_sym_reply_sage<1><<<grid, 256, 0, st>>>(d, s->d_peers, L, s->rank, N, rows, count, kSageR);
    else if (fast && dim == 256) k_sym_reply_sage<2><<<grid, 256, 0, st>>>(d, s->d_peers, L, s->rank, N, rows, count, kSageR);
    else k_sym_reply_sage_generic<<<sym_grid((int64_t)N * rows * 32), 256, 0, st>>>(d, s->d_peers, L, s->rank, N, rows, count, dim); }
  EU_LAUNCHED();
  { EuProfScope ps(c, "k_sym_wait(sage)", rows); k_sym_wait<<<1, 32, 0, st>>>(s->base, s->d_peers, L, N); }
  EU_LAUNCHED();
  if (rows > 0) {
    EuProfScope ps(c, "k_sym_sage_reduce", rows);
    const float* part = (const float*)(s->base + L.off_rows);
    const unsigned int* flags = (const unsigned int*)(s->base + L.off_flags);
    if ((dim & 3) == 0 && ((uintptr_t)out & 15) == 0)
      k_sym_sage_reduce<float4><<<sym_grid(rows * dim / 4), 256, 0, st>>>((const float4*)part, flags, N, rows, dim / 4, count, kSageR, (float4*)out);
    else
      k_sym_sage_reduce<float><<<sym_grid(rows * dim), 256, 0, st>>>(part, flags, N, rows, dim, count, kSageR, out);
    EU_LAUNCHED();
  }
  return EU_OK;
}

}  // extern "C"
