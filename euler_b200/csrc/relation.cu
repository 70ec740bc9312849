// RelationConv's typed mean aggregation, forward and backward, over the edge lists of RelationDataFlow blocks (f32 data,
// i32 indices).
//
// Reference semantics (file:line in the upstream alibaba/euler tree):
//   RelationConv.__call__ / apply_edge   tf_euler/python/convolution/relation_conv.py:53-70 (aggr = 'mean'), up to apply_node
//   scatter_mean                         tf_euler/python/euler_ops/mp_ops.py:65-69
//
// For W = matrix f32[R, D, F] and edge e = (dst_e, src_e) of relation rel_e:
//   out[i] = (sum over the edges e with dst_e = i of W[rel_e] . x_src[src_e]) / fl(cnt_i + 1e-7)
//
// Upstream runs one matvec per edge.  The transform is linear, so the edges are grouped by pair p = (target, relation) first:
//   S_p    = sum over the edges of p of x_src[src_e]                          (k_rel_chunk_sums, k_seg_combine)
//   out[i] = (sum over the pairs p of i of W[r_p] . S_p) / fl(cnt_i + 1e-7)   (k_rel_out)
// so the matvecs drop from E to P (the distinct pairs) and nothing of size E*D is written.  Fixed orders:
//   - S_p: the pair's edges in key order, cut into chunks of kSegChunk consecutive edges counted from the pair's first edge;
//     each chunk summed left to right, then the chunk sums added in chunk order.  The bits depend on the pair's own edge
//     sequence only, never on the launch configuration or on other pairs.
//   - out[i, d]: one __fmaf_rn chain over the pairs of i in key order and, within a pair, over f ascending; then one
//     __fdiv_rn by fl(fl(cnt_i) + 1e-7f), scatter_mean's divisor.  A target without edges gets exact zeros.
// Backward, with gm_i = g_i / fl(cnt_i + 1e-7):
//   gS_p              = W[r_p]^T . gm_{i(p)}                      (k_rel_gs: one __fmaf_rn chain over d ascending)
//   grad_x_src[j]     = sum over the edges e with src_e = j of gS_{pair(e)}
//                       (the stable order by source and k_gat_bwd_src, weight 1, the edge's pair as its row)
//   grad_matrix[r]    = sum over the pairs p with r_p = r of gm_{i(p)} (x) S_p
//                       (the pairs in stable relation order, chunks of kRelPairChunk pairs counted from the relation's first
//                       pair, each a __fmaf_rn chain; the chunk sums added in chunk order)
// Every sum runs in a fixed order: no atomics, the same bits on every run; unused sources and relations get exact zeros.
//
// Order: the (dst, rel) keys of RelationDataFlow blocks arrive non-decreasing (the full hop lists a node's edges type by type
// in list order); then the edges are walked as given.  Otherwise a stable radix sort on the composite key dst * R + rel orders
// them, so the result equals, bit for bit, the call on the stably sorted edge list.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "segment.cuh"

namespace eu {

constexpr int kRelPairChunk = 256;   // pairs per chunk of a relation's grad_matrix sum
constexpr int kRelUnroll = 8;        // source rows in flight per lane in the chunk sums

// The pairs of target i: [*pb, *pe) (pair_dst is non-decreasing), and scatter_mean's divisor fl(fl(cnt_i) + 1e-7f).
__device__ __forceinline__ float rel_target(const int32_t* __restrict__ pair_dst, const int32_t* __restrict__ pair_start, int64_t P,
                                            int64_t i, int64_t* pb, int64_t* pe) {
  *pb = key_lower_bound(pair_dst, P, i);
  *pe = key_lower_bound(pair_dst, P, i + 1);
  const int64_t cnt = (int64_t)__ldg(pair_start + *pe) - __ldg(pair_start + *pb);
  return __fadd_rn((float)cnt, 1e-7f);
}

// head[k] = 1 where position k starts a pair (k = 0, or its key differs from position k - 1's).  The keys are skey (the
// sorted composite keys) when given; otherwise dst * R + rel of the edges as given, and then flags[0] = 1 if a key decreases
// and flags[1] = 1 if a relation lies outside [0, R).
__global__ void k_rel_heads(const int32_t* __restrict__ dst, const int32_t* __restrict__ rel,
                            const unsigned long long* __restrict__ skey, int64_t E, int64_t R, int32_t* __restrict__ head,
                            int* __restrict__ flags) {
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < E; k += (int64_t)gridDim.x * blockDim.x) {
    if (skey) {
      head[k] = k == 0 || __ldg(skey + k) != __ldg(skey + k - 1);
      continue;
    }
    const int32_t r = __ldg(rel + k);
    if (r < 0 || r >= R) flags[1] = 1;
    const int64_t key = (int64_t)__ldg(dst + k) * R + r;
    int h = 1;
    if (k > 0) {
      const int64_t prev = (int64_t)__ldg(dst + k - 1) * R + __ldg(rel + k - 1);
      if (prev > key) flags[0] = 1;
      h = prev != key;
    }
    head[k] = h;
  }
}

// the composite sort keys dst * R + rel and the identity permutation
__global__ void k_rel_keys(const int32_t* __restrict__ dst, const int32_t* __restrict__ rel, int64_t E, int64_t R,
                           unsigned long long* __restrict__ key, int32_t* __restrict__ iota) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < E; e += (int64_t)gridDim.x * blockDim.x) {
    key[e] = (unsigned long long)((int64_t)__ldg(dst + e) * R + __ldg(rel + e));
    iota[e] = (int32_t)e;
  }
}

// From pid (the inclusive scan of head: position k belongs to pair pid[k] - 1): each pair's first position, target and
// relation, pair_start[P] = E, and (when given) the pair of every edge.
__global__ void k_rel_pairs(const int32_t* __restrict__ head, const int32_t* __restrict__ pid, const int32_t* __restrict__ perm,
                            const int32_t* __restrict__ dst, const int32_t* __restrict__ rel, int64_t E,
                            int32_t* __restrict__ pair_start, int32_t* __restrict__ pair_dst, int32_t* __restrict__ pair_rel,
                            int32_t* __restrict__ pair_of_edge) {
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < E; k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t ed = edge_at(perm, k);
    const int32_t p = __ldg(pid + k) - 1;
    if (__ldg(head + k)) {
      pair_start[p] = (int32_t)k;
      pair_dst[p] = __ldg(dst + ed);
      pair_rel[p] = __ldg(rel + ed);
    }
    if (pair_of_edge) pair_of_edge[ed] = p;
    if (k == E - 1) pair_start[p + 1] = (int32_t)E;
  }
}

__global__ void k_rel_fill(float* __restrict__ v, int64_t n, float x) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) v[i] = x;
}

// G lanes per chunk c (lanes over the F columns, 4 per lane with float4).  Chunk c - chunk_off[p] of pair p covers the
// positions [pair_start[p] + (c - chunk_off[p]) * kSegChunk, ...) up to kSegChunk of them, summed left to right from +0.  A
// pair of one chunk writes S[p]; the chunks of a longer pair write partial[c] for k_seg_combine.
template <bool VEC>
__global__ void __launch_bounds__(256) k_rel_chunk_sums(const float* __restrict__ x_src, const int32_t* __restrict__ src,
                                                        const int32_t* __restrict__ perm, const int32_t* __restrict__ pair_start,
                                                        const int32_t* __restrict__ chunk_off, int64_t P, int64_t slots, int F,
                                                        int G, float* __restrict__ S, float* __restrict__ partial) {
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t c = tid >> (31 - __clz(G));
  const int sub = (int)(tid & (G - 1));
  if (c >= slots || c >= __ldg(chunk_off + P)) return;
  const int64_t p = key_upper_bound(chunk_off, P + 1, c) - 1;
  const int64_t c0 = __ldg(chunk_off + p), nch = __ldg(chunk_off + p + 1) - c0;
  const int64_t b = __ldg(pair_start + p) + (c - c0) * kSegChunk;
  const int64_t e = min(b + kSegChunk, (int64_t)__ldg(pair_start + p + 1));
  float* o = nch == 1 ? S + p * F : partial + c * F;
  if (VEC) {
    for (int d = sub * 4; d < F; d += G * 4) {
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int64_t k0 = b; k0 < e; k0 += kRelUnroll) {
        float4 x[kRelUnroll];
#pragma unroll
        for (int q = 0; q < kRelUnroll; ++q)
          if (k0 + q < e) x[q] = __ldg(reinterpret_cast<const float4*>(x_src + (int64_t)__ldg(src + edge_at(perm, k0 + q)) * F + d));
#pragma unroll
        for (int q = 0; q < kRelUnroll; ++q) {
          if (k0 + q < e) {
            acc.x = __fadd_rn(acc.x, x[q].x); acc.y = __fadd_rn(acc.y, x[q].y);
            acc.z = __fadd_rn(acc.z, x[q].z); acc.w = __fadd_rn(acc.w, x[q].w);
          }
        }
      }
      *reinterpret_cast<float4*>(o + d) = acc;
    }
  } else {
    for (int d = sub; d < F; d += G) {
      float acc = 0.f;
      for (int64_t k0 = b; k0 < e; k0 += kRelUnroll) {
        float x[kRelUnroll];
#pragma unroll
        for (int q = 0; q < kRelUnroll; ++q)
          if (k0 + q < e) x[q] = __ldg(x_src + (int64_t)__ldg(src + edge_at(perm, k0 + q)) * F + d);
#pragma unroll
        for (int q = 0; q < kRelUnroll; ++q)
          if (k0 + q < e) acc = __fadd_rn(acc, x[q]);
      }
      o[d] = acc;
    }
  }
}

// Wt[r, f, d] = W[r, d, f]: k_rel_out's lanes (over d) then read consecutive words
__global__ void k_rel_transpose(const float* __restrict__ W, int64_t R, int D, int F, float* __restrict__ Wt) {
  const int64_t n = R * D * F;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / ((int64_t)D * F), rem = t - r * D * F, f = rem / D, d = rem - f * D;
    Wt[t] = __ldg(W + (r * D + d) * F + f);
  }
}

// out[i, d] = (sum over the pairs p of i, in key order, of sum_f W[r_p, d, f] * S[p, f]) / fl(cnt_i + 1e-7): one __fmaf_rn
// chain over (p, f); one thread per (i, d).  Wt is W transposed (k_rel_transpose).
__global__ void __launch_bounds__(256) k_rel_out(const float* __restrict__ Wt, const float* __restrict__ S,
                                                 const int32_t* __restrict__ pair_start, const int32_t* __restrict__ pair_dst,
                                                 const int32_t* __restrict__ pair_rel, int64_t P, int64_t n_dst, int D, int F,
                                                 float* __restrict__ out) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= n_dst * D) return;
  const int64_t i = t / D, d = t - i * D;
  int64_t pb, pe;
  const float den = rel_target(pair_dst, pair_start, P, i, &pb, &pe);
  float acc = 0.f;
  for (int64_t p = pb; p < pe; ++p) {
    const float* w = Wt + (int64_t)__ldg(pair_rel + p) * F * D + d;
    const float* s = S + p * F;
    for (int f = 0; f < F; ++f) acc = __fmaf_rn(__ldg(w + (int64_t)f * D), __ldg(s + f), acc);
  }
  out[t] = __fdiv_rn(acc, den);
}

// gm[i, d] = g[i, d] / fl(cnt_i + 1e-7) (one __fdiv_rn); one thread per (i, d)
__global__ void k_rel_gm(const float* __restrict__ g, const int32_t* __restrict__ pair_start, const int32_t* __restrict__ pair_dst,
                         int64_t P, int64_t n_dst, int D, float* __restrict__ gm) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= n_dst * D) return;
  int64_t pb, pe;
  const float den = rel_target(pair_dst, pair_start, P, t / D, &pb, &pe);
  gm[t] = __fdiv_rn(__ldg(g + t), den);
}

// gS[p, f] = sum_d W[r_p, d, f] * gm[i(p), d]: one __fmaf_rn chain over d ascending; one thread per (p, f)
__global__ void __launch_bounds__(256) k_rel_gs(const float* __restrict__ W, const float* __restrict__ gm,
                                                const int32_t* __restrict__ pair_dst, const int32_t* __restrict__ pair_rel, int64_t P,
                                                int D, int F, float* __restrict__ gS) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= P * F) return;
  const int64_t p = t / F, f = t - p * F;
  const float* w = W + (int64_t)__ldg(pair_rel + p) * D * F + f;
  const float* g = gm + (int64_t)__ldg(pair_dst + p) * D;
  float acc = 0.f;
  for (int d = 0; d < D; ++d) acc = __fmaf_rn(__ldg(w + (int64_t)d * F), __ldg(g + d), acc);
  gS[t] = acc;
}

// One block row per chunk c of the relation-sorted pairs: chunk c - roff[r] of relation r covers its positions
// [rstart[r] + (c - roff[r]) * kRelPairChunk, ...) up to kRelPairChunk of them.  partial[c, d, f] = sum over those pairs, in
// order, of gm[i(p), d] * S[p, f] (one __fmaf_rn chain); threads over the D*F elements.
__global__ void __launch_bounds__(256) k_rel_gw_partials(const float* __restrict__ gm, const float* __restrict__ S,
                                                         const int32_t* __restrict__ pair_dst, const int32_t* __restrict__ rperm,
                                                         const int32_t* __restrict__ rstart, const int32_t* __restrict__ roff,
                                                         int64_t R, int D, int F, float* __restrict__ partial) {
  const int64_t c = blockIdx.x;
  if (c >= __ldg(roff + R)) return;   // block-uniform
  const int64_t r = key_upper_bound(roff, R + 1, c) - 1;
  const int64_t b = __ldg(rstart + r) + (c - __ldg(roff + r)) * kRelPairChunk;
  const int64_t e = min(b + kRelPairChunk, (int64_t)__ldg(rstart + r + 1));
  const int64_t DF = (int64_t)D * F;
  for (int64_t el = blockIdx.y * (int64_t)blockDim.x + threadIdx.x; el < DF; el += (int64_t)gridDim.y * blockDim.x) {
    const int64_t d = el / F, f = el - d * F;
    float acc = 0.f;
    for (int64_t q = b; q < e; ++q) {
      const int64_t p = __ldg(rperm + q);
      acc = __fmaf_rn(__ldg(gm + (int64_t)__ldg(pair_dst + p) * D + d), __ldg(S + p * F + f), acc);
    }
    partial[c * DF + el] = acc;
  }
}

// grad_matrix[r, el] = the chunk sums of relation r added in chunk order from +0 (zero for an unused relation); one thread
// per (r, el)
__global__ void k_rel_gw_combine(const float* __restrict__ partial, const int32_t* __restrict__ roff, int64_t R, int64_t DF,
                                 float* __restrict__ grad_matrix) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= R * DF) return;
  const int64_t r = t / DF, el = t - r * DF;
  float acc = 0.f;
  for (int64_t c = __ldg(roff + r), c1 = __ldg(roff + r + 1); c < c1; ++c) acc = __fadd_rn(acc, __ldg(partial + c * DF + el));
  grad_matrix[t] = acc;
}

// The pairs of one call, in the ctx scratch.  Layout (offsets fixed once `sorted` is known, so a call that does not grow the
// scratch keeps what it has computed):
//   flags | head [E] | pid [E] | scan temp | [sort: keys in, keys out (u64 [E] each), iota, perm ([E] each), cub temp]
//   | pair_start [P+1] | pair_dst [P] | pair_rel [P] | nc [P+1] | chunk_off [P+1] | S [P, F] | chunk sums [P + E/kSegChunk, F]
//   | the backward's part (extra bytes)
struct RelPairs {
  bool sorted = true;
  int64_t P = 0, slots = 0;
  size_t o_head = 0, o_pid = 0, o_scan = 0, scan_bytes = 0, o_sort = 0, sort_tmp = 0, o_ps = 0, o_pd = 0, o_pr = 0, o_nc = 0,
         o_coff = 0, o_S = 0, o_part = 0, o_extra = 0, total = 0;
  const int32_t* perm = nullptr;
  int32_t *pair_start = nullptr, *pair_dst = nullptr, *pair_rel = nullptr, *chunk_off = nullptr;
  float* S = nullptr;
};

static void rel_layout(RelPairs* L, int64_t E, int64_t P, int F, size_t extra) {
  L->P = P;
  L->slots = P + E / kSegChunk;   // >= the chunks: sum over pairs of ceil(len / K) <= P + E / K
  L->o_head = 256;
  L->o_pid = L->o_head + a256(4 * (size_t)E);
  L->o_scan = L->o_pid + a256(4 * (size_t)E);
  L->o_sort = L->o_scan + a256(L->scan_bytes);
  L->o_ps = L->o_sort + (L->sorted ? 0 : 2 * a256(8 * (size_t)E) + 2 * a256(4 * (size_t)E) + a256(L->sort_tmp));
  L->o_pd = L->o_ps + a256(4 * (size_t)(P + 1));
  L->o_pr = L->o_pd + a256(4 * (size_t)P);
  L->o_nc = L->o_pr + a256(4 * (size_t)P);
  L->o_coff = L->o_nc + a256(4 * (size_t)(P + 1));
  L->o_S = L->o_coff + a256(4 * (size_t)(P + 1));
  L->o_part = L->o_S + a256(4 * (size_t)P * F);
  L->o_extra = L->o_part + a256(4 * (size_t)L->slots * F);
  L->total = L->o_extra + extra;
}

// Sort (when unsorted) and mark the pair heads, then scan them into pid, in the scratch laid out by L
static int rel_heads(eu_ctx* c, const RelPairs& L, const int32_t* rel, const int32_t* dst, int64_t E, int64_t n_dst, int64_t R) {
  cudaStream_t s = c->stream;
  char* m = (char*)c->d_misc;
  int32_t* head = (int32_t*)(m + L.o_head);
  int32_t* pid = (int32_t*)(m + L.o_pid);
  const unsigned long long* skey = nullptr;
  if (!L.sorted) {
    EuProfScope ps(c, "rel_sort", E);
    unsigned long long* kin = (unsigned long long*)(m + L.o_sort);
    unsigned long long* kout = (unsigned long long*)(m + L.o_sort + a256(8 * (size_t)E));
    int32_t* iota = (int32_t*)(m + L.o_sort + 2 * a256(8 * (size_t)E));
    int32_t* perm = (int32_t*)(m + L.o_sort + 2 * a256(8 * (size_t)E) + a256(4 * (size_t)E));
    void* tmp = m + L.o_sort + 2 * a256(8 * (size_t)E) + 2 * a256(4 * (size_t)E);
    k_rel_keys<<<stride_grid(E), 256, 0, s>>>(dst, rel, E, R, kin, iota);
    EU_LAUNCHED();
    size_t t = L.sort_tmp;
    EU_CUDA(cub::DeviceRadixSort::SortPairs(tmp, t, kin, kout, iota, perm, (int)E, 0,
                                            radix_bits((unsigned long long)n_dst * (unsigned long long)R), s));
    EU_LAUNCHED();
    skey = kout;
  }
  EuProfScope ps(c, "rel_heads", E);
  k_rel_heads<<<stride_grid(E), 256, 0, s>>>(dst, rel, skey, E, R, head, (int*)m);
  EU_LAUNCHED();
  size_t t = L.scan_bytes;
  EU_CUDA(cub::DeviceScan::InclusiveSum(m + L.o_scan, t, head, pid, (int)E, s));
  EU_LAUNCHED();
  return EU_OK;
}

// Everything the forward and backward passes share, for E > 0: check the relations, order the edges by (dst, rel) when they
// are not ordered yet, find the pairs and their row sums S.  `extra` = the bytes the caller needs after them, a function of P.
// Synchronises once when the keys arrive non-decreasing (the flags and P), twice otherwise (the flags, then P after the sort).
template <class Extra>
static int rel_prepare(eu_ctx* c, const float* x_src, const int32_t* rel, const int32_t* dst, const int32_t* src, int64_t E,
                       int64_t n_dst, int64_t R, int F, const char* who, Extra extra, RelPairs* L) {
  cudaStream_t s = c->stream;
  size_t a = 0, b = 0;
  EU_CUDA(cub::DeviceScan::InclusiveSum(nullptr, a, (const int32_t*)nullptr, (int32_t*)nullptr, (int)E, s));
  EU_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, b, (const int32_t*)nullptr, (int32_t*)nullptr, (int)(std::max(E, R) + 1), s));
  L->scan_bytes = std::max(a, b);
  L->sorted = true;
  rel_layout(L, E, 0, F, 0);
  int rc = ctx_misc(c, (int64_t)L->total);
  if (rc) return rc;
  EU_CUDA(cudaMemsetAsync(c->d_misc, 0, 2 * sizeof(int), s));
  if ((rc = rel_heads(c, *L, rel, dst, E, n_dst, R))) return rc;
  int flags[2] = {0, 0}, P = 0;
  EU_CUDA(cudaMemcpyAsync(flags, c->d_misc, sizeof(flags), cudaMemcpyDeviceToHost, s));
  EU_CUDA(cudaMemcpyAsync(&P, (char*)c->d_misc + L->o_pid + 4 * (size_t)(E - 1), sizeof(int), cudaMemcpyDeviceToHost, s));
  EU_CUDA(cudaStreamSynchronize(s));
  if (flags[1]) {
    set_error("%s: a relation lies outside [0, num_relations = %lld)", who, (long long)R);
    return EU_ERR_INVALID;
  }
  if (flags[0]) {   // unsorted: the sort's scratch, the sort, the heads again and P (a second synchronisation)
    L->sorted = false;
    EU_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, L->sort_tmp, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                            (const int32_t*)nullptr, (int32_t*)nullptr, (int)E, 0,
                                            radix_bits((unsigned long long)n_dst * (unsigned long long)R), s));
    rel_layout(L, E, 0, F, 0);
    if ((rc = ctx_misc(c, (int64_t)L->total))) return rc;
    if ((rc = rel_heads(c, *L, rel, dst, E, n_dst, R))) return rc;
    EU_CUDA(cudaMemcpyAsync(&P, (char*)c->d_misc + L->o_pid + 4 * (size_t)(E - 1), sizeof(int), cudaMemcpyDeviceToHost, s));
    EU_CUDA(cudaStreamSynchronize(s));
  }
  rel_layout(L, E, P, F, extra((int64_t)P));
  if ((int64_t)L->total > c->misc_bytes) {   // the growth reallocates: order and mark the pairs again (no read-back needed)
    if ((rc = ctx_misc(c, (int64_t)L->total))) return rc;
    if ((rc = rel_heads(c, *L, rel, dst, E, n_dst, R))) return rc;
  }
  char* m = (char*)c->d_misc;
  L->perm = L->sorted ? nullptr : (const int32_t*)(m + L->o_sort + 2 * a256(8 * (size_t)E) + a256(4 * (size_t)E));
  L->pair_start = (int32_t*)(m + L->o_ps);
  L->pair_dst = (int32_t*)(m + L->o_pd);
  L->pair_rel = (int32_t*)(m + L->o_pr);
  L->chunk_off = (int32_t*)(m + L->o_coff);
  L->S = (float*)(m + L->o_S);
  int32_t* nc = (int32_t*)(m + L->o_nc);
  {
    EuProfScope ps(c, "rel_pairs", E);
    k_rel_pairs<<<stride_grid(E), 256, 0, s>>>((const int32_t*)(m + L->o_head), (const int32_t*)(m + L->o_pid), L->perm, dst, rel, E,
                                            L->pair_start, L->pair_dst, L->pair_rel, nullptr);
    EU_LAUNCHED();
    if ((rc = seg_chunk_offsets(c, L->pair_start, P, kSegChunk, nc, m + L->o_scan, L->scan_bytes, L->chunk_off))) return rc;
  }
  {
    const bool vec = F % 4 == 0 && aligned16(x_src);
    const int G = group_lanes(vec ? F / 4 : F);
    float* part = (float*)(m + L->o_part);
    EuProfScope ps(c, "rel_pair_sums", E);
    const unsigned blocks = (unsigned)ceil_div(L->slots * G, 256);
    if (vec) k_rel_chunk_sums<true><<<blocks, 256, 0, s>>>(x_src, src, L->perm, L->pair_start, L->chunk_off, P, L->slots, F, G, L->S, part);
    else k_rel_chunk_sums<false><<<blocks, 256, 0, s>>>(x_src, src, L->perm, L->pair_start, L->chunk_off, P, L->slots, F, G, L->S, part);
    EU_LAUNCHED();
    k_seg_combine<<<(unsigned)ceil_div(P * F, 256), 256, 0, s>>>(L->chunk_off, part, P, F, L->S);
    EU_LAUNCHED();
  }
  return EU_OK;
}

static int rel_check_args(const char* who, int64_t E, int64_t n_dst, int64_t n_src, int64_t R, int64_t D, int64_t F) {
  if (E >= ((int64_t)1 << 31) || n_dst >= ((int64_t)1 << 31) || n_src >= ((int64_t)1 << 31) || R * D * F >= ((int64_t)1 << 31)) {
    set_error("%s: 2^31 or more edges, rows or matrix entries are not supported", who);
    return EU_ERR_UNSUPPORTED;
  }
  return EU_OK;
}

}  // namespace eu

using namespace eu;

extern "C" {

int eu_relation_aggregate(eu_ctx* c, const float* x_src, const float* matrix, const int32_t* rel, const int32_t* dst,
                          const int32_t* src, int64_t E, int64_t n_dst, int64_t n_src, int32_t num_relations, int32_t dim,
                          int32_t fea_dim, float* out) {
  const char* who = "eu_relation_aggregate";
  if (!c || num_relations < 1 || dim < 1 || fea_dim < 1 || E < 0 || n_dst < 0 || n_src < 0 || (E > 0 && (n_dst == 0 || n_src == 0)) ||
      (E > 0 && (!x_src || !matrix || !rel || !dst || !src)) || (n_dst > 0 && !out)) {
    set_error("%s: bad argument", who);
    return EU_ERR_INVALID;
  }
  int rc = rel_check_args(who, E, n_dst, n_src, num_relations, dim, fea_dim);
  if (rc) return rc;
  EU_CUDA(cudaSetDevice(c->g->device));
  if (n_dst == 0) return EU_OK;
  cudaStream_t s = c->stream;
  const int64_t R = num_relations, D = dim, F = fea_dim;
  if (E == 0) {                                        // no edge: every target's mean is 0 / 1e-7 = 0
    EU_CUDA(cudaMemsetAsync(out, 0, 4 * (size_t)(n_dst * D), s));
    return EU_OK;
  }
  RelPairs L;   // after the pairs: the transposed matrix [R, F, D]
  if ((rc = rel_prepare(c, x_src, rel, dst, src, E, n_dst, R, (int)F, who, [&](int64_t) { return a256(4 * (size_t)(R * D * F)); }, &L)))
    return rc;
  float* Wt = (float*)((char*)c->d_misc + L.o_extra);
  EuProfScope ps(c, "rel_out", E);
  k_rel_transpose<<<stride_grid(R * D * F), 256, 0, s>>>(matrix, R, (int)D, (int)F, Wt);
  EU_LAUNCHED();
  k_rel_out<<<(unsigned)ceil_div(n_dst * D, 256), 256, 0, s>>>(Wt, L.S, L.pair_start, L.pair_dst, L.pair_rel, L.P, n_dst, (int)D,
                                                               (int)F, out);
  EU_LAUNCHED();
  return EU_OK;
}

int eu_relation_aggregate_backward(eu_ctx* c, const float* grad_out, const float* x_src, const float* matrix, const int32_t* rel,
                                   const int32_t* dst, const int32_t* src, int64_t E, int64_t n_dst, int64_t n_src,
                                   int32_t num_relations, int32_t dim, int32_t fea_dim, float* grad_x_src, float* grad_matrix) {
  const char* who = "eu_relation_aggregate_backward";
  if (!c || num_relations < 1 || dim < 1 || fea_dim < 1 || E < 0 || n_dst < 0 || n_src < 0 || (E > 0 && (n_dst == 0 || n_src == 0)) ||
      (E > 0 && (!grad_out || !x_src || !matrix || !rel || !dst || !src)) || (n_src > 0 && !grad_x_src) || !grad_matrix) {
    set_error("%s: bad argument", who);
    return EU_ERR_INVALID;
  }
  int rc = rel_check_args(who, E, n_dst, n_src, num_relations, dim, fea_dim);
  if (rc) return rc;
  EU_CUDA(cudaSetDevice(c->g->device));
  cudaStream_t s = c->stream;
  const int64_t R = num_relations, D = dim, F = fea_dim, DF = D * F;
  if (E == 0) {                                        // no edge: every gradient is zero
    if (n_src > 0) EU_CUDA(cudaMemsetAsync(grad_x_src, 0, 4 * (size_t)(n_src * F), s));
    EU_CUDA(cudaMemsetAsync(grad_matrix, 0, 4 * (size_t)(R * DF), s));
    return EU_OK;
  }
  // after the pairs: gm [n_dst, D] | gS [P, F] | ones [E] | pair of each edge [E] | the src order | the relation order of the
  // pairs | rstart, rnc, roff [R+1] each | grad_matrix chunk sums [min(R, P) + P / kRelPairChunk + 1, D, F]
  auto rslots = [&](int64_t P) { return std::min(R, P) + P / kRelPairChunk + 1; };
  size_t o_gm = 0, o_gs = 0, o_ones = 0, o_poe = 0, o_sord = 0, o_rord = 0, o_rst = 0, o_rnc = 0, o_roff = 0, o_gw = 0;
  auto extra = [&](int64_t P) {
    o_gm = 0;
    o_gs = o_gm + a256(4 * (size_t)(n_dst * D));
    o_ones = o_gs + a256(4 * (size_t)P * F);
    o_poe = o_ones + a256(4 * (size_t)E);
    o_sord = o_poe + a256(4 * (size_t)E);
    o_rord = o_sord + order_bytes(E, n_src);
    o_rst = o_rord + order_bytes(P, R);
    o_rnc = o_rst + a256(4 * (size_t)(R + 1));
    o_roff = o_rnc + a256(4 * (size_t)(R + 1));
    o_gw = o_roff + a256(4 * (size_t)(R + 1));
    return o_gw + a256(4 * (size_t)rslots(P) * DF);
  };
  RelPairs L;
  if ((rc = rel_prepare(c, x_src, rel, dst, src, E, n_dst, R, (int)F, who, extra, &L))) return rc;
  const int64_t P = L.P;
  char* x = (char*)c->d_misc + L.o_extra;
  float* gm = (float*)(x + o_gm);
  float* gS = (float*)(x + o_gs);
  float* ones = (float*)(x + o_ones);
  int32_t* poe = (int32_t*)(x + o_poe);
  int32_t* rst = (int32_t*)(x + o_rst);
  int32_t* rnc = (int32_t*)(x + o_rnc);
  int32_t* roff = (int32_t*)(x + o_roff);
  float* gw = (float*)(x + o_gw);
  char* m = (char*)c->d_misc;
  {
    EuProfScope ps(c, "rel_bwd_gs", P);
    k_rel_gm<<<(unsigned)ceil_div(n_dst * D, 256), 256, 0, s>>>(grad_out, L.pair_start, L.pair_dst, P, n_dst, (int)D, gm);
    EU_LAUNCHED();
    k_rel_gs<<<(unsigned)ceil_div(P * F, 256), 256, 0, s>>>(matrix, gm, L.pair_dst, L.pair_rel, P, (int)D, (int)F, gS);
    EU_LAUNCHED();
  }
  {
    EuProfScope ps(c, "rel_bwd_src", E);
    k_rel_pairs<<<stride_grid(E), 256, 0, s>>>((const int32_t*)(m + L.o_head), (const int32_t*)(m + L.o_pid), L.perm, dst, rel, E,
                                            L.pair_start, L.pair_dst, L.pair_rel, poe);
    EU_LAUNCHED();
    k_rel_fill<<<stride_grid(E), 256, 0, s>>>(ones, E, 1.f);
    EU_LAUNCHED();
    EdgeOrder sord;
    if ((rc = order_by(c, src, E, n_src, x + o_sord, &sord))) return rc;
    if ((rc = segmented_row_sum(c, gS, ones, sord, poe, E, n_src, (int)F, grad_x_src))) return rc;
  }
  {
    EuProfScope ps(c, "rel_bwd_matrix", P);
    EdgeOrder rord;
    if ((rc = order_by(c, L.pair_rel, P, R, x + o_rord, &rord))) return rc;
    k_seg_starts<<<stride_grid(R + 1), 256, 0, s>>>(rord.key, P, R, rst);
    EU_LAUNCHED();
    if ((rc = seg_chunk_offsets(c, rst, R, kRelPairChunk, rnc, m + L.o_scan, L.scan_bytes, roff))) return rc;
    const dim3 grid((unsigned)rslots(P), (unsigned)std::min<int64_t>(ceil_div(DF, 256), 65535));
    k_rel_gw_partials<<<grid, 256, 0, s>>>(gm, L.S, L.pair_dst, rord.perm, rst, roff, R, (int)D, (int)F, gw);
    EU_LAUNCHED();
    k_rel_gw_combine<<<(unsigned)ceil_div(R * DF, 256), 256, 0, s>>>(gw, roff, R, DF, grad_matrix);
    EU_LAUNCHED();
  }
  return EU_OK;
}

}  // extern "C"
