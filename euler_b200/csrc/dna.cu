// DNAConv's attention aggregation, forward and backward, over the edge lists of dataflow blocks (f32 data, i32 indices).
//
// Reference semantics (file:line in the upstream alibaba/euler tree):
//   DNAConv.__call__ / apply_edge / multi_head / attention   tf_euler/python/convolution/dna_conv.py:115-170 (aggr = 'mean')
//   restricted_softmax                                       dna_conv.py:72-80
//   scatter_mean                                             tf_euler/python/euler_ops/mp_ops.py:65-69
//
// H heads of width C, dim = H * C; q f32[n_dst, dim] (lin_q of the targets), k and v f32[n_src, dim] (lin_k, lin_v of the
// sources), n0 f32[n_dst] and n1 f32[n_src] (gcn_norm).  For edge e = (i = dst_e, j = src_e):
//   s[e,h,h']  = <q_i[h], k_j[h']> / sqrt(C)                       (every query head against every key head)
//   m[e,h]     = max(0, max_h' s[e,h,h'])
//   a[e,h,h']  = exp(s - m) / (sum_h'' exp(s[e,h,h''] - m) + exp(-m))
//   msg[e,h,:] = fl(n0_i * n1_j) * sum_h' a[e,h,h'] * v_j[h']
//   out_i      = sum over the edges of i of msg_e / fl(fl(cnt_i) + 1e-7)
// The linear maps act on each row, so they run once per node (in torch, before this op) instead of once per edge; the
// weights are not normalised across a target's edges (the softmax runs over the heads of one edge), so a target's sum can
// be cut into fixed chunks and spread over many CTAs.
//
// Fixed orders, no atomics, the same bits on every run:
//   - each dot: k_agnn_dot's order over the C columns of one head (lane l of a G-lane group accumulates its 4-column
//     chunks l, l + G, ... with one __fmaf_rn per column, then a butterfly at xor distances G/2 .. 1), the same with float4
//     and scalar loads; then one __fdiv_rn by sqrtf(C), the max, one expf each, the h''-ascending __fadd_rn sum plus
//     exp(-m), one __fdiv_rn.
//   - a segment sum (k_dna_chunk_sums): the segment's edges in order, in chunks of kSegChunk counted from its first edge;
//     per edge the inner sum over h' ascending (one __fmul_rn, then __fmaf_rn), times the edge weight (one __fmul_rn),
//     added left to right from +0; the chunk sums added in chunk order (k_seg_combine); the forward then divides once.
// Backward, with gm_i = g_i / fl(cnt_i + 1e-7) and w_e = fl(n0_i * n1_j):
//   da[e,h,h'] = w_e * <gm_i[h], v_j[h']>,  t = a * (da - sum_h'' a * da) / sqrt(C)          (k_dna_edge<.., true>)
//   grad_q_i[h]  = sum_{dst_e = i} sum_h' t[e,h,h'] * k_j[h']      (the dst order)
//   grad_k_j[h'] = sum_{src_e = j} sum_h  t[e,h,h'] * q_i[h]       (a stable order by src, the coefficients transposed)
//   grad_v_j[h'] = sum_{src_e = j} w_e * sum_h a[e,h,h'] * gm_i[h]
// each a k_dna_chunk_sums pass.  n0 and n1 get no gradient.
//
// Order: unsorted dst (GCNDataFlow with self loops appends the loops) is ordered by segment.cu's stable radix sort after one
// flag read-back; the result is bit-identical to the call on the stably sorted edge list.
#include <cmath>

#include "segment.cuh"

namespace eu {

constexpr int kDnaMaxHeads = 8;   // the heads one edge's scores are held for in registers
constexpr int kDnaUnroll = 4;     // edges in flight per lane in the chunk sums

// <x[0, C), y[0, C)> in k_agnn_dot's order (see the file comment); every lane of the group returns the same bits
template <bool VEC>
__device__ __forceinline__ float dna_dot(const float* __restrict__ x, const float* __restrict__ y, int C, int G, int sub,
                                         unsigned gm) {
  float acc = 0.f;
  for (int d = sub * 4; d < C; d += G * 4) {
    if (VEC) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(x + d)), b = __ldg(reinterpret_cast<const float4*>(y + d));
      acc = __fmaf_rn(a.x, b.x, acc); acc = __fmaf_rn(a.y, b.y, acc);
      acc = __fmaf_rn(a.z, b.z, acc); acc = __fmaf_rn(a.w, b.w, acc);
    } else {
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (d + q < C) acc = __fmaf_rn(__ldg(x + d + q), __ldg(y + d + q), acc);
    }
  }
  for (int o = G >> 1; o > 0; o >>= 1) acc = __fadd_rn(acc, __shfl_xor_sync(gm, acc, o, G));
  return acc;
}

// G lanes per edge e, H <= kDnaMaxHeads.  Forward (BWD = false): x = q (by dst), y = k (by src); writes alpha[e, h, h'].
// Backward: x = gm (by dst), y = v (by src), alpha given; writes t[e, h, h'] = a * (da - sum_h'' a * da) / sqrt(C) with
// da = w_e * <gm_i[h], v_j[h']>.
template <bool VEC, bool BWD>
__global__ void __launch_bounds__(256) k_dna_edge(const float* __restrict__ x, const float* __restrict__ y,
                                                  const float* __restrict__ n0, const float* __restrict__ n1,
                                                  const int32_t* __restrict__ dst, const int32_t* __restrict__ src, int64_t E,
                                                  int H, int C, int G, float sc, const float* __restrict__ alpha_in,
                                                  float* __restrict__ res) {
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t e = tid >> (31 - __clz(G));
  const int sub = (int)(tid & (G - 1));
  if (e >= E) return;   // group-uniform
  const unsigned gm = group_mask(G);
  const int64_t HC = (int64_t)H * C;
  const int64_t i = __ldg(dst + e), j = __ldg(src + e);
  const float* xr = x + i * HC;
  const float* yr = y + j * HC;
  const float w = BWD ? __fmul_rn(__ldg(n0 + i), __ldg(n1 + j)) : 0.f;
  const int64_t HH = (int64_t)H * H;
  for (int h = 0; h < H; ++h) {
    float v[kDnaMaxHeads];
#pragma unroll
    for (int hp = 0; hp < kDnaMaxHeads; ++hp)
      if (hp < H) v[hp] = dna_dot<VEC>(xr + h * C, yr + hp * C, C, G, sub, gm);
    const int64_t base = e * HH + (int64_t)h * H;
    if (!BWD) {
      float m = 0.f;                                     // restricted_softmax: the max clipped below at 0
#pragma unroll
      for (int hp = 0; hp < kDnaMaxHeads; ++hp) {
        if (hp < H) {
          v[hp] = __fdiv_rn(v[hp], sc);
          m = v[hp] > m ? v[hp] : m;
        }
      }
      float den = 0.f;
#pragma unroll
      for (int hp = 0; hp < kDnaMaxHeads; ++hp) {
        if (hp < H) {
          v[hp] = expf(__fsub_rn(v[hp], m));
          den = __fadd_rn(den, v[hp]);
        }
      }
      den = __fadd_rn(den, expf(-m));
#pragma unroll
      for (int hp = 0; hp < kDnaMaxHeads; ++hp)
        if (hp < H && (hp & (G - 1)) == sub) res[base + hp] = __fdiv_rn(v[hp], den);
    } else {
      float a[kDnaMaxHeads];
      float S = 0.f;
#pragma unroll
      for (int hp = 0; hp < kDnaMaxHeads; ++hp) {
        if (hp < H) {
          a[hp] = __ldg(alpha_in + base + hp);
          v[hp] = __fmul_rn(w, v[hp]);
          S = __fadd_rn(S, __fmul_rn(a[hp], v[hp]));
        }
      }
#pragma unroll
      for (int hp = 0; hp < kDnaMaxHeads; ++hp)
        if (hp < H && (hp & (G - 1)) == sub) res[base + hp] = __fdiv_rn(__fmul_rn(a[hp], __fsub_rn(v[hp], S)), sc);
    }
  }
}

// G lanes per chunk c of the segments of an edge order (positions key-sorted, perm: position -> edge, null = identity).
// Chunk c - chunk_off[p] of segment p covers the positions [start[p] + (c - chunk_off[p]) * kSegChunk, ...), up to
// kSegChunk of them.  For output head h and column c of the head, summed left to right from +0:
//   sum over those edges of w_e * (sum over h' ascending of coef[e, h, h'] * rows[ridx_e, h' * C + c])
// (TRANS: coef[e, h', h]; w_e = fl(n0[dst_e] * n1[src_e]) when n0 is given, else no multiply).  A segment of one chunk
// writes seg[p]; the chunks of a longer one write partial[c] for k_seg_combine.  VEC: C % 4 == 0, 16-byte aligned rows.
template <bool VEC, bool TRANS>
__global__ void __launch_bounds__(256) k_dna_chunk_sums(const float* __restrict__ rows, const int32_t* __restrict__ ridx,
                                                        const float* __restrict__ coef, const float* __restrict__ n0,
                                                        const float* __restrict__ n1, const int32_t* __restrict__ dst,
                                                        const int32_t* __restrict__ src, const int32_t* __restrict__ perm,
                                                        const int32_t* __restrict__ start, const int32_t* __restrict__ chunk_off,
                                                        int64_t n, int64_t slots, int H, int C, int G, float* __restrict__ seg,
                                                        float* __restrict__ partial) {
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t c = tid >> (31 - __clz(G));
  const int sub = (int)(tid & (G - 1));
  if (c >= slots || c >= __ldg(chunk_off + n)) return;
  const int64_t p = key_upper_bound(chunk_off, n + 1, c) - 1;
  const int64_t c0 = __ldg(chunk_off + p), nch = __ldg(chunk_off + p + 1) - c0;
  const int64_t b = __ldg(start + p) + (c - c0) * kSegChunk;
  const int64_t e = min(b + kSegChunk, (int64_t)__ldg(start + p + 1));
  const int HC = H * C;   // < 2^31: checked by the launcher
  const int64_t HH = (int64_t)H * H;
  float* o = nch == 1 ? seg + p * HC : partial + c * HC;
  const int cs = TRANS ? H : 1, ho = TRANS ? 1 : H;   // coef[e, h, h'] = coef[e * HH + h * ho + h' * cs]
  if (VEC) {
    for (int d = sub * 4; d < HC; d += G * 4) {
      const int h = d / C, cc = d - h * C;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int64_t k0 = b; k0 < e; k0 += kDnaUnroll) {
        int64_t ed[kDnaUnroll];
        const float* r[kDnaUnroll];
        float4 in[kDnaUnroll];
#pragma unroll
        for (int q = 0; q < kDnaUnroll; ++q) {
          ed[q] = k0 + q < e ? edge_at(perm, k0 + q) : 0;
          r[q] = rows + (int64_t)__ldg(ridx + ed[q]) * HC + cc;
        }
        for (int hp = 0; hp < H; ++hp) {
          float4 x[kDnaUnroll];
          float cf[kDnaUnroll];
#pragma unroll
          for (int q = 0; q < kDnaUnroll; ++q) {
            if (k0 + q < e) {
              x[q] = __ldg(reinterpret_cast<const float4*>(r[q] + hp * C));
              cf[q] = __ldg(coef + ed[q] * HH + h * ho + hp * cs);
            }
          }
#pragma unroll
          for (int q = 0; q < kDnaUnroll; ++q) {
            if (k0 + q < e) {
              if (hp == 0) {
                in[q] = make_float4(__fmul_rn(cf[q], x[q].x), __fmul_rn(cf[q], x[q].y), __fmul_rn(cf[q], x[q].z), __fmul_rn(cf[q], x[q].w));
              } else {
                in[q].x = __fmaf_rn(cf[q], x[q].x, in[q].x); in[q].y = __fmaf_rn(cf[q], x[q].y, in[q].y);
                in[q].z = __fmaf_rn(cf[q], x[q].z, in[q].z); in[q].w = __fmaf_rn(cf[q], x[q].w, in[q].w);
              }
            }
          }
        }
#pragma unroll
        for (int q = 0; q < kDnaUnroll; ++q) {
          if (k0 + q < e) {
            if (n0) {
              const float w = __fmul_rn(__ldg(n0 + __ldg(dst + ed[q])), __ldg(n1 + __ldg(src + ed[q])));
              in[q] = make_float4(__fmul_rn(w, in[q].x), __fmul_rn(w, in[q].y), __fmul_rn(w, in[q].z), __fmul_rn(w, in[q].w));
            }
            acc.x = __fadd_rn(acc.x, in[q].x); acc.y = __fadd_rn(acc.y, in[q].y);
            acc.z = __fadd_rn(acc.z, in[q].z); acc.w = __fadd_rn(acc.w, in[q].w);
          }
        }
      }
      *reinterpret_cast<float4*>(o + d) = acc;
    }
  } else {
    for (int d = sub; d < HC; d += G) {
      const int h = d / C, cc = d - h * C;
      float acc = 0.f;
      for (int64_t k0 = b; k0 < e; k0 += kDnaUnroll) {
        int64_t ed[kDnaUnroll];
        const float* r[kDnaUnroll];
        float in[kDnaUnroll];
#pragma unroll
        for (int q = 0; q < kDnaUnroll; ++q) {
          ed[q] = k0 + q < e ? edge_at(perm, k0 + q) : 0;
          r[q] = rows + (int64_t)__ldg(ridx + ed[q]) * HC + cc;
        }
        for (int hp = 0; hp < H; ++hp) {
          float x[kDnaUnroll], cf[kDnaUnroll];
#pragma unroll
          for (int q = 0; q < kDnaUnroll; ++q) {
            if (k0 + q < e) {
              x[q] = __ldg(r[q] + hp * C);
              cf[q] = __ldg(coef + ed[q] * HH + h * ho + hp * cs);
            }
          }
#pragma unroll
          for (int q = 0; q < kDnaUnroll; ++q)
            if (k0 + q < e) in[q] = hp == 0 ? __fmul_rn(cf[q], x[q]) : __fmaf_rn(cf[q], x[q], in[q]);
        }
#pragma unroll
        for (int q = 0; q < kDnaUnroll; ++q) {
          if (k0 + q < e) {
            if (n0) in[q] = __fmul_rn(__fmul_rn(__ldg(n0 + __ldg(dst + ed[q])), __ldg(n1 + __ldg(src + ed[q]))), in[q]);
            acc = __fadd_rn(acc, in[q]);
          }
        }
      }
      o[d] = acc;
    }
  }
}

// v[i, d] = v[i, d] / fl(fl(cnt_i) + 1e-7) (or g[i, d] / ... into v when g is given): scatter_mean's divisor, one __fdiv_rn;
// cnt_i = start[i + 1] - start[i].  One thread per (i, d).
__global__ void k_dna_mean(const float* __restrict__ g, const int32_t* __restrict__ start, int64_t n, int dim, float* __restrict__ v) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= n * dim) return;
  const int64_t i = t / dim;
  const float den = __fadd_rn((float)(__ldg(start + i + 1) - __ldg(start + i)), 1e-7f);
  v[t] = __fdiv_rn(g ? __ldg(g + t) : v[t], den);
}

// seg[p] = the weighted segment sums of k_dna_chunk_sums over the segments S of the order o (E > 0), chunks combined
static int dna_seg_sums(eu_ctx* c, const SegPlan& S, const EdgeOrder& o, const float* rows, const int32_t* ridx, const float* coef,
                        bool trans, const float* n0, const float* n1, const int32_t* dst, const int32_t* src, int H, int C,
                        float* seg) {
  cudaStream_t s = c->stream;
  const int64_t HC = (int64_t)H * C;
  const bool vec = C % 4 == 0 && aligned16(rows) && aligned16(seg);
  const int G = group_lanes(vec ? HC / 4 : HC);
  const unsigned blocks = (unsigned)ceil_div(S.slots * G, 256);
#define EU_DNA_SUMS(V, T)                                                                                                   \
  k_dna_chunk_sums<V, T><<<blocks, 256, 0, s>>>(rows, ridx, coef, n0, n1, dst, src, o.perm, S.start, S.chunk_off, S.n, S.slots, \
                                                H, C, G, seg, S.partial)
  if (vec) { if (trans) EU_DNA_SUMS(true, true); else EU_DNA_SUMS(true, false); }
  else { if (trans) EU_DNA_SUMS(false, true); else EU_DNA_SUMS(false, false); }
#undef EU_DNA_SUMS
  EU_LAUNCHED();
  k_seg_combine<<<(unsigned)ceil_div(S.n * HC, 256), 256, 0, s>>>(S.chunk_off, S.partial, S.n, (int)HC, seg);
  EU_LAUNCHED();
  return EU_OK;
}

// k_dna_edge over E > 0 edges
template <bool BWD>
static int dna_edge(eu_ctx* c, const float* x, const float* y, const float* n0, const float* n1, const int32_t* dst,
                    const int32_t* src, int64_t E, int H, int C, const float* alpha_in, float* res) {
  const bool vec = C % 4 == 0 && aligned16(x) && aligned16(y);
  const int G = group_lanes(ceil_div(C, 4));   // one lane per 4-column chunk, both paths: the same order
  const unsigned blocks = (unsigned)ceil_div(E * G, 256);
  const float sc = sqrtf((float)C);
  if (vec) k_dna_edge<true, BWD><<<blocks, 256, 0, c->stream>>>(x, y, n0, n1, dst, src, E, H, C, G, sc, alpha_in, res);
  else k_dna_edge<false, BWD><<<blocks, 256, 0, c->stream>>>(x, y, n0, n1, dst, src, E, H, C, G, sc, alpha_in, res);
  EU_LAUNCHED();
  return EU_OK;
}

static int dna_check_args(const char* who, int64_t E, int64_t n_dst, int64_t n_src, int32_t heads, int32_t head_dim) {
  if (E >= ((int64_t)1 << 31) || n_dst >= ((int64_t)1 << 31) - 1 || n_src >= ((int64_t)1 << 31) - 1 ||
      (int64_t)heads * head_dim >= ((int64_t)1 << 31)) {
    set_error("%s: 2^31 or more edges, rows or columns are not supported", who);
    return EU_ERR_UNSUPPORTED;
  }
  if (heads > kDnaMaxHeads) {
    set_error("%s: heads = %d is not supported (at most %d)", who, (int)heads, kDnaMaxHeads);
    return EU_ERR_UNSUPPORTED;
  }
  return EU_OK;
}

}  // namespace eu

using namespace eu;

extern "C" {

int eu_dna_aggregate(eu_ctx* c, const float* q, const float* k, const float* v, const float* n0, const float* n1, const int32_t* dst,
                     const int32_t* src, int64_t E, int64_t n_dst, int64_t n_src, int32_t heads, int32_t head_dim, float* out,
                     float* alpha) {
  const char* who = "eu_dna_aggregate";
  if (!c || heads < 1 || head_dim < 1 || E < 0 || n_dst < 0 || n_src < 0 || (E > 0 && (n_dst == 0 || n_src == 0)) ||
      (E > 0 && (!q || !k || !v || !n0 || !n1 || !dst || !src)) || (n_dst > 0 && !out)) {
    set_error("%s: bad argument", who);
    return EU_ERR_INVALID;
  }
  int rc = dna_check_args(who, E, n_dst, n_src, heads, head_dim);
  if (rc) return rc;
  EU_CUDA(cudaSetDevice(c->g->device));
  if (n_dst == 0) return EU_OK;
  cudaStream_t s = c->stream;
  const int64_t H = heads, C = head_dim, HC = H * C;
  if (E == 0) {                                        // no edge: every target's mean is 0 / 1e-7 = 0
    EU_CUDA(cudaMemsetAsync(out, 0, 4 * (size_t)(n_dst * HC), s));
    return EU_OK;
  }
  // head: alpha scratch when the caller wants none; tail: the target segments
  TargetOrder to;
  if ((rc = order_targets(c, dst, E, n_dst, alpha ? 0 : a256(4 * (size_t)(E * H * H)), seg_plan_bytes(E, n_dst, HC), "dna_sort", &to)))
    return rc;
  const EdgeOrder& ord = to.ord;
  float* al = alpha ? alpha : (float*)to.head;
  {
    EuProfScope ps(c, "dna_scores", E);
    if ((rc = dna_edge<false>(c, q, k, nullptr, nullptr, dst, src, E, (int)H, (int)C, nullptr, al))) return rc;
  }
  EuProfScope ps(c, "dna_sums", E);
  SegPlan S;
  if ((rc = plan_segments(c, ord, E, n_dst, to.tail, &S))) return rc;
  if ((rc = dna_seg_sums(c, S, ord, v, src, al, false, n0, n1, dst, src, (int)H, (int)C, out))) return rc;
  k_dna_mean<<<(unsigned)ceil_div(n_dst * HC, 256), 256, 0, s>>>(nullptr, S.start, n_dst, (int)HC, out);
  EU_LAUNCHED();
  return EU_OK;
}

int eu_dna_aggregate_backward(eu_ctx* c, const float* grad_out, const float* q, const float* k, const float* v, const float* n0,
                              const float* n1, const float* alpha, const int32_t* dst, const int32_t* src, int64_t E, int64_t n_dst,
                              int64_t n_src, int32_t heads, int32_t head_dim, float* grad_q, float* grad_k, float* grad_v) {
  const char* who = "eu_dna_aggregate_backward";
  if (!c || heads < 1 || head_dim < 1 || E < 0 || n_dst < 0 || n_src < 0 || (E > 0 && (n_dst == 0 || n_src == 0)) ||
      (E > 0 && (!grad_out || !q || !k || !v || !n0 || !n1 || !alpha || !dst || !src)) || (n_dst > 0 && !grad_q) ||
      (n_src > 0 && (!grad_k || !grad_v))) {
    set_error("%s: bad argument", who);
    return EU_ERR_INVALID;
  }
  int rc = dna_check_args(who, E, n_dst, n_src, heads, head_dim);
  if (rc) return rc;
  EU_CUDA(cudaSetDevice(c->g->device));
  cudaStream_t s = c->stream;
  const int64_t H = heads, C = head_dim, HC = H * C;
  if (E == 0) {                                        // no edge: every gradient is zero
    if (n_dst > 0) EU_CUDA(cudaMemsetAsync(grad_q, 0, 4 * (size_t)(n_dst * HC), s));
    if (n_src > 0) {
      EU_CUDA(cudaMemsetAsync(grad_k, 0, 4 * (size_t)(n_src * HC), s));
      EU_CUDA(cudaMemsetAsync(grad_v, 0, 4 * (size_t)(n_src * HC), s));
    }
    return EU_OK;
  }
  // head: gm [n_dst, dim] | t [E, H, H]; tail: the src order | the target segments | the source segments
  const size_t o_dseg = order_bytes(E, n_src), o_sseg = o_dseg + seg_plan_bytes(E, n_dst, HC);
  TargetOrder to;
  if ((rc = order_targets(c, dst, E, n_dst, a256(4 * (size_t)(n_dst * HC)) + a256(4 * (size_t)(E * H * H)),
                          o_sseg + seg_plan_bytes(E, n_src, HC), "dna_sort", &to)))
    return rc;
  float* gm = (float*)to.head;
  float* t = (float*)(to.head + a256(4 * (size_t)(n_dst * HC)));
  const EdgeOrder& dord = to.ord;
  EdgeOrder sord;
  SegPlan SD, SS;
  {
    EuProfScope ps(c, "dna_bwd_scores", E);
    if ((rc = plan_segments(c, dord, E, n_dst, to.tail + o_dseg, &SD))) return rc;
    k_dna_mean<<<(unsigned)ceil_div(n_dst * HC, 256), 256, 0, s>>>(grad_out, SD.start, n_dst, (int)HC, gm);
    EU_LAUNCHED();
    if ((rc = dna_edge<true>(c, gm, v, n0, n1, dst, src, E, (int)H, (int)C, alpha, t))) return rc;
  }
  {
    EuProfScope ps(c, "dna_bwd_q", E);
    if ((rc = dna_seg_sums(c, SD, dord, k, src, t, false, nullptr, nullptr, dst, src, (int)H, (int)C, grad_q))) return rc;
  }
  {
    EuProfScope ps(c, "dna_bwd_sort_src", E);
    if ((rc = order_by(c, src, E, n_src, to.tail, &sord))) return rc;
    if ((rc = plan_segments(c, sord, E, n_src, to.tail + o_sseg, &SS))) return rc;
  }
  {
    EuProfScope ps(c, "dna_bwd_kv", E);
    if ((rc = dna_seg_sums(c, SS, sord, q, dst, t, true, nullptr, nullptr, dst, src, (int)H, (int)C, grad_k))) return rc;
    if ((rc = dna_seg_sums(c, SS, sord, gm, dst, alpha, true, n0, n1, dst, src, (int)H, (int)C, grad_v))) return rc;
  }
  return EU_OK;
}

}  // extern "C"
