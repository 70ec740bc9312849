// The attention readouts of the graph pools, forward and backward: AttentionPool (aggr = 'add') and one Set2SetPool step.
//
// Reference semantics (file:line relative to /root/reference):
//   AttentionPool.__call__   tf_euler/python/graph_pool/attention_pool.py (gate -> scatter_softmax -> gate * x -> scatter_add)
//   Set2SetPool.__call__     tf_euler/python/graph_pool/set2set_pool.py (e = <x_n, q[g(n)]> -> scatter_softmax -> a * x ->
//                            scatter_add, per processing step)
//   scatter_softmax          tf_euler/python/euler_ops/mp_ops.py:76-79 (scatter_max initialised to -1e9)
//
// Rows n of x [N, D] belong to graph g(n) = index[n] in [0, B).  A graph's rows are walked in the stable order of index
// (order_targets: a sorted index is walked as given), cut into the chunks of a fixed-order segment sum (segment.cuh):
//   m_b = max(-1e9, max of its logits)          (per chunk, then over the chunks: max is exact in any order)
//   s_b = sum of expf(l_n - m_b)                 (fixed-order chunked sum)
//   alpha_n = expf(l_n - m_b) / s_b,  r_b = sum of alpha_n * x_n   (fixed-order chunked row sum)
// with l_n the given logit (AttentionPool's gate) or <x_n, q_b> (Set2Set; k_agnn_dot's fixed order).  One rounded operation
// at a time, so for graphs of at most 256 rows walked in order the result is the composition's bit for bit; a graph of no
// rows gets a zero row.  Backward, with g = grad_r:
//   d_n = <x_n, g_b> (k_agnn_dot's order),  S_b = sum alpha_n * d_n (chunked),  dl_n = alpha_n * (d_n - S_b)
//   grad_x_n = alpha_n * g_b (+ dl_n * q_b),  grad_logits = dl,  grad_q_b = sum dl_n * x_n (chunked)
// No atomics anywhere: every result is the same from run to run.
#include "segment.cuh"

namespace eu {

constexpr int kRoUnroll = 8;   // rows in flight per lane in the chunked row sums

// the segment p of chunk c, its first chunk c0 and chunk count nch, and the chunk's positions [b, e)
__device__ __forceinline__ void ro_chunk(const int32_t* __restrict__ start, const int32_t* __restrict__ chunk_off, int64_t n,
                                         int64_t c, int64_t* p, int64_t* c0, int64_t* nch, int64_t* b, int64_t* e) {
  *p = key_upper_bound(chunk_off, n + 1, c) - 1;
  *c0 = __ldg(chunk_off + *p);
  *nch = __ldg(chunk_off + *p + 1) - *c0;
  *b = __ldg(start + *p) + (c - *c0) * kSegChunk;
  *e = min(*b + kSegChunk, (int64_t)__ldg(start + *p + 1));
}

// a warp per chunk: cmax[c] = max(-1e9, the chunk's logits)
__global__ void __launch_bounds__(256) k_ro_chunk_max(const float* __restrict__ lg, const int32_t* __restrict__ perm,
                                                      const int32_t* __restrict__ start, const int32_t* __restrict__ chunk_off,
                                                      int64_t n, int64_t slots, float* __restrict__ cmax) {
  const int64_t c = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (c >= slots || c >= __ldg(chunk_off + n)) return;   // warp-uniform
  int64_t p, c0, nch, b, e;
  ro_chunk(start, chunk_off, n, c, &p, &c0, &nch, &b, &e);
  float m = -1e9f;                                        // scatter_max's initial value; a NaN logit never wins
  for (int64_t k = b + lane; k < e; k += 32) {
    const float u = __ldg(lg + edge_at(perm, k));
    m = u > m ? u : m;
  }
  for (int o = 16; o > 0; o >>= 1) {
    const float v = __shfl_xor_sync(0xffffffffu, m, o);
    m = v > m ? v : m;
  }
  if (lane == 0) cmax[c] = m;
}

// A warp per chunk.  EXP: w[row] = expf(lg[row] - m_p) with m_p the max of the segment's chunk maxima, and the chunk's sum
// of w; otherwise the chunk's sum of a[row] * w[row].  Sums run left to right from +0; a segment of one chunk writes seg[p],
// the chunks of a longer one partial[c] for k_seg_combine.  lg and w may alias (each row is read and written by one lane).
template <bool EXP>
__global__ void __launch_bounds__(256) k_ro_chunk_scalar(const float* lg, const float* __restrict__ a,
                                                         const float* __restrict__ cmax, const int32_t* __restrict__ perm,
                                                         const int32_t* __restrict__ start, const int32_t* __restrict__ chunk_off,
                                                         int64_t n, int64_t slots, float* w, float* __restrict__ seg,
                                                         float* __restrict__ partial) {
  const int64_t c = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (c >= slots || c >= __ldg(chunk_off + n)) return;   // warp-uniform
  int64_t p, c0, nch, b, e;
  ro_chunk(start, chunk_off, n, c, &p, &c0, &nch, &b, &e);
  float m = -1e9f;
  if (EXP) {
    for (int64_t k = c0 + lane; k < c0 + nch; k += 32) { const float v = __ldg(cmax + k); m = v > m ? v : m; }
    for (int o = 16; o > 0; o >>= 1) { const float v = __shfl_xor_sync(0xffffffffu, m, o); m = v > m ? v : m; }
  }
  float s = 0.f;
  for (int64_t k0 = b; k0 < e; k0 += 32) {                // warp-uniform trip count
    const int64_t k = k0 + lane;
    float v = 0.f;
    if (k < e) {
      const int64_t r = edge_at(perm, k);
      if (EXP) { v = expf(__fsub_rn(lg[r], m)); w[r] = v; }
      else v = __fmul_rn(__ldg(a + r), w[r]);
    }
    const int cnt = e - k0 < 32 ? (int)(e - k0) : 32;
    for (int j = 0; j < cnt; ++j) s = __fadd_rn(s, __shfl_sync(0xffffffffu, v, j));
  }
  if (lane == 0) (nch == 1 ? seg[p] : partial[c]) = s;
}

// out[n] = w[n] / den[index[n]] (DL: out[n] = a[n] * (w[n] - den[index[n]])); one thread per row
template <bool DL>
__global__ void k_ro_rows(const float* __restrict__ a, const float* w, const float* __restrict__ den,
                          const int32_t* __restrict__ index, int64_t N, float* out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < N; i += (int64_t)gridDim.x * blockDim.x) {
    const float d = __ldg(den + __ldg(index + i));
    out[i] = DL ? __fmul_rn(__ldg(a + i), __fsub_rn(w[i], d)) : __fdiv_rn(w[i], d);
  }
}

// G lanes per chunk (chunks as in k_ro_chunk_max): the chunk's sum of w[row] * x[row, :], left to right from +0, into
// seg[p, :] (a segment of one chunk) or partial[c, :].  VEC: D % 4 == 0 and 16-byte aligned rows.
template <bool VEC>
__global__ void __launch_bounds__(256) k_ro_chunk_rows(const float* __restrict__ x, const float* __restrict__ w,
                                                       const int32_t* __restrict__ perm, const int32_t* __restrict__ start,
                                                       const int32_t* __restrict__ chunk_off, int64_t n, int64_t slots, int D,
                                                       int G, float* __restrict__ seg, float* __restrict__ partial) {
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t c = tid >> (31 - __clz(G));
  const int sub = (int)(tid & (G - 1));
  if (c >= slots || c >= __ldg(chunk_off + n)) return;
  int64_t p, c0, nch, b, e;
  ro_chunk(start, chunk_off, n, c, &p, &c0, &nch, &b, &e);
  float* o = nch == 1 ? seg + p * D : partial + c * D;
  if (VEC) {
    for (int d = sub * 4; d < D; d += G * 4) {
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int64_t k0 = b; k0 < e; k0 += kRoUnroll) {
        float4 v[kRoUnroll];
        float a[kRoUnroll];
#pragma unroll
        for (int q = 0; q < kRoUnroll; ++q) {
          if (k0 + q < e) {
            const int64_t r = edge_at(perm, k0 + q);
            v[q] = __ldg(reinterpret_cast<const float4*>(x + r * D + d));
            a[q] = __ldg(w + r);
          }
        }
#pragma unroll
        for (int q = 0; q < kRoUnroll; ++q) {
          if (k0 + q < e) {
            acc.x = __fadd_rn(acc.x, __fmul_rn(a[q], v[q].x)); acc.y = __fadd_rn(acc.y, __fmul_rn(a[q], v[q].y));
            acc.z = __fadd_rn(acc.z, __fmul_rn(a[q], v[q].z)); acc.w = __fadd_rn(acc.w, __fmul_rn(a[q], v[q].w));
          }
        }
      }
      *reinterpret_cast<float4*>(o + d) = acc;
    }
  } else {
    for (int d = sub; d < D; d += G) {
      float acc = 0.f;
      for (int64_t k0 = b; k0 < e; k0 += kRoUnroll) {
        float v[kRoUnroll], a[kRoUnroll];
#pragma unroll
        for (int q = 0; q < kRoUnroll; ++q) {
          if (k0 + q < e) {
            const int64_t r = edge_at(perm, k0 + q);
            v[q] = __ldg(x + r * D + d);
            a[q] = __ldg(w + r);
          }
        }
#pragma unroll
        for (int q = 0; q < kRoUnroll; ++q)
          if (k0 + q < e) acc = __fadd_rn(acc, __fmul_rn(a[q], v[q]));
      }
      o[d] = acc;
    }
  }
}

// grad_x[n, :] = alpha[n] * g[index[n], :] (+ dl[n] * q[index[n], :] when q is given); one thread per 4 columns (VEC) or column
template <bool VEC>
__global__ void k_ro_grad_x(const float* __restrict__ g, const float* __restrict__ q, const float* __restrict__ alpha,
                            const float* __restrict__ dl, const int32_t* __restrict__ index, int64_t N, int D,
                            float* __restrict__ gx) {
  const int W = VEC ? D / 4 : D;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < N * W; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / W;
    const int d = (int)(t - i * W) * (VEC ? 4 : 1);
    const int64_t bo = (int64_t)__ldg(index + i) * D + d;
    const float al = __ldg(alpha + i), l = q ? __ldg(dl + i) : 0.f;
    if (VEC) {
      const float4 gv = __ldg(reinterpret_cast<const float4*>(g + bo));
      float4 r = make_float4(__fmul_rn(al, gv.x), __fmul_rn(al, gv.y), __fmul_rn(al, gv.z), __fmul_rn(al, gv.w));
      if (q) {
        const float4 qv = __ldg(reinterpret_cast<const float4*>(q + bo));
        r.x = __fadd_rn(r.x, __fmul_rn(l, qv.x)); r.y = __fadd_rn(r.y, __fmul_rn(l, qv.y));
        r.z = __fadd_rn(r.z, __fmul_rn(l, qv.z)); r.w = __fadd_rn(r.w, __fmul_rn(l, qv.w));
      }
      *reinterpret_cast<float4*>(gx + i * D + d) = r;
    } else {
      float r = __fmul_rn(al, __ldg(g + bo));
      if (q) r = __fadd_rn(r, __fmul_rn(l, __ldg(q + bo)));
      gx[i * D + d] = r;
    }
  }
}

// seg[b, :] = sum over the rows of segment b of w[row] * x[row, :] (chunked; a segment of no rows gets zeros)
static int ro_row_sums(eu_ctx* c, const SegPlan& S, const EdgeOrder& o, const float* x, const float* w, int D, float* seg) {
  cudaStream_t s = c->stream;
  const bool vec = D % 4 == 0 && aligned16(x) && aligned16(seg);
  const int G = group_lanes(vec ? D / 4 : D);
  const unsigned blocks = (unsigned)ceil_div(S.slots * G, 256);
  if (vec) k_ro_chunk_rows<true><<<blocks, 256, 0, s>>>(x, w, o.perm, S.start, S.chunk_off, S.n, S.slots, D, G, seg, S.partial);
  else k_ro_chunk_rows<false><<<blocks, 256, 0, s>>>(x, w, o.perm, S.start, S.chunk_off, S.n, S.slots, D, G, seg, S.partial);
  EU_LAUNCHED();
  k_seg_combine<<<(unsigned)ceil_div(S.n * D, 256), 256, 0, s>>>(S.chunk_off, S.partial, S.n, D, seg);
  EU_LAUNCHED();
  return EU_OK;
}

// the chunked scalar sums of k_ro_chunk_scalar into seg [n], chunks combined
template <bool EXP>
static int ro_scalar_sums(eu_ctx* c, const SegPlan& S, const EdgeOrder& o, const float* lg, const float* a, const float* cmax,
                          float* w, float* seg) {
  cudaStream_t s = c->stream;
  k_ro_chunk_scalar<EXP><<<(unsigned)ceil_div(S.slots * 32, 256), 256, 0, s>>>(lg, a, cmax, o.perm, S.start, S.chunk_off, S.n,
                                                                              S.slots, w, seg, S.partial);
  EU_LAUNCHED();
  k_seg_combine<<<(unsigned)ceil_div(S.n, 256), 256, 0, s>>>(S.chunk_off, S.partial, S.n, 1, seg);
  EU_LAUNCHED();
  return EU_OK;
}

static int ro_check(const char* who, int64_t N, int64_t B, int32_t dim) {
  if (N >= ((int64_t)1 << 31) || B >= ((int64_t)1 << 31) - 1 || N * (int64_t)dim >= ((int64_t)1 << 40)) {
    set_error("%s: 2^31 or more rows or graphs are not supported", who);
    return EU_ERR_UNSUPPORTED;
  }
  return EU_OK;
}

}  // namespace eu

using namespace eu;

extern "C" {

int eu_graph_attention_readout(eu_ctx* c, const float* x, const int32_t* index, int64_t N, int64_t B, int32_t dim,
                               const float* logits, const float* q, float* out, float* alpha) {
  const char* who = "eu_graph_attention_readout";
  if (!c || dim < 1 || N < 0 || B < 0 || (N > 0 && B == 0) || (!logits == !q) ||
      (N > 0 && (!x || !index || !alpha)) || (B > 0 && !out)) {
    set_error("%s: bad argument (exactly one of logits and q)", who);
    return EU_ERR_INVALID;
  }
  int rc = ro_check(who, N, B, dim);
  if (rc) return rc;
  EU_CUDA(cudaSetDevice(c->g->device));
  if (B == 0) return EU_OK;
  cudaStream_t s = c->stream;
  if (N == 0) {   // otherwise k_seg_combine writes the zero row of a graph of no rows
    EU_CUDA(cudaMemsetAsync(out, 0, 4 * (size_t)(B * dim), s));
    return EU_OK;
  }
  // head: chunk maxima [B + N / 256] | exp sums [B]; tail: the graph segments
  const int64_t slots = B + N / kSegChunk;
  const size_t o_sum = a256(4 * (size_t)slots);
  TargetOrder t;
  if ((rc = order_targets(c, index, N, B, o_sum + a256(4 * (size_t)B), seg_plan_bytes(N, B, dim), "readout_sort", &t))) return rc;
  float* cmax = (float*)t.head;
  float* ssum = (float*)(t.head + o_sum);
  const EdgeOrder& ord = t.ord;
  EuProfScope ps(c, "readout_fwd", N);
  SegPlan S;
  if ((rc = plan_segments(c, ord, N, B, t.tail, &S))) return rc;
  const float* lg = logits;
  if (q) {   // Set2Set: the logits <x_n, q[g(n)]> into alpha
    if ((rc = agnn_dot(c, x, q, nullptr, index, N, dim, nullptr, alpha, nullptr))) return rc;
    lg = alpha;
  }
  k_ro_chunk_max<<<(unsigned)ceil_div(S.slots * 32, 256), 256, 0, s>>>(lg, ord.perm, S.start, S.chunk_off, B, S.slots, cmax);
  EU_LAUNCHED();
  if ((rc = ro_scalar_sums<true>(c, S, ord, lg, nullptr, cmax, alpha, ssum))) return rc;   // alpha <- exp, ssum <- their sums
  k_ro_rows<false><<<stride_grid(N), 256, 0, s>>>(nullptr, alpha, ssum, index, N, alpha);
  EU_LAUNCHED();
  return ro_row_sums(c, S, ord, x, alpha, dim, out);
}

int eu_graph_attention_readout_backward(eu_ctx* c, const float* grad_out, const float* x, const int32_t* index, int64_t N,
                                        int64_t B, int32_t dim, const float* q, const float* alpha, float* grad_x,
                                        float* grad_logits, float* grad_q) {
  const char* who = "eu_graph_attention_readout_backward";
  if (!c || dim < 1 || N < 0 || B < 0 || (N > 0 && B == 0) ||
      (N > 0 && (!grad_out || !x || !index || !alpha || !grad_x || (!q && !grad_logits))) || (q && B > 0 && !grad_q)) {
    set_error("%s: bad argument", who);
    return EU_ERR_INVALID;
  }
  int rc = ro_check(who, N, B, dim);
  if (rc) return rc;
  EU_CUDA(cudaSetDevice(c->g->device));
  cudaStream_t s = c->stream;
  if (N == 0) {
    if (q && B > 0) EU_CUDA(cudaMemsetAsync(grad_q, 0, 4 * (size_t)(B * dim), s));
    return EU_OK;
  }
  // head: d, then dl [N] | S [B]; tail: the graph segments
  const size_t o_S = a256(4 * (size_t)N);
  TargetOrder t;
  if ((rc = order_targets(c, index, N, B, o_S + a256(4 * (size_t)B), seg_plan_bytes(N, B, dim), "readout_sort", &t))) return rc;
  float* dl = (float*)t.head;
  float* S_b = (float*)(t.head + o_S);
  const EdgeOrder& ord = t.ord;
  EuProfScope ps(c, "readout_bwd", N);
  SegPlan S;
  if ((rc = plan_segments(c, ord, N, B, t.tail, &S))) return rc;
  if ((rc = agnn_dot(c, x, grad_out, nullptr, index, N, dim, nullptr, dl, nullptr))) return rc;    // d_n = <x_n, g_b>
  if ((rc = ro_scalar_sums<false>(c, S, ord, nullptr, alpha, nullptr, dl, S_b))) return rc;       // S_b = sum alpha * d
  float* dlo = q ? dl : grad_logits;
  k_ro_rows<true><<<stride_grid(N), 256, 0, s>>>(alpha, dl, S_b, index, N, dlo);                  // dl = alpha (d - S)
  EU_LAUNCHED();
  const bool vec = dim % 4 == 0 && aligned16(grad_out) && aligned16(grad_x) && (!q || aligned16(q));
  const int64_t W = vec ? dim / 4 : dim;
  if (vec) k_ro_grad_x<true><<<stride_grid(N * W), 256, 0, s>>>(grad_out, q, alpha, dlo, index, N, dim, grad_x);
  else k_ro_grad_x<false><<<stride_grid(N * W), 256, 0, s>>>(grad_out, q, alpha, dlo, index, N, dim, grad_x);
  EU_LAUNCHED();
  if (q) return ro_row_sums(c, S, ord, x, dl, dim, grad_q);                                       // grad_q = sum dl * x
  return EU_OK;
}

}  // extern "C"
