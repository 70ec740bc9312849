// GATConv's attention aggregation, forward and backward, over the edge lists of dataflow blocks (f32 data, i32 indices).
//
// Reference semantics (file:line relative to /root/reference):
//   GATConv.__call__ / apply_edge   tf_euler/python/convolution/gat_conv.py:53-78 with aggr = 'add', after its `fc`
//   scatter_softmax                 tf_euler/python/euler_ops/mp_ops.py:76-79 (scatter_max initialised to -1e9)
//
// For head h and edge e = (dst_e, src_e):
//   u[e,h]     = leaky_relu(s_dst[dst_e,h] + s_src[src_e,h], 0.2)
//   alpha[e,h] = scatter_softmax(u, dst, n_dst)
//   out[i, h*C:(h+1)*C] = sum over the edges e with dst_e = i of alpha[e,h] * h_src[src_e, h*C:(h+1)*C]
//
// Forward: a group of G lanes per target row, as k_scatter_sorted.  The arithmetic is the composition gather -> add ->
// leaky_relu -> scatter_softmax -> multiply -> scatter_add over the sorted path, one rounded operation at a time
// (__fadd_rn / __fmul_rn: nvcc would contract to FMA), with the segment sums left to right in edge order; so for
// non-decreasing dst the output and alpha are that composition's bit for bit.  Unsorted dst is ordered by a stable radix
// sort first and the same kernel runs through the permutation.
//
// Backward: one kernel per target row (d_alpha, du, grad_s_dst; du to scratch), a stable radix sort of the edges by source,
// one kernel per source row (grad_h_src, grad_s_src).  Every sum runs in edge order within its segment: deterministic, no
// atomics.
//
// AGNNConv's aggregation (agnn_conv.py:32-54, aggr = 'add') is the same softmax and weighted sum with H = 1, C = dim and a
// cosine logit per edge, u[e] = beta * <nrm_dst[dst_e], nrm_src[src_e]>, computed edge-parallel first (k_agnn_dot) and read
// by k_gat_fwd<VEC, true>.  Its backward reuses k_agnn_dot (d_alpha), k_gat_bwd_src (every segmented row sum, by target and
// by source) and the orders above; see eu_agnn_aggregate_backward.
#include "segment.cuh"

namespace eu {

__device__ __forceinline__ float leaky(float x) { return x > 0.f ? x : __fmul_rn(x, 0.2f); }

constexpr int kGatUnroll = 8;   // source rows in flight per lane in the ordered column sums

// G lanes per target row r; its edges are positions [lb(r), lb(r+1)) of the dst-sorted order `key` (perm: position -> edge).
// Per head: the max of the logits (a group reduction: max is exact in any order), the exps (in parallel) and their sum (a
// serial chain in edge order, broadcast lane by lane), then alpha = exp / sum.  alpha doubles as the scratch of u and exp.
// Then the columns: lanes over H*C, edges in order, kGatUnroll source rows loaded ahead of the ordered adds.
// PRE: the logits are already in alpha (AGNN's beta * cos); s_dst and s_src are not read.
template <bool VEC, bool PRE>
__global__ void __launch_bounds__(256) k_gat_fwd(const float* __restrict__ h_src, const float* __restrict__ s_dst,
                                                 const float* __restrict__ s_src, const int32_t* __restrict__ key,
                                                 const int32_t* __restrict__ perm, const int32_t* __restrict__ src, int64_t E,
                                                 int64_t n_dst, int H, int C, int G, float* __restrict__ alpha,
                                                 float* __restrict__ out) {
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t r = tid >> (31 - __clz(G));
  const int sub = (int)(tid & (G - 1));
  if (r >= n_dst) return;   // group-uniform
  const unsigned gm = group_mask(G);
  const int64_t b = key_lower_bound(key, E, r), e = key_lower_bound(key, E, r + 1);
  const int HC = H * C;   // < 2^31: checked by the launcher
  for (int h = 0; h < H && b < e; ++h) {
    const float sd = PRE ? 0.f : __ldg(s_dst + r * H + h);
    float m = -1e9f;                                   // scatter_max's initial value; a NaN logit never wins
    for (int64_t k = b + sub; k < e; k += G) {
      const int64_t ed = edge_at(perm, k);
      float u;
      if (PRE) {
        u = alpha[ed * H + h];
      } else {
        u = leaky(__fadd_rn(sd, __ldg(s_src + (int64_t)__ldg(src + ed) * H + h)));
        alpha[ed * H + h] = u;
      }
      m = u > m ? u : m;
    }
    for (int o = G >> 1; o > 0; o >>= 1) {
      const float v = __shfl_xor_sync(gm, m, o, G);
      m = v > m ? v : m;
    }
    float s = 0.f;
    for (int64_t k0 = b; k0 < e; k0 += G) {             // group-uniform trip count
      const int64_t k = k0 + sub;
      float x = 0.f;
      if (k < e) {
        const int64_t ed = edge_at(perm, k);
        x = expf(__fsub_rn(alpha[ed * H + h], m));
        alpha[ed * H + h] = x;
      }
      const int n = e - k0 < G ? (int)(e - k0) : G;
      for (int j = 0; j < n; ++j) s = __fadd_rn(s, __shfl_sync(gm, x, j, G));
    }
    for (int64_t k = b + sub; k < e; k += G) {
      const int64_t ed = edge_at(perm, k);
      alpha[ed * H + h] = __fdiv_rn(alpha[ed * H + h], s);
    }
  }
  __syncwarp(gm);                                      // the column pass reads alphas other lanes of the group wrote
  float* o = out + r * (int64_t)HC;
  if (VEC) {
    for (int d = sub * 4; d < HC; d += G * 4) {
      const int h0 = d / C, h1 = (d + 1) / C, h2 = (d + 2) / C, h3 = (d + 3) / C;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int64_t k0 = b; k0 < e; k0 += kGatUnroll) {
        float4 x[kGatUnroll], a[kGatUnroll];
#pragma unroll
        for (int q = 0; q < kGatUnroll; ++q) {
          if (k0 + q < e) {
            const int64_t ed = edge_at(perm, k0 + q);
            x[q] = __ldg(reinterpret_cast<const float4*>(h_src + (int64_t)__ldg(src + ed) * HC + d));
            const float* al = alpha + ed * H;
            a[q] = make_float4(al[h0], al[h1], al[h2], al[h3]);
          }
        }
#pragma unroll
        for (int q = 0; q < kGatUnroll; ++q) {
          if (k0 + q < e) {
            acc.x = __fadd_rn(acc.x, __fmul_rn(x[q].x, a[q].x)); acc.y = __fadd_rn(acc.y, __fmul_rn(x[q].y, a[q].y));
            acc.z = __fadd_rn(acc.z, __fmul_rn(x[q].z, a[q].z)); acc.w = __fadd_rn(acc.w, __fmul_rn(x[q].w, a[q].w));
          }
        }
      }
      *reinterpret_cast<float4*>(o + d) = acc;
    }
  } else {
    for (int d = sub; d < HC; d += G) {
      const int hd = d / C;
      float acc = 0.f;
      for (int64_t k0 = b; k0 < e; k0 += kGatUnroll) {
        float x[kGatUnroll], a[kGatUnroll];
#pragma unroll
        for (int q = 0; q < kGatUnroll; ++q) {
          if (k0 + q < e) {
            const int64_t ed = edge_at(perm, k0 + q);
            x[q] = __ldg(h_src + (int64_t)__ldg(src + ed) * HC + d);
            a[q] = alpha[ed * H + hd];
          }
        }
#pragma unroll
        for (int q = 0; q < kGatUnroll; ++q)
          if (k0 + q < e) acc = __fadd_rn(acc, __fmul_rn(x[q], a[q]));
      }
      o[d] = acc;
    }
  }
}

// G lanes per target row r (edges as in k_gat_fwd).  Per head, lanes over the segment's edges:
//   d_alpha[e] = <g[r, h-slice], h_src[src_e, h-slice]>        (a serial dot product over the C columns)
//   S          = sum_seg alpha * d_alpha                         (serial in edge order)
//   du[e]      = alpha * (d_alpha - S) * (u > 0 ? 1 : 0.2)       (to scratch, indexed by edge)
//   grad_s_dst[r, h] = sum_seg du                                (serial in edge order)
__global__ void __launch_bounds__(256) k_gat_bwd_dst(const float* __restrict__ g, const float* __restrict__ h_src,
                                                     const float* __restrict__ alpha, const float* __restrict__ s_dst,
                                                     const float* __restrict__ s_src, const int32_t* __restrict__ key,
                                                     const int32_t* __restrict__ perm, const int32_t* __restrict__ src, int64_t E,
                                                     int64_t n_dst, int H, int C, int G, float* __restrict__ du,
                                                     float* __restrict__ grad_s_dst) {
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t r = tid >> (31 - __clz(G));
  const int sub = (int)(tid & (G - 1));
  if (r >= n_dst) return;   // group-uniform
  const unsigned gm = group_mask(G);
  const int64_t b = key_lower_bound(key, E, r), e = key_lower_bound(key, E, r + 1);
  const int HC = H * C;   // < 2^31: checked by the launcher
  for (int h = 0; h < H; ++h) {
    const float* gr = g + r * (int64_t)HC + h * C;
    float S = 0.f;
    for (int64_t k0 = b; k0 < e; k0 += G) {
      const int64_t k = k0 + sub;
      float v = 0.f;
      if (k < e) {
        const int64_t ed = edge_at(perm, k);
        const float* xs = h_src + (int64_t)__ldg(src + ed) * HC + h * C;
        float da = 0.f;
        for (int c = 0; c < C; ++c) da = fmaf(__ldg(gr + c), __ldg(xs + c), da);
        du[ed * H + h] = da;
        v = __fmul_rn(__ldg(alpha + ed * H + h), da);
      }
      const int n = e - k0 < G ? (int)(e - k0) : G;
      for (int j = 0; j < n; ++j) S = __fadd_rn(S, __shfl_sync(gm, v, j, G));
    }
    const float sd = b < e ? __ldg(s_dst + r * H + h) : 0.f;
    float T = 0.f;
    for (int64_t k0 = b; k0 < e; k0 += G) {
      const int64_t k = k0 + sub;
      float v = 0.f;
      if (k < e) {
        const int64_t ed = edge_at(perm, k);
        const float z = __fadd_rn(sd, __ldg(s_src + (int64_t)__ldg(src + ed) * H + h));
        v = __fmul_rn(__fmul_rn(__ldg(alpha + ed * H + h), __fsub_rn(du[ed * H + h], S)), z > 0.f ? 1.f : 0.2f);
        du[ed * H + h] = v;
      }
      const int n = e - k0 < G ? (int)(e - k0) : G;
      for (int j = 0; j < n; ++j) T = __fadd_rn(T, __shfl_sync(gm, v, j, G));
    }
    if (sub == 0) grad_s_dst[r * H + h] = T;
  }
}

// G lanes per source row j; its edges are positions [lb(j), lb(j+1)) of the src-sorted order `skey` (sperm: position ->
// edge, ascending edge index within a source: the sort is stable; null when skey is already sorted).
// grad_h_src[j, col] = sum alpha[e, head(col)] * g[dst_e, col], grad_s_src[j, h] = sum du[e, h] (when grad_s_src is given),
// both in edge order; a source without edges gets zeros.  AGNN's backward runs it as a plain segmented weighted row sum,
// also over the dst order.
template <bool VEC>
__global__ void __launch_bounds__(256) k_gat_bwd_src(const float* __restrict__ g, const float* __restrict__ alpha,
                                                     const float* __restrict__ du, const int32_t* __restrict__ skey,
                                                     const int32_t* __restrict__ sperm, const int32_t* __restrict__ dst, int64_t E,
                                                     int64_t n_src, int H, int C, int G, float* __restrict__ grad_h_src,
                                                     float* __restrict__ grad_s_src) {
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t j = tid >> (31 - __clz(G));
  const int sub = (int)(tid & (G - 1));
  if (j >= n_src) return;
  const int64_t b = key_lower_bound(skey, E, j), e = key_lower_bound(skey, E, j + 1);
  const int HC = H * C;   // < 2^31: checked by the launcher
  float* o = grad_h_src + j * (int64_t)HC;
  if (VEC) {
    for (int d = sub * 4; d < HC; d += G * 4) {
      const int h0 = d / C, h1 = (d + 1) / C, h2 = (d + 2) / C, h3 = (d + 3) / C;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int64_t k0 = b; k0 < e; k0 += kGatUnroll) {
        float4 x[kGatUnroll], a[kGatUnroll];
#pragma unroll
        for (int q = 0; q < kGatUnroll; ++q) {
          if (k0 + q < e) {
            const int64_t ed = edge_at(sperm, k0 + q);
            x[q] = __ldg(reinterpret_cast<const float4*>(g + (int64_t)__ldg(dst + ed) * HC + d));
            const float* al = alpha + ed * H;
            a[q] = make_float4(__ldg(al + h0), __ldg(al + h1), __ldg(al + h2), __ldg(al + h3));
          }
        }
#pragma unroll
        for (int q = 0; q < kGatUnroll; ++q) {
          if (k0 + q < e) {
            acc.x = __fadd_rn(acc.x, __fmul_rn(a[q].x, x[q].x)); acc.y = __fadd_rn(acc.y, __fmul_rn(a[q].y, x[q].y));
            acc.z = __fadd_rn(acc.z, __fmul_rn(a[q].z, x[q].z)); acc.w = __fadd_rn(acc.w, __fmul_rn(a[q].w, x[q].w));
          }
        }
      }
      *reinterpret_cast<float4*>(o + d) = acc;
    }
  } else {
    for (int d = sub; d < HC; d += G) {
      const int hd = d / C;
      float acc = 0.f;
      for (int64_t k0 = b; k0 < e; k0 += kGatUnroll) {
        float x[kGatUnroll], a[kGatUnroll];
#pragma unroll
        for (int q = 0; q < kGatUnroll; ++q) {
          if (k0 + q < e) {
            const int64_t ed = edge_at(sperm, k0 + q);
            x[q] = __ldg(g + (int64_t)__ldg(dst + ed) * HC + d);
            a[q] = __ldg(alpha + ed * H + hd);
          }
        }
#pragma unroll
        for (int q = 0; q < kGatUnroll; ++q)
          if (k0 + q < e) acc = __fadd_rn(acc, __fmul_rn(a[q], x[q]));
      }
      o[d] = acc;
    }
  }
  if (!grad_s_src) return;
  for (int h = sub; h < H; h += G) {
    float acc = 0.f;
    for (int64_t k = b; k < e; ++k) acc = __fadd_rn(acc, __ldg(du + edge_at(sperm, k) * H + h));
    grad_s_src[j * H + h] = acc;
  }
}

// G lanes per edge e (a power of two <= 32): dot[e] = <a[ia_e, :], b[ib_e, :]> over dim columns, and scaled[e] =
// beta[0] * dot[e] when scaled is given.  The order is fixed: lane l accumulates, one __fmaf_rn at a time, the columns of
// its 4-column chunks l, l + G, l + 2G, ..., each chunk left to right; then a butterfly over the G lanes, xor distances G/2,
// ..., 1 (both lanes of a pair add the same two values, so every lane ends with the same bits).  VEC (dim % 4 == 0,
// 16-byte aligned rows) changes only the loads: the bits do not depend on the alignment.
template <bool VEC>
__global__ void __launch_bounds__(256) k_agnn_dot(const float* __restrict__ a, const float* __restrict__ b,
                                                  const int32_t* __restrict__ ia, const int32_t* __restrict__ ib, int64_t E,
                                                  int dim, int G, const float* __restrict__ beta, float* __restrict__ dot,
                                                  float* __restrict__ scaled) {
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t e = tid >> (31 - __clz(G));
  const int sub = (int)(tid & (G - 1));
  if (e >= E) return;   // group-uniform
  const unsigned gm = group_mask(G);
  const float* ar = a + (int64_t)__ldg(ia + e) * dim;
  const float* br = b + (int64_t)__ldg(ib + e) * dim;
  float acc = 0.f;
#pragma unroll 4
  for (int d = sub * 4; d < dim; d += G * 4) {
    if (VEC) {
      const float4 x = __ldg(reinterpret_cast<const float4*>(ar + d)), y = __ldg(reinterpret_cast<const float4*>(br + d));
      acc = __fmaf_rn(x.x, y.x, acc); acc = __fmaf_rn(x.y, y.y, acc);
      acc = __fmaf_rn(x.z, y.z, acc); acc = __fmaf_rn(x.w, y.w, acc);
    } else {
      const int n = dim - d < 4 ? dim - d : 4;
      for (int q = 0; q < n; ++q) acc = __fmaf_rn(__ldg(ar + d + q), __ldg(br + d + q), acc);
    }
  }
  for (int o = G >> 1; o > 0; o >>= 1) acc = __fadd_rn(acc, __shfl_xor_sync(gm, acc, o, G));
  if (sub == 0) {
    if (dot) dot[e] = acc;
    if (scaled) scaled[e] = __fmul_rn(__ldg(beta), acc);
  }
}

// G lanes per target row r (edges as in k_gat_fwd), H = 1.  dw holds d_alpha[e] = <grad_out[dst_e], x_src[src_e]> on entry.
// In edge order: S = sum alpha * d_alpha; du = alpha * (d_alpha - S); dw[e] = beta * du (the gradient of cos[e]);
// part[r] = sum du * cos (this target's share of grad_beta).
__global__ void __launch_bounds__(256) k_agnn_bwd_dst(const float* __restrict__ alpha, const float* __restrict__ cos,
                                                      const float* __restrict__ beta, const int32_t* __restrict__ key,
                                                      const int32_t* __restrict__ perm, int64_t E, int64_t n_dst, int G,
                                                      float* __restrict__ dw, float* __restrict__ part) {
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t r = tid >> (31 - __clz(G));
  const int sub = (int)(tid & (G - 1));
  if (r >= n_dst) return;   // group-uniform
  const unsigned gm = group_mask(G);
  const int64_t b = key_lower_bound(key, E, r), e = key_lower_bound(key, E, r + 1);
  float S = 0.f;
  for (int64_t k0 = b; k0 < e; k0 += G) {
    const int64_t k = k0 + sub;
    float v = 0.f;
    if (k < e) {
      const int64_t ed = edge_at(perm, k);
      v = __fmul_rn(__ldg(alpha + ed), dw[ed]);
    }
    const int n = e - k0 < G ? (int)(e - k0) : G;
    for (int j = 0; j < n; ++j) S = __fadd_rn(S, __shfl_sync(gm, v, j, G));
  }
  const float bt = __ldg(beta);
  float P = 0.f;
  for (int64_t k0 = b; k0 < e; k0 += G) {
    const int64_t k = k0 + sub;
    float v = 0.f;
    if (k < e) {
      const int64_t ed = edge_at(perm, k);
      const float du = __fmul_rn(__ldg(alpha + ed), __fsub_rn(dw[ed], S));
      dw[ed] = __fmul_rn(bt, du);
      v = __fmul_rn(du, __ldg(cos + ed));
    }
    const int n = e - k0 < G ? (int)(e - k0) : G;
    for (int j = 0; j < n; ++j) P = __fadd_rn(P, __shfl_sync(gm, v, j, G));
  }
  if (sub == 0) part[r] = P;
}

constexpr int kAgnnSumThreads = 1024;

// *out = sum of v[0, n) in a fixed order: thread t adds v[t], v[t + 1024], ... left to right, then a shared-memory tree
// (strides 512, ..., 1).  One block.
__global__ void __launch_bounds__(kAgnnSumThreads) k_agnn_sum(const float* __restrict__ v, int64_t n, float* __restrict__ out) {
  __shared__ float sh[kAgnnSumThreads];
  float acc = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += kAgnnSumThreads) acc = __fadd_rn(acc, __ldg(v + i));
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int s = kAgnnSumThreads / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) sh[threadIdx.x] = __fadd_rn(sh[threadIdx.x], sh[threadIdx.x + s]);
    __syncthreads();
  }
  if (threadIdx.x == 0) *out = sh[0];
}

// k_agnn_dot over E > 0 edges: dot[e] = <a[ia_e], b[ib_e]>, scaled[e] = beta * dot[e] (either output may be null)
static int agnn_dot(eu_ctx* c, const float* a, const float* b, const int32_t* ia, const int32_t* ib, int64_t E, int dim,
                    const float* beta, float* dot, float* scaled) {
  const bool vec = dim % 4 == 0 && aligned16(a) && aligned16(b);
  const int G = group_lanes(ceil_div(dim, 4));   // one lane per 4-column chunk, both paths: the same order
  const unsigned blocks = (unsigned)ceil_div(E * G, 256);
  if (vec) k_agnn_dot<true><<<blocks, 256, 0, c->stream>>>(a, b, ia, ib, E, dim, G, beta, dot, scaled);
  else k_agnn_dot<false><<<blocks, 256, 0, c->stream>>>(a, b, ia, ib, E, dim, G, beta, dot, scaled);
  EU_LAUNCHED();
  return EU_OK;
}

// out[r, :] = sum of w[e] * rows[idx_e, :] over the edges of segment r of the order o, in edge order (k_gat_bwd_src, H = 1)
int segmented_row_sum(eu_ctx* c, const float* rows, const float* w, const EdgeOrder& o, const int32_t* idx, int64_t E, int64_t n,
                      int dim, float* out) {
  const bool vec = dim % 4 == 0 && aligned16(rows) && aligned16(out);
  const int G = group_lanes(vec ? dim / 4 : dim);
  const unsigned blocks = (unsigned)ceil_div(n * G, 256);
  if (vec) k_gat_bwd_src<true><<<blocks, 256, 0, c->stream>>>(rows, w, nullptr, o.key, o.perm, idx, E, n, 1, dim, G, out, nullptr);
  else k_gat_bwd_src<false><<<blocks, 256, 0, c->stream>>>(rows, w, nullptr, o.key, o.perm, idx, E, n, 1, dim, G, out, nullptr);
  EU_LAUNCHED();
  return EU_OK;
}

}  // namespace eu

using namespace eu;

extern "C" {

int eu_gat_aggregate(eu_ctx* c, const float* h_src, const float* s_dst, const float* s_src, const int32_t* dst, const int32_t* src,
                     int64_t E, int64_t n_dst, int64_t n_src, int32_t heads, int32_t head_dim, float* out, float* alpha) {
  if (!c || heads < 1 || head_dim < 1 || E < 0 || n_dst < 0 || n_src < 0 || (E > 0 && (n_dst == 0 || n_src == 0)) ||
      (E > 0 && (!h_src || !s_dst || !s_src || !dst || !src)) || (n_dst > 0 && !out)) {
    set_error("eu_gat_aggregate: bad argument");
    return EU_ERR_INVALID;
  }
  if (E >= ((int64_t)1 << 31) || n_dst >= ((int64_t)1 << 31) || n_src >= ((int64_t)1 << 31) || (int64_t)heads * head_dim >= ((int64_t)1 << 31)) {
    set_error("eu_gat_aggregate: 2^31 or more edges, rows or columns are not supported");
    return EU_ERR_UNSUPPORTED;
  }
  EU_CUDA(cudaSetDevice(c->g->device));
  if (n_dst == 0) return EU_OK;
  cudaStream_t s = c->stream;
  const int64_t H = heads, HC = H * head_dim;
  // head: alpha scratch when the caller wants none
  TargetOrder t;
  int rc = order_targets(c, dst, E, n_dst, alpha ? 0 : a256(4 * (size_t)(E * H)), 0, nullptr, &t);
  if (rc) return rc;
  const EdgeOrder& ord = t.ord;
  float* al = alpha ? alpha : (float*)t.head;
  const bool vec = HC % 4 == 0 && aligned16(h_src) && aligned16(out);
  const int G = group_lanes(vec ? HC / 4 : HC);
  const unsigned blocks = (unsigned)ceil_div(n_dst * G, 256);
  EuProfScope ps(c, "gat_fwd", E);
  if (vec) k_gat_fwd<true, false><<<blocks, 256, 0, s>>>(h_src, s_dst, s_src, ord.key, ord.perm, src, E, n_dst, heads, head_dim, G, al, out);
  else k_gat_fwd<false, false><<<blocks, 256, 0, s>>>(h_src, s_dst, s_src, ord.key, ord.perm, src, E, n_dst, heads, head_dim, G, al, out);
  EU_LAUNCHED();
  return EU_OK;
}

int eu_gat_aggregate_backward(eu_ctx* c, const float* grad_out, const float* h_src, const float* alpha, const float* s_dst,
                              const float* s_src, const int32_t* dst, const int32_t* src, int64_t E, int64_t n_dst, int64_t n_src,
                              int32_t heads, int32_t head_dim, float* grad_h_src, float* grad_s_dst, float* grad_s_src) {
  if (!c || heads < 1 || head_dim < 1 || E < 0 || n_dst < 0 || n_src < 0 || (E > 0 && (n_dst == 0 || n_src == 0)) ||
      (E > 0 && (!grad_out || !h_src || !alpha || !s_dst || !s_src || !dst || !src)) || (n_dst > 0 && !grad_s_dst) ||
      (n_src > 0 && (!grad_h_src || !grad_s_src))) {
    set_error("eu_gat_aggregate_backward: bad argument");
    return EU_ERR_INVALID;
  }
  if (E >= ((int64_t)1 << 31) || n_dst >= ((int64_t)1 << 31) || n_src >= ((int64_t)1 << 31) || (int64_t)heads * head_dim >= ((int64_t)1 << 31)) {
    set_error("eu_gat_aggregate_backward: 2^31 or more edges, rows or columns are not supported");
    return EU_ERR_UNSUPPORTED;
  }
  EU_CUDA(cudaSetDevice(c->g->device));
  cudaStream_t s = c->stream;
  const int64_t H = heads, HC = H * head_dim;
  if (E == 0) {                                        // no edge: every gradient is zero
    if (n_dst > 0) EU_CUDA(cudaMemsetAsync(grad_s_dst, 0, 4 * (size_t)(n_dst * H), s));
    if (n_src > 0) {
      EU_CUDA(cudaMemsetAsync(grad_h_src, 0, 4 * (size_t)(n_src * HC), s));
      EU_CUDA(cudaMemsetAsync(grad_s_src, 0, 4 * (size_t)(n_src * H), s));
    }
    return EU_OK;
  }
  // head: du [E, H]; tail: the src order
  TargetOrder t;
  int rc = order_targets(c, dst, E, n_dst, a256(4 * (size_t)(E * H)), order_bytes(E, n_src), nullptr, &t);
  if (rc) return rc;
  float* du = (float*)t.head;
  const EdgeOrder& dord = t.ord;
  EdgeOrder sord;
  {
    const int G = 32;   // lanes over a segment's edges
    EuProfScope ps(c, "gat_bwd_dst", E);
    k_gat_bwd_dst<<<(unsigned)ceil_div(n_dst * G, 256), 256, 0, s>>>(grad_out, h_src, alpha, s_dst, s_src, dord.key, dord.perm, src, E,
                                                                    n_dst, heads, head_dim, G, du, grad_s_dst);
    EU_LAUNCHED();
  }
  if ((rc = order_by(c, src, E, n_src, t.tail, &sord))) return rc;
  {
    const bool vec = HC % 4 == 0 && aligned16(grad_out) && aligned16(grad_h_src);
    const int G = group_lanes(vec ? HC / 4 : HC);
    EuProfScope ps(c, "gat_bwd_src", E);
    if (vec) k_gat_bwd_src<true><<<(unsigned)ceil_div(n_src * G, 256), 256, 0, s>>>(grad_out, alpha, du, sord.key, sord.perm, dst, E, n_src,
                                                                                   heads, head_dim, G, grad_h_src, grad_s_src);
    else k_gat_bwd_src<false><<<(unsigned)ceil_div(n_src * G, 256), 256, 0, s>>>(grad_out, alpha, du, sord.key, sord.perm, dst, E, n_src,
                                                                                heads, head_dim, G, grad_h_src, grad_s_src);
    EU_LAUNCHED();
  }
  return EU_OK;
}

int eu_agnn_aggregate(eu_ctx* c, const float* x_src, const float* nrm_dst, const float* nrm_src, const float* beta,
                      const int32_t* dst, const int32_t* src, int64_t E, int64_t n_dst, int64_t n_src, int32_t dim, float* out,
                      float* alpha, float* cos) {
  if (!c || dim < 1 || E < 0 || n_dst < 0 || n_src < 0 || (E > 0 && (n_dst == 0 || n_src == 0)) ||
      (E > 0 && (!x_src || !nrm_dst || !nrm_src || !beta || !dst || !src)) || (n_dst > 0 && !out)) {
    set_error("eu_agnn_aggregate: bad argument");
    return EU_ERR_INVALID;
  }
  if (E >= ((int64_t)1 << 31) || n_dst >= ((int64_t)1 << 31) || n_src >= ((int64_t)1 << 31)) {
    set_error("eu_agnn_aggregate: 2^31 or more edges or rows are not supported");
    return EU_ERR_UNSUPPORTED;
  }
  EU_CUDA(cudaSetDevice(c->g->device));
  if (n_dst == 0) return EU_OK;
  cudaStream_t s = c->stream;
  // head: logit / exp / alpha scratch when the caller wants no alpha
  TargetOrder t;
  int rc = order_targets(c, dst, E, n_dst, alpha ? 0 : a256(4 * (size_t)E), 0, nullptr, &t);
  if (rc) return rc;
  const EdgeOrder& ord = t.ord;
  float* al = alpha ? alpha : (float*)t.head;
  if (E > 0) {
    EuProfScope ps(c, "agnn_cos", E);
    if ((rc = agnn_dot(c, nrm_dst, nrm_src, dst, src, E, dim, beta, cos, al))) return rc;   // cos and the logits beta * cos
  }
  const bool vec = dim % 4 == 0 && aligned16(x_src) && aligned16(out);
  // a warp per target whatever dim is: the softmax phase walks a segment G edges at a time, so at small dim the
  // column-phase width (GAT's group_lanes) would make a hub's softmax chains several times longer; the bits do not depend on G
  const int G = 32;
  const unsigned blocks = (unsigned)ceil_div(n_dst * G, 256);
  EuProfScope ps(c, "agnn_fwd", E);
  if (vec) k_gat_fwd<true, true><<<blocks, 256, 0, s>>>(x_src, nullptr, nullptr, ord.key, ord.perm, src, E, n_dst, 1, dim, G, al, out);
  else k_gat_fwd<false, true><<<blocks, 256, 0, s>>>(x_src, nullptr, nullptr, ord.key, ord.perm, src, E, n_dst, 1, dim, G, al, out);
  EU_LAUNCHED();
  return EU_OK;
}

int eu_agnn_aggregate_backward(eu_ctx* c, const float* grad_out, const float* x_src, const float* nrm_dst, const float* nrm_src,
                               const float* beta, const float* alpha, const float* cos, const int32_t* dst, const int32_t* src,
                               int64_t E, int64_t n_dst, int64_t n_src, int32_t dim, float* grad_x_src, float* grad_nrm_dst,
                               float* grad_nrm_src, float* grad_beta) {
  if (!c || dim < 1 || E < 0 || n_dst < 0 || n_src < 0 || (E > 0 && (n_dst == 0 || n_src == 0)) ||
      (E > 0 && (!grad_out || !x_src || !nrm_dst || !nrm_src || !beta || !alpha || !cos || !dst || !src)) ||
      (n_dst > 0 && !grad_nrm_dst) || (n_src > 0 && (!grad_x_src || !grad_nrm_src)) || !grad_beta) {
    set_error("eu_agnn_aggregate_backward: bad argument");
    return EU_ERR_INVALID;
  }
  if (E >= ((int64_t)1 << 31) || n_dst >= ((int64_t)1 << 31) || n_src >= ((int64_t)1 << 31)) {
    set_error("eu_agnn_aggregate_backward: 2^31 or more edges or rows are not supported");
    return EU_ERR_UNSUPPORTED;
  }
  EU_CUDA(cudaSetDevice(c->g->device));
  cudaStream_t s = c->stream;
  if (E == 0) {                                        // no edge: every gradient is zero
    if (n_dst > 0) EU_CUDA(cudaMemsetAsync(grad_nrm_dst, 0, 4 * (size_t)(n_dst * dim), s));
    if (n_src > 0) {
      EU_CUDA(cudaMemsetAsync(grad_x_src, 0, 4 * (size_t)(n_src * dim), s));
      EU_CUDA(cudaMemsetAsync(grad_nrm_src, 0, 4 * (size_t)(n_src * dim), s));
    }
    EU_CUDA(cudaMemsetAsync(grad_beta, 0, sizeof(float), s));
    return EU_OK;
  }
  // head: d_alpha, then beta * du [E] | per-target partials of grad_beta [n_dst]; tail: the src order
  TargetOrder t;
  int rc = order_targets(c, dst, E, n_dst, a256(4 * (size_t)E) + a256(4 * (size_t)n_dst), order_bytes(E, n_src), nullptr, &t);
  if (rc) return rc;
  float* dw = (float*)t.head;
  float* part = (float*)(t.head + a256(4 * (size_t)E));
  const EdgeOrder& dord = t.ord;
  EdgeOrder sord;
  {
    EuProfScope ps(c, "agnn_bwd_dalpha", E);
    if ((rc = agnn_dot(c, grad_out, x_src, dst, src, E, dim, nullptr, dw, nullptr))) return rc;
  }
  {
    const int G = 32;   // lanes over a segment's edges
    EuProfScope ps(c, "agnn_bwd_dst", E);
    k_agnn_bwd_dst<<<(unsigned)ceil_div(n_dst * G, 256), 256, 0, s>>>(alpha, cos, beta, dord.key, dord.perm, E, n_dst, G, dw, part);
    EU_LAUNCHED();
  }
  {
    EuProfScope ps(c, "agnn_bwd_nrm_dst", E);
    if ((rc = segmented_row_sum(c, nrm_src, dw, dord, src, E, n_dst, dim, grad_nrm_dst))) return rc;
  }
  {
    EuProfScope ps(c, "agnn_bwd_beta", n_dst);
    k_agnn_sum<<<1, kAgnnSumThreads, 0, s>>>(part, n_dst, grad_beta);
    EU_LAUNCHED();
  }
  if ((rc = order_by(c, src, E, n_src, t.tail, &sord))) return rc;
  {
    EuProfScope ps(c, "agnn_bwd_src", E);
    if ((rc = segmented_row_sum(c, grad_out, alpha, sord, dst, E, n_src, dim, grad_x_src))) return rc;
    if ((rc = segmented_row_sum(c, nrm_dst, dw, sord, dst, E, n_src, dim, grad_nrm_src))) return rc;
  }
  return EU_OK;
}

}  // extern "C"
