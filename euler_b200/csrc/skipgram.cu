// The unsupervised skip-gram step of DeepWalk, node2vec and LINE, forward and backward: id embeddings, dot products with a
// positive and K negative context rows, the sigmoid cross-entropy mean and the rank of the positive among the negatives.
//
// Reference semantics (file:line in the upstream alibaba/euler tree):
//   UnsuperviseModel.__call__   tf_euler/python/mp_utils/base.py:50-91 (also solution/base_unsupervise.py)
//   PosNegLogits                tf_euler/python/solution/logits.py (matmul of the target row with the context rows)
//   xent_loss                   tf_euler/python/solution/losses.py (sigmoid_cross_entropy_with_logits, one reduce_mean over
//                               the positive and negative terms together)
//   mrr / hitk / mr             tf_euler/python/utils/metrics.py (top_k over concat([neg, pos], 2); the rank of the LAST entry)
//
// Pair row b has the target row t = target[src_b] and J = P + K context ids: pos[b, 0 .. P-1], then negs[b, 0 .. K-1].
//   logits[b, j] = <t, context[ctx_bj]>, in k_agnn_dot's fixed order: lane l of a group of G lanes (G = the power of two >=
//     ceil(dim / 4), at most 32) accumulates with __fmaf_rn from +0 the columns of its 4-column chunks l, l + G, l + 2G, ...,
//     each chunk left to right; then a butterfly over the G lanes, xor distances G/2 .. 1.  G depends on dim only.
//   rank[b] = #{j != P-1 : logits[b, j] >= logits[b, P-1]}: TF's top_k is stable (ties go to the lower index) and the last
//     positive is the last entry of concat([neg, pos], 2), so it ranks behind every entry that is not smaller.
//   loss = mean over the B J logits of max(x, 0) - x z + log1p(exp(-|x|)) (z = 1 for j < P): each term in f32, each row's
//     terms added in j order in f64, the rows added in a fixed order in f64 (k_f64_mean), one division, rounded to f32.
// An id outside [0, n_rows) is read as row 0 and flagged; the call returns EU_ERR_INVALID after its one synchronisation.
// Tables are f32 or bf16 (T, an eu_feat_dtype): a bf16 element is widened exactly to f32 as it is read and every other step
// is the f32 one, so a bf16 call gives the f32 call's bits on the widened tables.  The 4-wide loads (VEC) need dim % 4 == 0
// and each table aligned to four elements (16 bytes of f32, 8 of bf16); the scalar path sums in the same order.
//
// Backward, with g the upstream gradient (a device scalar) and N = B J: gN = g / fl(N) once, and per logit
//   c_bj = -gN / (1 + exp(x))  (j < P: (sigmoid(x) - 1) gN)      c_bj = gN / (1 + exp(-x))  (j >= P: sigmoid(x) gN).
// The gradients go to the tables through segment.cuh's id-table gradient path, the one the embedding and KG backward passes
// share: key lists sorted stably by row (plan_rows) and summed per distinct row in fixed chunks of kSegChunk entries
// (sum_distinct_rows), no atomics:
//   the src entries:     entry b has key src_b and value gt_b = sum over j of c_bj context[ctx_bj] (fma from +0, j order)
//   the context entries: entry (b, j) has key ctx_bj and value c_bj target[src_b], computed while it is summed
// Each chunk adds its entries' values left to right from +0, as acc = fma(w, row, acc) with w = 1 for a src entry (so a plain
// add) and w = c_bj for a context entry; a row of several chunks adds the chunk sums in chunk order from +0.  Separate
// tables: one list of the B src entries for the target table, one of the B J context entries for the context table.  One
// shared table: one list, the src entries first, then the context entries in (b, j) order.  Index scratch is O(B J) however
// many rows the tables have; a hub negative is spread over chunks of 256 entries.
#include "segment.cuh"

namespace eu {

constexpr int kSgRows = 4;     // context rows in flight per lane in the dot and target-gradient loops
constexpr int kSgRegs = 4;     // target chunks kept in registers per lane (dim <= 512 with 32 lanes)

// acc += the dot of the columns [d, min(d + 4, dim)) of a and b, one __fmaf_rn per column, left to right
__device__ __forceinline__ float sg_fma4(float4 a, float4 b, float acc, int n) {
  acc = __fmaf_rn(a.x, b.x, acc);
  if (n > 1) acc = __fmaf_rn(a.y, b.y, acc);
  if (n > 2) acc = __fmaf_rn(a.z, b.z, acc);
  if (n > 3) acc = __fmaf_rn(a.w, b.w, acc);
  return acc;
}

// the context id of entry (b, j): pos[b, j] for j < P, negs[b, j - P] after
__device__ __forceinline__ int64_t sg_ctx_id(const int64_t* __restrict__ pos, const int64_t* __restrict__ negs, int64_t b, int P,
                                             int K, int j) {
  return j < P ? __ldg(pos + b * P + j) : __ldg(negs + b * K + (j - P));
}

// one f32 term of sigmoid_cross_entropy_with_logits (z = 1 for a positive)
__device__ __forceinline__ float sg_xent(float x, bool positive) {
  float r = fmaxf(x, 0.f);
  if (positive) r = __fsub_rn(r, x);
  return __fadd_rn(r, log1pf(expf(-fabsf(x))));
}

// G lanes per pair row b: the target row's first kSgRegs chunks of this lane in registers, kSgRows context rows in flight.
// Lane 0 writes the logits; after them the group counts the rank and lane 0 adds the row's loss terms.
template <bool VEC, typename T>
__global__ void __launch_bounds__(256) k_sg_fwd(const int64_t* __restrict__ src, const int64_t* __restrict__ pos,
                                                const int64_t* __restrict__ negs, int64_t B, int P, int K,
                                                const T* __restrict__ target, const T* __restrict__ context, int64_t n_rows,
                                                int dim, int G, float* logits, int32_t* __restrict__ rank,
                                                double* __restrict__ rowloss, int* bad) {
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t b = tid >> (31 - __clz(G));
  const int sub = (int)(tid & (G - 1));
  if (b >= B) return;   // group-uniform
  const unsigned gm = group_mask(G);
  const int J = P + K;
  const int nck = ((dim + 3) / 4 + G - 1) / G;   // chunks of the lane with the most
  const T* tr = target + row_of(__ldg(src + b), n_rows, bad) * dim;
  float4 treg[kSgRegs];
#pragma unroll
  for (int i = 0; i < kSgRegs; ++i) {
    const int d = (sub + i * G) * 4;
    treg[i] = i < nck && d < dim ? row_load4<VEC>(tr, d, dim) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  float* lrow = logits + b * J;
  for (int j0 = 0; j0 < J; j0 += kSgRows) {
    const T* cr[kSgRows];
#pragma unroll
    for (int u = 0; u < kSgRows; ++u)
      cr[u] = j0 + u < J ? context + row_of(sg_ctx_id(pos, negs, b, P, K, j0 + u), n_rows, bad) * dim : nullptr;
    float acc[kSgRows];
#pragma unroll
    for (int u = 0; u < kSgRows; ++u) acc[u] = 0.f;
    for (int i = 0; i < nck; ++i) {
      const int d = (sub + i * G) * 4;
      if (d >= dim) break;
      float4 t;
      if (i < kSgRegs) {
#pragma unroll
        for (int r = 0; r < kSgRegs; ++r)
          if (r == i) t = treg[r];
      } else {
        t = row_load4<VEC>(tr, d, dim);
      }
      const int n = dim - d < 4 ? dim - d : 4;
      float4 x[kSgRows];
#pragma unroll
      for (int u = 0; u < kSgRows; ++u)
        if (cr[u]) x[u] = row_load4<VEC>(cr[u], d, dim);
#pragma unroll
      for (int u = 0; u < kSgRows; ++u)
        if (cr[u]) acc[u] = sg_fma4(t, x[u], acc[u], n);
    }
#pragma unroll
    for (int u = 0; u < kSgRows; ++u) {
      for (int o = G >> 1; o > 0; o >>= 1) acc[u] = __fadd_rn(acc[u], __shfl_xor_sync(gm, acc[u], o, G));
      if (sub == 0 && j0 + u < J) lrow[j0 + u] = acc[u];
    }
  }
  __syncwarp(gm);   // lane 0's logits are visible to its group
  const float xl = lrow[P - 1];
  int cnt = 0;
  for (int j = sub; j < J; j += G) cnt += j != P - 1 && lrow[j] >= xl;
  for (int o = G >> 1; o > 0; o >>= 1) cnt += __shfl_xor_sync(gm, cnt, o, G);
  if (sub != 0) return;
  rank[b] = cnt;
  double s = 0.0;
  for (int j = 0; j < J; ++j) s += (double)sg_xent(lrow[j], j < P);
  rowloss[b] = s;
}

// coef[b J + j] = c_bj (see the top of the file); one thread per logit
__global__ void k_sg_coef(const float* __restrict__ logits, const float* __restrict__ grad_loss, int64_t N, int P, int J,
                          float* __restrict__ coef) {
  const float gN = __fdiv_rn(__ldg(grad_loss), (float)N);
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < N; e += (int64_t)gridDim.x * blockDim.x) {
    const float x = __ldg(logits + e);
    coef[e] = (int)(e % J) < P ? __fdiv_rn(-gN, __fadd_rn(1.f, expf(x))) : __fdiv_rn(gN, __fadd_rn(1.f, expf(-x)));
  }
}

// The int32 keys of the entries: key[b] = src_b for b < n_src (0 or B), then key[n_src + b J + j] = ctx_bj.  An id outside
// [0, n_rows) becomes row 0 and sets *bad.
__global__ void k_sg_keys(const int64_t* __restrict__ src, const int64_t* __restrict__ pos, const int64_t* __restrict__ negs,
                          int64_t B, int P, int K, int64_t n_src, bool ctx_entries, int64_t n_rows, int32_t* __restrict__ key,
                          int* bad) {
  const int J = P + K;
  const int64_t E = n_src + (ctx_entries ? B * J : 0);
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < E; e += (int64_t)gridDim.x * blockDim.x) {
    int64_t v;
    if (e < n_src) {
      v = __ldg(src + e);
    } else {
      const int64_t t = e - n_src, b = t / J;
      v = sg_ctx_id(pos, negs, b, P, K, (int)(t - b * J));
    }
    key[e] = (int32_t)row_of(v, n_rows, bad);
  }
}

// G lanes per pair row b: gt[b, :] = sum over j of coef[b, j] * context[ctx_bj, :], fma from +0 in j order
template <bool VEC, typename T>
__global__ void __launch_bounds__(256) k_sg_target_rows(const int64_t* __restrict__ pos, const int64_t* __restrict__ negs, int64_t B,
                                                        int P, int K, const float* __restrict__ coef,
                                                        const T* __restrict__ context, int64_t n_rows, int dim, int G,
                                                        float* __restrict__ gt) {
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t b = tid >> (31 - __clz(G));
  const int sub = (int)(tid & (G - 1));
  if (b >= B) return;
  const int J = P + K;
  int ignored = 0;   // the keys pass flags bad ids
  for (int d = sub * 4; d < dim; d += G * 4) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j0 = 0; j0 < J; j0 += kSgRows) {
      float4 x[kSgRows];
      float w[kSgRows];
#pragma unroll
      for (int u = 0; u < kSgRows; ++u) {
        if (j0 + u < J) {
          x[u] = row_load4<VEC>(context + row_of(sg_ctx_id(pos, negs, b, P, K, j0 + u), n_rows, &ignored) * dim, d, dim);
          w[u] = __ldg(coef + b * J + j0 + u);
        }
      }
#pragma unroll
      for (int u = 0; u < kSgRows; ++u) {
        if (j0 + u < J) {
          acc.x = __fmaf_rn(w[u], x[u].x, acc.x); acc.y = __fmaf_rn(w[u], x[u].y, acc.y);
          acc.z = __fmaf_rn(w[u], x[u].z, acc.z); acc.w = __fmaf_rn(w[u], x[u].w, acc.w);
        }
      }
    }
    float* o = gt + b * dim + d;
    if (VEC) {
      *reinterpret_cast<float4*>(o) = acc;
    } else {
      o[0] = acc.x;
      if (d + 1 < dim) o[1] = acc.y;
      if (d + 2 < dim) o[2] = acc.z;
      if (d + 3 < dim) o[3] = acc.w;
    }
  }
}

static int sg_check(eu_ctx* c, const int64_t* src, const int64_t* pos, const int64_t* negs, int64_t B, int32_t P, int32_t K,
                    const void* target, const void* context, int64_t n_rows, int32_t dim, int32_t dtype, const char* who) {
  if (!c || B < 0 || P < 1 || K < 0 || n_rows < 1 || dim < 1 || !target || !context ||
      (B > 0 && (!src || !pos || (K > 0 && !negs))) || !dtype_ok(dtype)) {
    set_error("%s: bad argument (B >= 0, P >= 1, K >= 0, n_rows and dim >= 1, tables and ids given, a known table dtype)", who);
    return EU_ERR_INVALID;
  }
  if (n_rows >= ((int64_t)1 << 31) || !entries_fit(B * ((int64_t)P + K + 1))) {   // the longest list: one shared table's
    set_error("%s: 2^31 or more table rows, or B (P + K + 1) entries with their chunks, are not supported", who);
    return EU_ERR_UNSUPPORTED;
  }
  return EU_OK;
}

// The backward pass both output forms share.  shared: one list into the target outputs.  sparse: the COO of
// each list, its distinct count read back; dense: the gradient tables, zeroed first.  One synchronisation at the end.
static int sg_backward(eu_ctx* c, const float* grad_loss, const int64_t* src, const int64_t* pos, const int64_t* negs, int64_t B,
                       int32_t P, int32_t K, const void* target, const void* context, int64_t n_rows, int32_t dim, int32_t dtype,
                       const float* logits, bool shared, bool sparse, float* out_t, float* out_c, int64_t* rows_t,
                       int64_t* rows_c, int64_t* n_t, int64_t* n_c, const char* who) {
  cudaStream_t s = c->stream;
  EU_CUDA(cudaSetDevice(c->g->device));
  if (!sparse) {
    EU_CUDA(cudaMemsetAsync(out_t, 0, 4 * (size_t)n_rows * dim, s));
    if (!shared) EU_CUDA(cudaMemsetAsync(out_c, 0, 4 * (size_t)n_rows * dim, s));
  }
  if (n_t) *n_t = 0;
  if (n_c) *n_c = 0;
  const int J = P + K;
  const int64_t N = B * J;
  if (B == 0) return EU_OK;
  RowList Lt, Lc;   // the target table's entries (shared: every entry) and the context table's
  Lt.E = shared ? B + N : B;
  Lc.E = shared ? 0 : N;
  Lt.n_rows = Lc.n_rows = n_rows;
  // flag and the two distinct counts (256 B) | coef [N] | gt [B, dim] | list t: keys, plan | list c: keys, plan
  const size_t o_coef = 256, o_gt = o_coef + a256(4 * (size_t)N), o_kt = o_gt + a256(4 * (size_t)B * dim);
  const size_t o_pt = o_kt + a256(4 * (size_t)Lt.E), o_kc = o_pt + row_plan_bytes(Lt.E, n_rows, dim);
  const size_t o_pc = o_kc + a256(4 * (size_t)Lc.E), total = o_pc + row_plan_bytes(Lc.E, n_rows, dim);
  int rc = ctx_misc(c, (int64_t)total);
  if (rc) return rc;
  char* m = (char*)c->d_misc;
  int* bad = (int*)m;
  float* coef = (float*)(m + o_coef);
  float* gt = (float*)(m + o_gt);
  Lt.key = (int32_t*)(m + o_kt);
  Lc.key = (int32_t*)(m + o_kc);
  EU_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), s));
  {
    EuProfScope ps(c, "skipgram_bwd_order", Lt.E + Lc.E);
    k_sg_keys<<<stride_grid(Lt.E), 256, 0, s>>>(src, pos, negs, B, P, K, B, shared, n_rows, Lt.key, bad);
    EU_LAUNCHED();
    if ((rc = plan_rows(c, m + o_pt, &Lt))) return rc;
    if (Lc.E) {
      k_sg_keys<<<stride_grid(Lc.E), 256, 0, s>>>(src, pos, negs, B, P, K, 0, true, n_rows, Lc.key, bad);
      EU_LAUNCHED();
      if ((rc = plan_rows(c, m + o_pc, &Lc))) return rc;
    }
  }
  EuProfScope ps(c, "skipgram_bwd_sums", Lt.E + Lc.E);
  k_sg_coef<<<stride_grid(N), 256, 0, s>>>(logits, grad_loss, N, P, J, coef);
  EU_LAUNCHED();
  const bool vec = dim % 4 == 0 && aligned4_elems(context, dtype) && aligned16(gt);
  const int G = group_lanes(ceil_div(dim, 4));
  const unsigned blocks = (unsigned)ceil_div(B * G, 256);
  with_dtype(dtype, [&](auto t) {
    using T = typename decltype(t)::type;
    auto k = vec ? k_sg_target_rows<true, T> : k_sg_target_rows<false, T>;
    k<<<blocks, 256, 0, s>>>(pos, negs, B, P, K, coef, static_cast<const T*>(context), n_rows, dim, G, gt);
  });
  EU_LAUNCHED();
  RowEntries R;   // the target list: the B src entries (gt rows), then the context entries; the context list: those only
  R.n_src = B;
  R.gt = gt;
  R.J = J;
  R.coef = coef;
  R.src = src;
  R.target = target;
  R.target_dtype = dtype;
  R.n_rows = n_rows;
  if ((rc = sum_distinct_rows(c, R, Lt, dim, !sparse, out_t, rows_t))) return rc;
  R.n_src = 0;
  if ((rc = sum_distinct_rows(c, R, Lc, dim, !sparse, out_c, rows_c))) return rc;
  bool h_bad = false;
  const int32_t* nd[2] = {Lt.P.nd, Lc.P.nd};
  int64_t n[2] = {0, 0};
  if ((rc = read_back(c, bad, &h_bad, sparse ? 2 : 0, nd, n))) return rc;
  if (h_bad) {
    set_error("%s: an id lies outside the table's rows [0, %lld)", who, (long long)n_rows);
    return EU_ERR_INVALID;
  }
  if (n_t) *n_t = n[0];
  if (n_c) *n_c = n[1];
  return EU_OK;
}

// the forward pass of both table types
static int sg_forward(eu_ctx* c, const int64_t* src, const int64_t* pos, const int64_t* negs, int64_t B, int32_t P, int32_t K,
                      const void* target, const void* context, int64_t n_rows, int32_t dim, int32_t dtype, float* logits,
                      int32_t* rank, float* loss, const char* who) {
  int rc = sg_check(c, src, pos, negs, B, P, K, target, context, n_rows, dim, dtype, who);
  if (rc) return rc;
  if (!loss || (B > 0 && (!logits || !rank))) {
    set_error("%s: bad argument (logits, rank and loss are required)", who);
    return EU_ERR_INVALID;
  }
  EU_CUDA(cudaSetDevice(c->g->device));
  EuProfScope ps(c, "skipgram_fwd", B);
  bool h_bad = false;
  rc = mean_loss(c, B, B * (int64_t)(P + K), loss, &h_bad, [&](int* bad, double* rowloss) -> int {
    const bool vec = dim % 4 == 0 && aligned4_elems(target, dtype) && aligned4_elems(context, dtype);
    const int G = group_lanes(ceil_div(dim, 4));   // one lane per 4-column chunk, both paths: the same order
    const unsigned blocks = (unsigned)ceil_div(B * G, 256);
    with_dtype(dtype, [&](auto t) {
      using T = typename decltype(t)::type;
      auto k = vec ? k_sg_fwd<true, T> : k_sg_fwd<false, T>;
      k<<<blocks, 256, 0, c->stream>>>(src, pos, negs, B, P, K, static_cast<const T*>(target), static_cast<const T*>(context), n_rows,
                                       dim, G, logits, rank, rowloss, bad);
    });
    EU_LAUNCHED();
    return EU_OK;
  });
  if (rc) return rc;
  if (h_bad) {
    set_error("%s: an id lies outside the table's rows [0, %lld)", who, (long long)n_rows);
    return EU_ERR_INVALID;
  }
  return EU_OK;
}

static int sg_backward_dense(eu_ctx* c, const float* grad_loss, const int64_t* src, const int64_t* pos, const int64_t* negs,
                             int64_t B, int32_t P, int32_t K, const void* target, const void* context, int64_t n_rows,
                             int32_t dim, int32_t dtype, const float* logits, float* grad_target, float* grad_context,
                             const char* who) {
  int rc = sg_check(c, src, pos, negs, B, P, K, target, context, n_rows, dim, dtype, who);
  if (rc) return rc;
  if (!grad_loss || !grad_target || !grad_context || (B > 0 && !logits)) {
    set_error("%s: bad argument (grad_loss, logits and both gradient tables are required)", who);
    return EU_ERR_INVALID;
  }
  return sg_backward(c, grad_loss, src, pos, negs, B, P, K, target, context, n_rows, dim, dtype, logits, grad_target == grad_context,
                     false, grad_target, grad_context, nullptr, nullptr, nullptr, nullptr, who);
}

static int sg_backward_sparse(eu_ctx* c, const float* grad_loss, const int64_t* src, const int64_t* pos, const int64_t* negs,
                              int64_t B, int32_t P, int32_t K, const void* target, const void* context, int64_t n_rows,
                              int32_t dim, int32_t dtype, const float* logits, int64_t* rows_target, float* values_target,
                              int64_t* n_target, int64_t* rows_context, float* values_context, int64_t* n_context, const char* who) {
  int rc = sg_check(c, src, pos, negs, B, P, K, target, context, n_rows, dim, dtype, who);
  if (rc) return rc;
  const bool shared = !rows_context;
  if (!grad_loss || !n_target || (B > 0 && (!logits || !rows_target || !values_target)) ||
      (!shared && (!n_context || (B > 0 && !values_context)))) {
    set_error("%s: bad argument", who);
    return EU_ERR_INVALID;
  }
  return sg_backward(c, grad_loss, src, pos, negs, B, P, K, target, context, n_rows, dim, dtype, logits, shared, true, values_target,
                     values_context, rows_target, rows_context, n_target, n_context, who);
}

}  // namespace eu

using namespace eu;

extern "C" {

int eu_skipgram_loss(eu_ctx* c, const int64_t* src, const int64_t* pos, const int64_t* negs, int64_t B, int32_t P, int32_t K,
                     const float* target, const float* context, int64_t n_rows, int32_t dim, float* logits, int32_t* rank,
                     float* loss) {
  return sg_forward(c, src, pos, negs, B, P, K, target, context, n_rows, dim, EU_FEAT_F32, logits, rank, loss, "eu_skipgram_loss");
}

int eu_skipgram_loss_dtype(eu_ctx* c, const int64_t* src, const int64_t* pos, const int64_t* negs, int64_t B, int32_t P, int32_t K,
                           const void* target, const void* context, int64_t n_rows, int32_t dim, int32_t table_dtype,
                           float* logits, int32_t* rank, float* loss) {
  return sg_forward(c, src, pos, negs, B, P, K, target, context, n_rows, dim, table_dtype, logits, rank, loss,
                    "eu_skipgram_loss_dtype");
}

int eu_skipgram_loss_backward(eu_ctx* c, const float* grad_loss, const int64_t* src, const int64_t* pos, const int64_t* negs,
                              int64_t B, int32_t P, int32_t K, const float* target, const float* context, int64_t n_rows,
                              int32_t dim, const float* logits, float* grad_target, float* grad_context) {
  return sg_backward_dense(c, grad_loss, src, pos, negs, B, P, K, target, context, n_rows, dim, EU_FEAT_F32, logits, grad_target,
                           grad_context, "eu_skipgram_loss_backward");
}

int eu_skipgram_loss_backward_dtype(eu_ctx* c, const float* grad_loss, const int64_t* src, const int64_t* pos, const int64_t* negs,
                                    int64_t B, int32_t P, int32_t K, const void* target, const void* context, int64_t n_rows,
                                    int32_t dim, int32_t table_dtype, const float* logits, float* grad_target,
                                    float* grad_context) {
  return sg_backward_dense(c, grad_loss, src, pos, negs, B, P, K, target, context, n_rows, dim, table_dtype, logits, grad_target,
                           grad_context, "eu_skipgram_loss_backward_dtype");
}

int eu_skipgram_loss_backward_sparse(eu_ctx* c, const float* grad_loss, const int64_t* src, const int64_t* pos, const int64_t* negs,
                                     int64_t B, int32_t P, int32_t K, const float* target, const float* context, int64_t n_rows,
                                     int32_t dim, const float* logits, int64_t* rows_target, float* values_target,
                                     int64_t* n_target, int64_t* rows_context, float* values_context, int64_t* n_context) {
  return sg_backward_sparse(c, grad_loss, src, pos, negs, B, P, K, target, context, n_rows, dim, EU_FEAT_F32, logits, rows_target,
                            values_target, n_target, rows_context, values_context, n_context, "eu_skipgram_loss_backward_sparse");
}

int eu_skipgram_loss_backward_sparse_dtype(eu_ctx* c, const float* grad_loss, const int64_t* src, const int64_t* pos,
                                           const int64_t* negs, int64_t B, int32_t P, int32_t K, const void* target,
                                           const void* context, int64_t n_rows, int32_t dim, int32_t table_dtype,
                                           const float* logits, int64_t* rows_target, float* values_target, int64_t* n_target,
                                           int64_t* rows_context, float* values_context, int64_t* n_context) {
  return sg_backward_sparse(c, grad_loss, src, pos, negs, B, P, K, target, context, n_rows, dim, table_dtype, logits, rows_target,
                            values_target, n_target, rows_context, values_context, n_context,
                            "eu_skipgram_loss_backward_sparse_dtype");
}

}  // extern "C"
