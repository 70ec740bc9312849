// The knowledge-graph embedding step of TransE, TransH, TransR, TransD and DistMult, forward and backward: the mapped id rows
// of each sampled triple and its corrupted triples, their scores, the margin loss and the rank of the true triple.
//
// Reference semantics (file:line in the upstream alibaba/euler tree):
//   TransX.call / calculate_energy   examples/TransX/transX.py:104-162 (tile, scores, front then tail negatives)
//   TransE / H / R / D               examples/TransX/trans{E,H,R,D}.py (row maps and loss_fn)
//   DistMult                         examples/distmult/distmult.py:60-79
//   _mrr / _mr / _hit10              examples/TransX/transX.py:81-100 (top_k over concat([neg, pos], 2))
//
// Triple b has ids src_b, dst_b, rel_b and K negatives neg[b, k].  n(x) = x / sqrt(max(sum x^2, 1e-12)) (TF's l2_normalize; the
// reciprocal square root correctly rounded, __frsqrt_rn).  With r = n(relation[rel_b]) the entity row e of an id maps to
//   TransE, DistMult  y = n(e)
//   TransH            y = e - (e . h) h,  h = n(hyper[rel_b])                  (not normalised)
//   TransR            y = n(e M),         M = transfer[rel_b] as [ent_dim, rel_dim], e not normalised
//   TransD            y = n(e + (e . et) rt),  et = entity_transfer[id], rt = relation_transfer[rel_b]
// and a triple (a, r, c) scores -||(a + r) - c||_1 or _2 (TransX) or sum a (r c) (DistMult).  scores[b] = the true triple
// (s, r, d), then with corrupt 'front' the K triples (neg_k, r, d), with 'tail' (s, r, neg_k), with 'both' the front K then the
// tail K: W = 1 + C K scores per triple.
//
// Every reduction over columns is a warp's: lane l holds the 4-column chunks l, l + 32, ... (kKgCh of them), accumulates its
// columns left to right from +0, then a butterfly over xor distances 16 .. 1.  The order depends on the dim only, and float4
// and scalar loads feed the same operations.  A block maps the triple's own rows once (warps 0 and 1), stages TransR's M in
// shared memory, and scores a tile of kKgTile negatives, a warp per negative; no [B, K, dim] rows exist.
//
// The row pass (k_kg_rows, one block per triple) adds the C K negative scores: thread t adds entries t, t + 256, ... left to
// right in f32, then a shared-memory tree over strides 128 .. 1; mean = sum / (C K) (one division), h = (margin + mean) - pos,
// rowloss = max(h, 0), rank = #{j : neg_j >= pos} (TF's stable top_k ranks the last entry behind every entry not smaller).  The
// row losses are added in f64 by k_f64_mean and divided once by B.
//
// Backward (grad_loss g read on the device): the row pass recomputes h from the saved scores; a row is active when h >= 0 (TF's
// maximum sends the gradient to its first argument on equality): cp = -g / B, cn = (g / B) / (C K), else both 0.  The score
// gradients are c (-sign(x)) (L1; sign(0) = 0), c (-x / ||x||) (L2; 0 at x = 0, where TF gives NaN), and for DistMult the
// products of the other two rows.  n's gradient is inv (gy - (y . gy) y) when sum x^2 >= 1e-12, else inv gy.  Passes:
//   k_kg_bwd_neg     per negative (b, k): its front and tail terms summed into one gradient of y, chained to the entity row
//                    (and TransD's entity_transfer row): one entry each; F[b, k] / T[b, k] keep its front / tail terms for the
//                    triple's own rows, U[b, 2 + k] the gradient that reaches the relation-side auxiliary row.
//   k_kg_bwd_triple  per triple: F and T summed over k in order from +0 in f64, rounded once; the src and dst entries and
//                    the relation entry.
//   k_kg_bwd_raux    per triple: hyper (TransH), relation_transfer (TransD) or M (TransR) summed over src, dst, negatives in
//                    that order in f64, rounded once: one relation-side entry per triple.  (These sums run over K + 2 terms,
//                    4 099 at K = 4 097, where f32 would lose about 1e-5 of the largest entry.)
// The entries are then summed per distinct table row by segment.cuh's id-table gradient path, the one the embedding and
// skip-gram backward passes share (plan_rows: stable order by row; sum_distinct_rows: 256-entry chunks left to right, chunk
// sums in chunk order): no atomics, the same bits on every run.  Entity entries are listed src (B), dst
// (B), then negatives (b, k); relation entries by triple.  Scratch is O(B (2 + K) dim) (TransR: plus B ent_dim rel_dim), never
// O(n_rows).  An id outside its table is read as row 0 and flagged: EU_ERR_INVALID after the call's one synchronisation.
//
// Tables are f32 or bf16 (Tab, an eu_feat_dtype; one type for all of a call's tables).  Every read of a table element widens
// bf16 to f32 exactly (row_load4, feat_ld; TransR's M is staged widened) and every other step is the f32 one, so a bf16 call
// gives the f32 call's bits on the widened tables: scores, rank, loss, embeddings and gradients alike, all of them f32.  The
// 4-wide loads (VEC) need both dims % 4 == 0 and each table aligned to four elements (16 bytes of f32, 8 of bf16).
#include <atomic>

#include "segment.cuh"

namespace eu {

constexpr int kKgMaxDim = 512;              // ent_dim and rel_dim bound: kKgCh float4 chunks per lane
constexpr int kKgCh = kKgMaxDim / 128;
constexpr int kKgMaxMat = 16384;            // TransR: the bound on ent_dim * rel_dim (M is staged in shared memory)
constexpr int kKgTile = 256;                // negatives per block
constexpr int kKgWarps = 8;
constexpr int kKgThreads = 32 * kKgWarps;
constexpr float kKgEps = 1e-12f;

enum { KG_TRANSE = EU_KG_TRANSE, KG_TRANSH = EU_KG_TRANSH, KG_TRANSR = EU_KG_TRANSR, KG_TRANSD = EU_KG_TRANSD,
       KG_DISTMULT = EU_KG_DISTMULT };

struct KgArgs {
  int l1, front, tail, C, K;
  float margin;
  int64_t B;
  const int64_t *src, *dst, *rel, *neg;
  const void *ent, *relt, *eaux, *raux;   // of the kernels' table type Tab
  int64_t n_ent, n_rel;
  int ent_dim, rel_dim;   // rel_dim is also the width of a mapped entity row and of every score
  int ldm;                // TransR: the row stride of the staged M (rel_dim rounded up to 4, plus 4 against bank conflicts)
};

// shared memory: the triple's rows s, d, r, the relation-side row a (h or rt), the sums f, t (kKgMaxDim floats each), then
// for TransR two rows per warp and M [ent_dim, ldm]
struct KgSmem {
  float *s, *d, *r, *a, *f, *t, *w, *m;
};

__device__ __forceinline__ KgSmem kg_smem(float* base) {
  KgSmem S;
  S.s = base; S.d = base + kKgMaxDim; S.r = base + 2 * kKgMaxDim; S.a = base + 3 * kKgMaxDim;
  S.f = base + 4 * kKgMaxDim; S.t = base + 5 * kKgMaxDim; S.w = base + 6 * kKgMaxDim;
  S.m = S.w + 2 * kKgWarps * kKgMaxDim;
  return S;
}

static size_t kg_smem_bytes(int model, int ent_dim, int ldm) {
  return 4 * (6 * (size_t)kKgMaxDim + (model == KG_TRANSR ? 2 * (size_t)kKgWarps * kKgMaxDim + (size_t)ent_dim * ldm : 0));
}
// the most TransR can take within its bounds: ent_dim * ldm <= ent_dim * (rel_dim + 7) <= kKgMaxMat + 7 kKgMaxDim
constexpr size_t kKgMaxSmem = 4 * (6 * (size_t)kKgMaxDim + 2 * (size_t)kKgWarps * kKgMaxDim + kKgMaxMat + 7 * (size_t)kKgMaxDim);

// TransR's kernels need more than 48 KB of dynamic shared memory: raise a kernel's limit to kKgMaxSmem once per device
template <class Kern>
static int kg_allow_smem(Kern* k, int device, std::atomic<unsigned long long>* done) {
  const unsigned long long bit = 1ull << (device & 63);
  if (done->load(std::memory_order_relaxed) & bit) return EU_OK;
  EU_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kKgMaxSmem));
  done->fetch_or(bit, std::memory_order_relaxed);
  return EU_OK;
}

// ---------------------------------------------------------------------------- warp rows
struct KgRow {
  float4 v[kKgCh];   // lane l's chunks l, l + 32, ...; zero past the row's end
};

__device__ __forceinline__ KgRow kg_zero() {
  KgRow r;
#pragma unroll
  for (int i = 0; i < kKgCh; ++i) r.v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  return r;
}
__device__ __forceinline__ int kg_col(int i) { return ((int)(threadIdx.x & 31) + 32 * i) * 4; }
__device__ __forceinline__ float& kg_c(float4& v, int c) { return c == 0 ? v.x : c == 1 ? v.y : c == 2 ? v.z : v.w; }
__device__ __forceinline__ float kg_c(const float4& v, int c) { return c == 0 ? v.x : c == 1 ? v.y : c == 2 ? v.z : v.w; }

// f(i, c) for each column 4 (lane + 32 i) + c < dim of this lane, in column order
template <class Fn>
__device__ __forceinline__ void kg_each(int dim, Fn f) {
#pragma unroll
  for (int i = 0; i < kKgCh; ++i) {
    const int d = kg_col(i);
#pragma unroll
    for (int c = 0; c < 4; ++c)
      if (d + c < dim) f(i, c);
  }
}

__device__ __forceinline__ float kg_wsum(float x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x = __fadd_rn(x, __shfl_xor_sync(0xffffffffu, x, o));
  return x;
}

// a table row widened to f32
template <bool VEC, typename Tab>
__device__ __forceinline__ KgRow kg_load(const Tab* __restrict__ row, int dim) {
  KgRow r;
#pragma unroll
  for (int i = 0; i < kKgCh; ++i) {
    const int d = kg_col(i);
    r.v[i] = d < dim ? row_load4<VEC, Tab>(row, d, dim) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  return r;
}

// a row of shared memory (16-byte aligned, zero-padded to a multiple of 4)
__device__ __forceinline__ KgRow kg_lds(const float* row, int dim) {
  KgRow r;
#pragma unroll
  for (int i = 0; i < kKgCh; ++i) {
    const int d = kg_col(i);
    r.v[i] = d < dim ? *reinterpret_cast<const float4*>(row + d) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  return r;
}
__device__ __forceinline__ void kg_sts(float* row, const KgRow& r, int dim) {
#pragma unroll
  for (int i = 0; i < kKgCh; ++i) {
    const int d = kg_col(i);
    if (d < dim) *reinterpret_cast<float4*>(row + d) = r.v[i];
  }
}
// a row of global memory: float4 stores when dim % 4 == 0 (the scratch rows are then 16-byte aligned)
__device__ __forceinline__ void kg_stg(float* row, const KgRow& r, int dim) {
  if (dim % 4 == 0) {
#pragma unroll
    for (int i = 0; i < kKgCh; ++i) {
      const int d = kg_col(i);
      if (d < dim) *reinterpret_cast<float4*>(row + d) = r.v[i];
    }
    return;
  }
  kg_each(dim, [&](int i, int c) { row[kg_col(i) + c] = kg_c(r.v[i], c); });
}

__device__ __forceinline__ float kg_dot(const KgRow& a, const KgRow& b, int dim) {
  float acc = 0.f;
  kg_each(dim, [&](int i, int c) { acc = __fmaf_rn(kg_c(a.v[i], c), kg_c(b.v[i], c), acc); });
  return kg_wsum(acc);
}

struct KgNorm {
  float inv;   // 1 / sqrt(max(sum x^2, eps))
  bool act;    // sum x^2 >= eps: the gradient reaches sum x^2
};

// x <- n(x)
__device__ __forceinline__ KgNorm kg_norm(KgRow& x, int dim) {
  const float ss = kg_dot(x, x, dim);
  KgNorm n;
  n.inv = __frsqrt_rn(fmaxf(ss, kKgEps));
  n.act = ss >= kKgEps;
  kg_each(dim, [&](int i, int c) { kg_c(x.v[i], c) = __fmul_rn(kg_c(x.v[i], c), n.inv); });
  return n;
}

// the gradient of x from that of y = n(x)
__device__ __forceinline__ KgRow kg_norm_back(const KgRow& y, KgNorm n, const KgRow& gy, int dim) {
  const float p = n.act ? kg_dot(y, gy, dim) : 0.f;
  KgRow g = kg_zero();
  kg_each(dim, [&](int i, int c) { kg_c(g.v[i], c) = __fmul_rn(n.inv, __fmaf_rn(-p, kg_c(y.v[i], c), kg_c(gy.v[i], c))); });
  return g;
}

// the score of (a, r, c) over dim columns
template <int M>
__device__ __forceinline__ float kg_score(int l1, const KgRow& a, const KgRow& r, const KgRow& cc, int dim) {
  float acc = 0.f;
  kg_each(dim, [&](int i, int c) {
    const float av = kg_c(a.v[i], c), rv = kg_c(r.v[i], c), cv = kg_c(cc.v[i], c);
    if (M == KG_DISTMULT) {
      acc = __fmaf_rn(av, __fmul_rn(rv, cv), acc);
    } else {
      const float x = __fsub_rn(__fadd_rn(av, rv), cv);
      acc = l1 ? __fadd_rn(acc, fabsf(x)) : __fmaf_rn(x, x, acc);
    }
  });
  acc = kg_wsum(acc);
  if (M == KG_DISTMULT) return acc;
  return l1 ? -acc : -__fsqrt_rn(acc);
}

// TransX: w * d(score)/dx for x = (a + r) - c: -w sign(x) (L1), -w x / ||x|| (L2, 0 at x = 0)
__device__ __forceinline__ KgRow kg_gx(int l1, float w, const KgRow& a, const KgRow& r, const KgRow& cc, int dim) {
  KgRow x = kg_zero();
  kg_each(dim, [&](int i, int c) { kg_c(x.v[i], c) = __fsub_rn(__fadd_rn(kg_c(a.v[i], c), kg_c(r.v[i], c)), kg_c(cc.v[i], c)); });
  if (l1) {
    kg_each(dim, [&](int i, int c) {
      const float v = kg_c(x.v[i], c);
      kg_c(x.v[i], c) = v > 0.f ? -w : v < 0.f ? w : 0.f;
    });
    return x;
  }
  const float nn = kg_dot(x, x, dim);
  const float s = nn > 0.f ? __fmul_rn(-w, __frsqrt_rn(nn)) : 0.f;
  kg_each(dim, [&](int i, int c) { kg_c(x.v[i], c) = __fmul_rn(s, kg_c(x.v[i], c)); });
  return x;
}

// ---------------------------------------------------------------------------- entity rows
struct KgMap {
  KgRow y;      // the mapped row (rel_dim columns)
  KgRow e, t;   // the entity row; TransD: its entity_transfer row
  KgNorm n;
  float dot;    // TransH: e . h; TransD: e . et
};

// the mapped row of entity table row `row`; TransR uses the warp's row buffer w
template <int M, bool VEC, typename Tab>
__device__ __forceinline__ void kg_map(const KgArgs& A, int64_t row, const KgSmem& S, float* w, KgMap& m) {
  m.e = kg_load<VEC>(static_cast<const Tab*>(A.ent) + row * A.ent_dim, A.ent_dim);
  m.dot = 0.f;
  m.n.inv = 1.f;
  m.n.act = false;
  if (M == KG_TRANSE || M == KG_DISTMULT) {
    m.y = m.e;
    m.n = kg_norm(m.y, A.ent_dim);
  } else if (M == KG_TRANSH) {
    const KgRow h = kg_lds(S.a, A.ent_dim);
    m.dot = kg_dot(m.e, h, A.ent_dim);
    m.y = kg_zero();
    kg_each(A.ent_dim, [&](int i, int c) { kg_c(m.y.v[i], c) = __fmaf_rn(-m.dot, kg_c(h.v[i], c), kg_c(m.e.v[i], c)); });
  } else if (M == KG_TRANSD) {
    m.t = kg_load<VEC>(static_cast<const Tab*>(A.eaux) + row * A.ent_dim, A.ent_dim);
    const KgRow rt = kg_lds(S.a, A.ent_dim);
    m.dot = kg_dot(m.e, m.t, A.ent_dim);
    m.y = kg_zero();
    kg_each(A.ent_dim, [&](int i, int c) { kg_c(m.y.v[i], c) = __fmaf_rn(m.dot, kg_c(rt.v[i], c), kg_c(m.e.v[i], c)); });
    m.n = kg_norm(m.y, A.ent_dim);
  } else {   // TransR: y_j = sum over i of e_i M_ij, fma in i order
    kg_sts(w, m.e, A.ent_dim);
    __syncwarp();
    m.y = kg_zero();
#pragma unroll
    for (int i = 0; i < kKgCh; ++i) {
      const int d = kg_col(i);
      if (d >= A.rel_dim) continue;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int k = 0; k < A.ent_dim; ++k) {
        const float ek = w[k];
        const float4 mv = *reinterpret_cast<const float4*>(S.m + k * A.ldm + d);
        acc.x = __fmaf_rn(ek, mv.x, acc.x); acc.y = __fmaf_rn(ek, mv.y, acc.y);
        acc.z = __fmaf_rn(ek, mv.z, acc.z); acc.w = __fmaf_rn(ek, mv.w, acc.w);
      }
      m.y.v[i] = acc;   // the staged M is zero past rel_dim
    }
    __syncwarp();
    m.n = kg_norm(m.y, A.rel_dim);
  }
}

// The entry of one entity row from the gradient gy of its mapped row: the entity-table row (and TransD's entity_transfer row)
// at entry `en` of Gent / Gea, and what reaches the relation-side row: U (the gradient of y for TransH, of the pre-normalised
// row for TransR and TransD) and sc = (TransH: e . h, gy . h; TransD: e . et, 0)
template <int M>
__device__ __forceinline__ void kg_entity_back(const KgArgs& A, const KgMap& m, const KgRow& gy, const KgSmem& S, float* w,
                                               int64_t en, float* Gent, float* Gea, float* U, float2* sc) {
  const int lane = threadIdx.x & 31;
  if (M == KG_TRANSE || M == KG_DISTMULT) {
    kg_stg(Gent + en * A.ent_dim, kg_norm_back(m.y, m.n, gy, A.ent_dim), A.ent_dim);
  } else if (M == KG_TRANSH) {
    const KgRow h = kg_lds(S.a, A.ent_dim);
    const float beta = kg_dot(gy, h, A.ent_dim);
    KgRow ge = kg_zero();
    kg_each(A.ent_dim, [&](int i, int c) { kg_c(ge.v[i], c) = __fmaf_rn(-beta, kg_c(h.v[i], c), kg_c(gy.v[i], c)); });
    kg_stg(Gent + en * A.ent_dim, ge, A.ent_dim);
    kg_stg(U, gy, A.ent_dim);
    if (lane == 0) *sc = make_float2(m.dot, beta);
  } else if (M == KG_TRANSD) {
    const KgRow gu = kg_norm_back(m.y, m.n, gy, A.ent_dim);
    const KgRow rt = kg_lds(S.a, A.ent_dim);
    const float gam = kg_dot(gu, rt, A.ent_dim);
    KgRow ge = kg_zero(), gt = kg_zero();
    kg_each(A.ent_dim, [&](int i, int c) {
      kg_c(ge.v[i], c) = __fmaf_rn(gam, kg_c(m.t.v[i], c), kg_c(gu.v[i], c));
      kg_c(gt.v[i], c) = __fmul_rn(gam, kg_c(m.e.v[i], c));
    });
    kg_stg(Gent + en * A.ent_dim, ge, A.ent_dim);
    kg_stg(Gea + en * A.ent_dim, gt, A.ent_dim);
    kg_stg(U, gu, A.ent_dim);
    if (lane == 0) *sc = make_float2(m.dot, 0.f);
  } else {   // TransR: ge_i = sum over j of M_ij gu_j, fma in j order
    const KgRow gu = kg_norm_back(m.y, m.n, gy, A.rel_dim);
    kg_stg(U, gu, A.rel_dim);
    float* wg = w + kKgMaxDim;
    kg_sts(wg, gu, A.rel_dim);
    __syncwarp();
    KgRow ge = kg_zero();
    kg_each(A.ent_dim, [&](int i, int c) {
      const float* mr = S.m + (kg_col(i) + c) * A.ldm;
      float acc = 0.f;
      for (int j = 0; j < A.rel_dim; ++j) acc = __fmaf_rn(mr[j], wg[j], acc);
      kg_c(ge.v[i], c) = acc;
    });
    __syncwarp();
    kg_stg(Gent + en * A.ent_dim, ge, A.ent_dim);
  }
}

// The triple's own rows into shared memory: r = n(relation row), a = h (TransH) or rt (TransD), M (TransR), then the mapped
// s and d.  Every thread of the block calls it.  M is staged widened to f32.
template <int M, bool VEC, typename Tab>
__device__ __forceinline__ void kg_stage(const KgArgs& A, int64_t b, const KgSmem& S, int* bad) {
  const int warp = threadIdx.x >> 5;
  const int64_t rb = row_of(__ldg(A.rel + b), A.n_rel, bad);
  if (M == KG_TRANSR) {
    const Tab* mr = static_cast<const Tab*>(A.raux) + rb * (int64_t)A.ent_dim * A.rel_dim;
    for (int t = threadIdx.x; t < A.ent_dim * A.ldm; t += blockDim.x) {
      const int i = t / A.ldm, j = t - i * A.ldm;
      S.m[t] = j < A.rel_dim ? feat_ld<Tab>(mr + (int64_t)i * A.rel_dim + j) : 0.f;
    }
  }
  if (warp == 0) {
    KgRow r = kg_load<VEC>(static_cast<const Tab*>(A.relt) + rb * A.rel_dim, A.rel_dim);
    kg_norm(r, A.rel_dim);
    kg_sts(S.r, r, A.rel_dim);
  } else if (warp == 1 && (M == KG_TRANSH || M == KG_TRANSD)) {
    KgRow a = kg_load<VEC>(static_cast<const Tab*>(A.raux) + rb * A.ent_dim, A.ent_dim);
    if (M == KG_TRANSH) kg_norm(a, A.ent_dim);
    kg_sts(S.a, a, A.ent_dim);
  }
  __syncthreads();
  if (warp < 2) {
    const int64_t id = __ldg((warp == 0 ? A.src : A.dst) + b);
    KgMap m;
    kg_map<M, VEC, Tab>(A, row_of(id, A.n_ent, bad), S, S.w + warp * 2 * kKgMaxDim, m);
    kg_sts(warp == 0 ? S.s : S.d, m.y, A.rel_dim);
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------- forward
// One block per (triple b, tile of kKgTile negatives); tile 0 also writes the true triple's score and the embeddings
template <int M, bool VEC, typename Tab>
__global__ void __launch_bounds__(kKgThreads) k_kg_fwd(KgArgs A, int tiles, float* __restrict__ scores, float* emb_s,
                                                        float* emb_r, float* emb_d, int* bad) {
  extern __shared__ float4 kg_sm4[];
  const KgSmem S = kg_smem(reinterpret_cast<float*>(kg_sm4));
  const int64_t b = blockIdx.x / tiles;
  const int tile = (int)(blockIdx.x - b * tiles);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  kg_stage<M, VEC, Tab>(A, b, S, bad);
  const int D = A.rel_dim;
  const KgRow s = kg_lds(S.s, D), d = kg_lds(S.d, D), r = kg_lds(S.r, D);
  float* srow = scores + b * (1 + (int64_t)A.C * A.K);
  if (tile == 0 && warp == 0) {
    const float p = kg_score<M>(A.l1, s, r, d, D);
    if (lane == 0) srow[0] = p;
  }
  if (tile == 0 && warp == 1 && emb_s) {
    for (int j = lane; j < D; j += 32) {
      emb_s[b * D + j] = S.s[j];
      emb_r[b * D + j] = S.r[j];
      emb_d[b * D + j] = S.d[j];
    }
  }
  float* wbuf = S.w + warp * 2 * kKgMaxDim;
  const int k1 = min(A.K, (tile + 1) * kKgTile);
  for (int k = tile * kKgTile + warp; k < k1; k += kKgWarps) {
    KgMap m;
    kg_map<M, VEC, Tab>(A, row_of(__ldg(A.neg + b * A.K + k), A.n_ent, bad), S, wbuf, m);
    if (A.front) {
      const float x = kg_score<M>(A.l1, m.y, r, d, D);
      if (lane == 0) srow[1 + k] = x;
    }
    if (A.tail) {
      const float x = kg_score<M>(A.l1, s, r, m.y, D);
      if (lane == 0) srow[1 + (A.front ? A.K : 0) + k] = x;
    }
  }
}

// One block of kKgThreads per triple (see the top of the file): forward, rank and rowloss; backward, coef = (cp, cn)
__global__ void __launch_bounds__(kKgThreads) k_kg_rows(const float* __restrict__ scores, int64_t B, int n, float margin,
                                                         int32_t* __restrict__ rank, double* __restrict__ rowloss,
                                                         const float* __restrict__ grad_loss, float2* __restrict__ coef) {
  __shared__ float sh[kKgThreads];
  __shared__ int shc[kKgThreads];
  const int64_t b = blockIdx.x;
  const float* row = scores + b * (1 + (int64_t)n);
  const float pos = __ldg(row);
  float acc = 0.f;
  int cnt = 0;
  for (int j = threadIdx.x; j < n; j += kKgThreads) {
    const float x = __ldg(row + 1 + j);
    acc = __fadd_rn(acc, x);
    cnt += x >= pos;
  }
  sh[threadIdx.x] = acc;
  shc[threadIdx.x] = cnt;
  __syncthreads();
  for (int s = kKgThreads / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) {
      sh[threadIdx.x] = __fadd_rn(sh[threadIdx.x], sh[threadIdx.x + s]);
      shc[threadIdx.x] += shc[threadIdx.x + s];
    }
    __syncthreads();
  }
  if (threadIdx.x != 0) return;
  const float h = __fsub_rn(__fadd_rn(margin, __fdiv_rn(sh[0], (float)n)), pos);
  if (rank) rank[b] = shc[0];
  if (rowloss) rowloss[b] = (double)fmaxf(h, 0.f);
  if (coef) {
    const float gB = __fdiv_rn(__ldg(grad_loss), (float)B);
    coef[b] = h >= 0.f ? make_float2(-gB, __fdiv_rn(gB, (float)n)) : make_float2(0.f, 0.f);
  }
}

// ---------------------------------------------------------------------------- backward
// The gradient of a mapped row y from its DistMult / TransX terms is assembled by the callers below.

// One block per (triple, tile), a warp per negative: the entity entries 2B + b K + k, F / T [b, k], U [b, 2 + k], sc [b, 2 + k]
template <int M, bool VEC, typename Tab>
__global__ void __launch_bounds__(kKgThreads) k_kg_bwd_neg(KgArgs A, int tiles, const float2* __restrict__ coef, float* F, float* T,
                                                            float* U, float2* sc, float* Gent, float* Gea, int* bad) {
  extern __shared__ float4 kg_sm4[];
  const KgSmem S = kg_smem(reinterpret_cast<float*>(kg_sm4));
  const int64_t b = blockIdx.x / tiles;
  const int tile = (int)(blockIdx.x - b * tiles);
  const int warp = threadIdx.x >> 5;
  kg_stage<M, VEC, Tab>(A, b, S, bad);
  const int D = A.rel_dim;
  const KgRow s = kg_lds(S.s, D), d = kg_lds(S.d, D), r = kg_lds(S.r, D);
  const float cn = coef[b].y;
  const int N = A.K + 2;
  float* wbuf = S.w + warp * 2 * kKgMaxDim;
  const int k1 = min(A.K, (tile + 1) * kKgTile);
  for (int k = tile * kKgTile + warp; k < k1; k += kKgWarps) {
    KgMap m;
    kg_map<M, VEC, Tab>(A, row_of(__ldg(A.neg + b * A.K + k), A.n_ent, bad), S, wbuf, m);
    KgRow gy = kg_zero();
    const int64_t bk = b * A.K + k;
    if (M == KG_DISTMULT) {
      if (A.front) {
        kg_each(D, [&](int i, int c) {
          kg_c(gy.v[i], c) = __fmul_rn(cn, __fmul_rn(kg_c(r.v[i], c), kg_c(d.v[i], c)));
        });
      }
      if (A.tail) {
        kg_each(D, [&](int i, int c) {
          kg_c(gy.v[i], c) = __fmaf_rn(cn, __fmul_rn(kg_c(s.v[i], c), kg_c(r.v[i], c)), kg_c(gy.v[i], c));
        });
      }
      KgRow cy = kg_zero();
      kg_each(D, [&](int i, int c) { kg_c(cy.v[i], c) = __fmul_rn(cn, kg_c(m.y.v[i], c)); });
      if (A.front) kg_stg(F + bk * D, cy, D);
      if (A.tail) kg_stg(T + bk * D, cy, D);
    } else {
      if (A.front) {
        const KgRow g = kg_gx(A.l1, cn, m.y, r, d, D);
        kg_stg(F + bk * D, g, D);
        gy = g;
      }
      if (A.tail) {
        const KgRow g = kg_gx(A.l1, cn, s, r, m.y, D);
        kg_stg(T + bk * D, g, D);
        kg_each(D, [&](int i, int c) { kg_c(gy.v[i], c) = __fsub_rn(kg_c(gy.v[i], c), kg_c(g.v[i], c)); });
      }
    }
    kg_entity_back<M>(A, m, gy, S, wbuf, 2 * A.B + bk, Gent, Gea, U + (b * N + 2 + k) * D, sc + b * N + 2 + k);
  }
}

// (The minimum of one block per SM lets ptxas use the registers it needs: without it, it capped this kernel at 80 and spilled.)
// One block per triple: SF, ST = F, T summed over k from +0 in f64; the src and dst entries (warps 0 and 1) and the relation entry
// (warp 2).  TransX: Gp = the true triple's term; gy_s = Gp + ST, gy_d = -(Gp + SF), gr = (Gp + SF) + ST.  DistMult:
// gy_s = fma(cp, r d, r ST), gy_d = fma(cp, s r, r SF), gr = fma(cp, s d, fma(d, SF, s ST)).
template <int M, bool VEC, typename Tab>
__global__ void __launch_bounds__(kKgThreads, 1) k_kg_bwd_triple(KgArgs A, const float2* __restrict__ coef, const float* __restrict__ F,
                                                               const float* __restrict__ T, float* U, float2* sc, float* Gent,
                                                               float* Gea, float* Grel, int* bad) {
  extern __shared__ float4 kg_sm4[];
  const KgSmem S = kg_smem(reinterpret_cast<float*>(kg_sm4));
  const int64_t b = blockIdx.x;
  const int warp = threadIdx.x >> 5;
  const int D = A.rel_dim, N = A.K + 2;
  for (int j = threadIdx.x; j < kKgMaxDim; j += kKgThreads) {
    double f = 0.0, t = 0.0;
    if (j < D) {
      for (int k = 0; k < A.K; ++k) {
        if (A.front) f += (double)__ldg(F + (b * A.K + k) * D + j);
        if (A.tail) t += (double)__ldg(T + (b * A.K + k) * D + j);
      }
    }
    S.f[j] = (float)f;
    S.t[j] = (float)t;
  }
  kg_stage<M, VEC, Tab>(A, b, S, bad);   // its barriers also publish S.f and S.t
  if (warp > 2) return;
  const float cp = coef[b].x;
  const KgRow s = kg_lds(S.s, D), d = kg_lds(S.d, D), r = kg_lds(S.r, D);
  const KgRow SF = kg_lds(S.f, D), ST = kg_lds(S.t, D);
  KgRow g = kg_zero();
  if (M == KG_DISTMULT) {
    if (warp == 0)
      kg_each(D, [&](int i, int c) {
        const float rv = kg_c(r.v[i], c);
        kg_c(g.v[i], c) = __fmaf_rn(cp, __fmul_rn(rv, kg_c(d.v[i], c)), __fmul_rn(rv, kg_c(ST.v[i], c)));
      });
    else if (warp == 1)
      kg_each(D, [&](int i, int c) {
        const float rv = kg_c(r.v[i], c);
        kg_c(g.v[i], c) = __fmaf_rn(cp, __fmul_rn(kg_c(s.v[i], c), rv), __fmul_rn(rv, kg_c(SF.v[i], c)));
      });
    else
      kg_each(D, [&](int i, int c) {
        const float sv = kg_c(s.v[i], c), dv = kg_c(d.v[i], c);
        kg_c(g.v[i], c) = __fmaf_rn(cp, __fmul_rn(sv, dv), __fmaf_rn(dv, kg_c(SF.v[i], c), __fmul_rn(sv, kg_c(ST.v[i], c))));
      });
  } else {
    g = kg_gx(A.l1, cp, s, r, d, D);
    if (warp == 0)
      kg_each(D, [&](int i, int c) { kg_c(g.v[i], c) = __fadd_rn(kg_c(g.v[i], c), kg_c(ST.v[i], c)); });
    else if (warp == 1)
      kg_each(D, [&](int i, int c) { kg_c(g.v[i], c) = -__fadd_rn(kg_c(g.v[i], c), kg_c(SF.v[i], c)); });
    else
      kg_each(D, [&](int i, int c) { kg_c(g.v[i], c) = __fadd_rn(__fadd_rn(kg_c(g.v[i], c), kg_c(SF.v[i], c)), kg_c(ST.v[i], c)); });
  }
  if (warp == 2) {
    const int64_t rb = row_of(__ldg(A.rel + b), A.n_rel, bad);
    KgRow y = kg_load<VEC>(static_cast<const Tab*>(A.relt) + rb * D, D);
    const KgNorm n = kg_norm(y, D);
    kg_stg(Grel + b * D, kg_norm_back(y, n, g, D), D);
    return;
  }
  KgMap m;
  float* wbuf = S.w + warp * 2 * kKgMaxDim;
  kg_map<M, VEC, Tab>(A, row_of(__ldg((warp == 0 ? A.src : A.dst) + b), A.n_ent, bad), S, wbuf, m);
  kg_entity_back<M>(A, m, g, S, wbuf, warp * A.B + b, Gent, Gea, U + (b * N + warp) * D, sc + b * N + warp);
}

// the entity row of entry n of triple b: src, dst, then the negatives
__device__ __forceinline__ int64_t kg_entity_of(const KgArgs& A, int64_t b, int n, int* bad) {
  const int64_t id = n == 0 ? __ldg(A.src + b) : n == 1 ? __ldg(A.dst + b) : __ldg(A.neg + b * A.K + (n - 2));
  return row_of(id, A.n_ent, bad);
}

// TransH and TransD, one block per triple, a thread per column, entries n = 0 .. K + 1 in order from +0:
//   TransH: gh_j = -(sum of alpha_n U_nj + beta_n e_nj), then through n() (warp 0);  TransD: grt_j = sum of delta_n U_nj;
//   f64 fmas, rounded once
template <int M, bool VEC, typename Tab>
__global__ void __launch_bounds__(kKgThreads) k_kg_bwd_raux(KgArgs A, const float* __restrict__ U, const float2* __restrict__ sc,
                                                             float* __restrict__ Graux) {
  __shared__ __align__(16) float sg[kKgMaxDim];
  const int64_t b = blockIdx.x;
  const int D = A.ent_dim, N = A.K + 2;
  int ignored = 0;
  for (int j = threadIdx.x; j < kKgMaxDim; j += kKgThreads) {
    double acc = 0.0;
    if (j < D) {
      for (int n = 0; n < N; ++n) {
        const float2 w = __ldg(sc + b * N + n);
        const float u = __ldg(U + (b * N + n) * D + j);
        acc = fma((double)w.x, (double)u, acc);
        if (M == KG_TRANSH)
          acc = fma((double)w.y, (double)feat_ld<Tab>(static_cast<const Tab*>(A.ent) + kg_entity_of(A, b, n, &ignored) * D + j), acc);
      }
    }
    if (M == KG_TRANSD && j < D) Graux[b * D + j] = (float)acc;
    sg[j] = (float)-acc;
  }
  if (M != KG_TRANSH) return;
  __syncthreads();
  if (threadIdx.x >= 32) return;
  KgRow y = kg_load<VEC>(static_cast<const Tab*>(A.raux) + row_of(__ldg(A.rel + b), A.n_rel, &ignored) * D, D);
  const KgNorm n = kg_norm(y, D);
  kg_stg(Graux + b * D, kg_norm_back(y, n, kg_lds(sg, D), D), D);
}

// TransR: gM[b, i, j] = sum over entries n of e_ni U_nj (e widened to f32, then exactly to f64), f64 fma in n order, rounded
// once; a thread per element
template <typename Tab>
__global__ void __launch_bounds__(256) k_kg_bwd_mat(KgArgs A, int blocks_per, const float* __restrict__ U, float* __restrict__ Graux) {
  const int64_t b = blockIdx.x / blocks_per;
  const int64_t t = (blockIdx.x - b * blocks_per) * 256 + threadIdx.x;
  const int64_t W = (int64_t)A.ent_dim * A.rel_dim;
  if (t >= W) return;
  const int i = (int)(t / A.rel_dim), j = (int)(t - (int64_t)i * A.rel_dim);
  const int N = A.K + 2;
  int ignored = 0;
  double acc = 0.0;
  for (int n = 0; n < N; ++n)
    acc = fma((double)feat_ld<Tab>(static_cast<const Tab*>(A.ent) + kg_entity_of(A, b, n, &ignored) * A.ent_dim + i),
              (double)__ldg(U + (b * N + n) * A.rel_dim + j), acc);
  Graux[b * W + t] = (float)acc;
}

// the int32 keys of the entity entries (src B, dst B, negatives B K) or of the relation entries (B)
__global__ void k_kg_keys(KgArgs A, bool entity, int64_t E, int32_t* __restrict__ key, int* bad) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < E; e += (int64_t)gridDim.x * blockDim.x) {
    if (!entity) {
      key[e] = (int32_t)row_of(__ldg(A.rel + e), A.n_rel, bad);
      continue;
    }
    const int64_t v = e < A.B ? __ldg(A.src + e) : e < 2 * A.B ? __ldg(A.dst + e - A.B) : __ldg(A.neg + e - 2 * A.B);
    key[e] = (int32_t)row_of(v, A.n_ent, bad);
  }
}

// ---------------------------------------------------------------------------- host side
static int kg_aux_width(int model, int ent_dim, int rel_dim) {
  return model == KG_TRANSH ? ent_dim : model == KG_TRANSR ? ent_dim * rel_dim : model == KG_TRANSD ? rel_dim : 0;
}

static int kg_args(eu_ctx* c, const eu_kg_problem* p, int dtype, KgArgs* A, const char* who) {
  if (!c || !p) {
    set_error("%s: bad argument", who);
    return EU_ERR_INVALID;
  }
  if (int rc = dtype_check(dtype, who, "table")) return rc;
  const int m = p->model;
  if (m < KG_TRANSE || m > KG_DISTMULT || p->corrupt < 1 || p->corrupt > 3 || p->B < 0 || p->K < 1 || p->ent_dim < 1 ||
      p->rel_dim < 1 || p->n_ent < 1 || p->n_rel < 1 || !p->table[0] || !p->table[1] || (p->B > 0 && (!p->src || !p->dst || !p->rel || !p->neg))) {
    set_error("%s: bad argument (model, corrupt 1..3, B >= 0, K >= 1, dims and table rows >= 1, ids and tables given)", who);
    return EU_ERR_INVALID;
  }
  if ((m == KG_TRANSH || m == KG_TRANSR || m == KG_TRANSD) && !p->table[3]) {
    set_error("%s: the model needs its relation-side table", who);
    return EU_ERR_INVALID;
  }
  if (m == KG_TRANSD && !p->table[2]) {
    set_error("%s: TransD needs its entity_transfer table", who);
    return EU_ERR_INVALID;
  }
  if (m != KG_TRANSR && p->ent_dim != p->rel_dim) {
    set_error("%s: ent_dim %d != rel_dim %d (only TransR maps between the two)", who, p->ent_dim, p->rel_dim);
    return EU_ERR_INVALID;
  }
  if (p->ent_dim > kKgMaxDim || p->rel_dim > kKgMaxDim || (m == KG_TRANSR && (int64_t)p->ent_dim * p->rel_dim > kKgMaxMat)) {
    set_error("%s: dims above %d, or a TransR ent_dim * rel_dim above %d, are not supported", who, kKgMaxDim, kKgMaxMat);
    return EU_ERR_UNSUPPORTED;
  }
  if (p->n_ent >= ((int64_t)1 << 31) || p->n_rel >= ((int64_t)1 << 31) || !entries_fit(p->B * ((int64_t)p->K + 2)) ||
      p->B * ceil_div(p->K, kKgTile) >= ((int64_t)1 << 31)) {
    set_error("%s: 2^31 or more table rows, or B (K + 2) entries with their chunks, are not supported", who);
    return EU_ERR_UNSUPPORTED;
  }
  A->l1 = p->l1 != 0;
  A->front = (p->corrupt & 1) != 0;
  A->tail = (p->corrupt & 2) != 0;
  A->C = A->front + A->tail;
  A->K = p->K;
  A->margin = p->margin;
  A->B = p->B;
  A->src = p->src; A->dst = p->dst; A->rel = p->rel; A->neg = p->neg;
  A->ent = p->table[0]; A->relt = p->table[1]; A->eaux = p->table[2]; A->raux = p->table[3];
  A->n_ent = p->n_ent; A->n_rel = p->n_rel;
  A->ent_dim = p->ent_dim; A->rel_dim = p->rel_dim;
  A->ldm = (int)(ceil_div(p->rel_dim, 4) * 4 + 4);
  return EU_OK;
}

static bool kg_vec(int model, const KgArgs& A, int dtype) {
  return A.ent_dim % 4 == 0 && A.rel_dim % 4 == 0 && aligned4_elems(A.ent, dtype) && aligned4_elems(A.relt, dtype) &&
         (!A.eaux || aligned4_elems(A.eaux, dtype)) && (model == KG_TRANSR || !A.raux || aligned4_elems(A.raux, dtype));
}

template <int M, bool VEC, typename Tab>
static int kg_launch_fwd(eu_ctx* c, const KgArgs& A, float* scores, float* es, float* er, float* ed, int* bad) {
  const size_t sm = kg_smem_bytes(M, A.ent_dim, A.ldm);
  if constexpr (M == KG_TRANSR) {
    static std::atomic<unsigned long long> done{0};
    if (int rc = kg_allow_smem(k_kg_fwd<M, VEC, Tab>, c->g->device, &done)) return rc;
  }
  const int tiles = (int)ceil_div(A.K, kKgTile);
  k_kg_fwd<M, VEC, Tab><<<(unsigned)(A.B * tiles), kKgThreads, sm, c->stream>>>(A, tiles, scores, es, er, ed, bad);
  EU_LAUNCHED();
  return EU_OK;
}

struct KgBwd {
  float2* coef = nullptr;
  float *F = nullptr, *T = nullptr, *U = nullptr, *Gent = nullptr, *Gea = nullptr, *Grel = nullptr, *Graux = nullptr;
  float2* sc = nullptr;
};

template <int M, bool VEC, typename Tab>
static int kg_launch_bwd(eu_ctx* c, const KgArgs& A, const KgBwd& W, int* bad) {
  cudaStream_t s = c->stream;
  const size_t sm = kg_smem_bytes(M, A.ent_dim, A.ldm);
  if constexpr (M == KG_TRANSR) {
    static std::atomic<unsigned long long> done_neg{0}, done_triple{0};
    if (int rc = kg_allow_smem(k_kg_bwd_neg<M, VEC, Tab>, c->g->device, &done_neg)) return rc;
    if (int rc = kg_allow_smem(k_kg_bwd_triple<M, VEC, Tab>, c->g->device, &done_triple)) return rc;
  }
  const int tiles = (int)ceil_div(A.K, kKgTile);
  k_kg_bwd_neg<M, VEC, Tab><<<(unsigned)(A.B * tiles), kKgThreads, sm, s>>>(A, tiles, W.coef, W.F, W.T, W.U, W.sc, W.Gent, W.Gea, bad);
  EU_LAUNCHED();
  k_kg_bwd_triple<M, VEC, Tab><<<(unsigned)A.B, kKgThreads, sm, s>>>(A, W.coef, W.F, W.T, W.U, W.sc, W.Gent, W.Gea, W.Grel, bad);
  EU_LAUNCHED();
  if constexpr (M == KG_TRANSH || M == KG_TRANSD) {
    k_kg_bwd_raux<M, VEC, Tab><<<(unsigned)A.B, kKgThreads, 0, s>>>(A, W.U, W.sc, W.Graux);
    EU_LAUNCHED();
  } else if constexpr (M == KG_TRANSR) {
    const int per = (int)ceil_div((int64_t)A.ent_dim * A.rel_dim, 256);
    k_kg_bwd_mat<Tab><<<(unsigned)(A.B * per), 256, 0, s>>>(A, per, W.U, W.Graux);
    EU_LAUNCHED();
  }
  return EU_OK;
}

template <int M>
static int kg_dispatch_fwd(eu_ctx* c, const KgArgs& A, int dtype, float* scores, float* es, float* er, float* ed, int* bad) {
  return with_dtype(dtype, [&](auto t) {
    using Tab = typename decltype(t)::type;
    return kg_vec(M, A, dtype) ? kg_launch_fwd<M, true, Tab>(c, A, scores, es, er, ed, bad)
                               : kg_launch_fwd<M, false, Tab>(c, A, scores, es, er, ed, bad);
  });
}
template <int M>
static int kg_dispatch_bwd(eu_ctx* c, const KgArgs& A, int dtype, const KgBwd& W, int* bad) {
  return with_dtype(dtype, [&](auto t) {
    using Tab = typename decltype(t)::type;
    return kg_vec(M, A, dtype) ? kg_launch_bwd<M, true, Tab>(c, A, W, bad) : kg_launch_bwd<M, false, Tab>(c, A, W, bad);
  });
}

// The backward pass both output forms share: out[t] is table t's dense gradient or COO values, rows[t] its COO rows
static int kg_backward(eu_ctx* c, const eu_kg_problem* p, int dtype, const float* grad_loss, const float* scores, bool sparse,
                       float* const* out, int64_t* const* rows, int64_t* counts, const char* who) {
  KgArgs A;
  int rc = kg_args(c, p, dtype, &A, who);
  if (rc) return rc;
  const int model = p->model;
  const bool has[4] = {true, true, model == KG_TRANSD, model == KG_TRANSH || model == KG_TRANSR || model == KG_TRANSD};
  const int aw = kg_aux_width(model, A.ent_dim, A.rel_dim);
  const int width[4] = {A.ent_dim, A.rel_dim, A.ent_dim, aw};
  const int64_t n_rows[4] = {A.n_ent, A.n_rel, A.n_ent, A.n_rel};
  if (!grad_loss || (A.B > 0 && !scores)) {
    set_error("%s: bad argument (grad_loss and scores are required)", who);
    return EU_ERR_INVALID;
  }
  for (int t = 0; t < 4; ++t) {
    if (has[t] && (!out || !out[t] || (sparse && (!rows || !rows[t] || !counts)))) {
      set_error("%s: bad argument (an output of table %d is missing)", who, t);
      return EU_ERR_INVALID;
    }
  }
  cudaStream_t s = c->stream;
  EU_CUDA(cudaSetDevice(c->g->device));
  for (int t = 0; t < 4; ++t) {
    if (!has[t]) continue;
    if (!sparse) EU_CUDA(cudaMemsetAsync(out[t], 0, 4 * (size_t)n_rows[t] * width[t], s));
    else counts[t] = 0;
  }
  if (A.B == 0) return EU_OK;
  const int64_t B = A.B, N = A.K + 2, E1 = B * N, D = A.rel_dim;
  RowList Le, Lr;   // the entity entries (src, dst, negatives), the relation entries (one per triple)
  Le.E = E1; Le.n_rows = A.n_ent;
  Lr.E = B; Lr.n_rows = A.n_rel;
  // flag and counts (256 B) | coef [B] | F | T [B K D] | U [B N D] | sc [B N] | Gent | Gea [E1 ent] | Grel [B rel] | Graux [B aw]
  // | entity list: keys, plan | relation list: keys, plan
  size_t o = 256;
  const size_t o_coef = o; o += a256(8 * (size_t)B);
  const size_t o_F = o; o += A.front ? a256(4 * (size_t)(B * A.K * D)) : 0;
  const size_t o_T = o; o += A.tail ? a256(4 * (size_t)(B * A.K * D)) : 0;
  const size_t o_U = o; o += a256(4 * (size_t)(E1 * D));
  const size_t o_sc = o; o += a256(8 * (size_t)E1);
  const size_t o_Ge = o; o += a256(4 * (size_t)E1 * A.ent_dim);
  const size_t o_Gea = o; o += has[2] ? a256(4 * (size_t)E1 * A.ent_dim) : 0;
  const size_t o_Gr = o; o += a256(4 * (size_t)B * A.rel_dim);
  const size_t o_Gra = o; o += has[3] ? a256(4 * (size_t)B * aw) : 0;
  const size_t o_Ke = o; o += a256(4 * (size_t)E1);
  const size_t o_Pe = o; o += row_plan_bytes(E1, A.n_ent, A.ent_dim);
  const size_t o_Kr = o; o += a256(4 * (size_t)B);
  const size_t o_Pr = o; o += row_plan_bytes(B, A.n_rel, std::max(A.rel_dim, aw));
  if ((rc = ctx_misc(c, (int64_t)o))) return rc;
  char* m = (char*)c->d_misc;
  int* bad = (int*)m;
  KgBwd W;
  W.coef = (float2*)(m + o_coef);
  W.F = (float*)(m + o_F);
  W.T = (float*)(m + o_T);
  W.U = (float*)(m + o_U);
  W.sc = (float2*)(m + o_sc);
  W.Gent = (float*)(m + o_Ge);
  W.Gea = (float*)(m + o_Gea);
  W.Grel = (float*)(m + o_Gr);
  W.Graux = (float*)(m + o_Gra);
  Le.key = (int32_t*)(m + o_Ke);
  Lr.key = (int32_t*)(m + o_Kr);
  EU_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), s));
  {
    EuProfScope ps(c, "kg_bwd_order", E1 + B);
    k_kg_keys<<<stride_grid(E1), 256, 0, s>>>(A, true, E1, Le.key, bad);
    EU_LAUNCHED();
    if ((rc = plan_rows(c, m + o_Pe, &Le))) return rc;
    k_kg_keys<<<stride_grid(B), 256, 0, s>>>(A, false, B, Lr.key, bad);
    EU_LAUNCHED();
    if ((rc = plan_rows(c, m + o_Pr, &Lr))) return rc;
  }
  {
    EuProfScope ps(c, "kg_bwd_rows", E1);
    k_kg_rows<<<(unsigned)B, kKgThreads, 0, s>>>(scores, B, A.C * A.K, A.margin, nullptr, nullptr, grad_loss, W.coef);
    EU_LAUNCHED();
    switch (model) {
      case KG_TRANSE: rc = kg_dispatch_bwd<KG_TRANSE>(c, A, dtype, W, bad); break;
      case KG_TRANSH: rc = kg_dispatch_bwd<KG_TRANSH>(c, A, dtype, W, bad); break;
      case KG_TRANSR: rc = kg_dispatch_bwd<KG_TRANSR>(c, A, dtype, W, bad); break;
      case KG_TRANSD: rc = kg_dispatch_bwd<KG_TRANSD>(c, A, dtype, W, bad); break;
      default: rc = kg_dispatch_bwd<KG_DISTMULT>(c, A, dtype, W, bad); break;
    }
    if (rc) return rc;
  }
  EuProfScope ps(c, "kg_bwd_sums", E1 + B);
  const float* vals[4] = {W.Gent, W.Grel, W.Gea, W.Graux};
  for (int t = 0; t < 4; ++t) {
    if (!has[t]) continue;
    RowEntries R;   // one stored row per entry
    R.n_src = t % 2 == 0 ? E1 : B;
    R.gt = vals[t];
    if ((rc = sum_distinct_rows(c, R, t % 2 == 0 ? Le : Lr, width[t], !sparse, out[t], sparse ? rows[t] : nullptr))) return rc;
  }
  bool h_bad = false;
  const int32_t* nd[2] = {Le.P.nd, Lr.P.nd};
  int64_t n[2] = {0, 0};
  if ((rc = read_back(c, bad, &h_bad, sparse ? 2 : 0, nd, n))) return rc;
  if (h_bad) {
    set_error("%s: an id lies outside its table's rows", who);
    return EU_ERR_INVALID;
  }
  if (sparse)
    for (int t = 0; t < 4; ++t)
      if (has[t]) counts[t] = n[t % 2];
  return EU_OK;
}

// The forward pass of both table types
static int kg_forward(eu_ctx* c, const eu_kg_problem* p, int dtype, float* scores, int32_t* rank, float* loss, float* src_emb,
                      float* rel_emb, float* dst_emb, const char* who) {
  KgArgs A;
  int rc = kg_args(c, p, dtype, &A, who);
  if (rc) return rc;
  if (!loss || (A.B > 0 && (!scores || !rank)) || (src_emb && A.B > 0 && (!rel_emb || !dst_emb))) {
    set_error("%s: bad argument (scores, rank and loss are required; the embeddings all or none)", who);
    return EU_ERR_INVALID;
  }
  EU_CUDA(cudaSetDevice(c->g->device));
  EuProfScope ps(c, "kg_fwd", A.B);
  bool h_bad = false;
  rc = mean_loss(c, A.B, A.B, loss, &h_bad, [&](int* bad, double* rowloss) -> int {
    int rc2;
    switch (p->model) {
      case KG_TRANSE: rc2 = kg_dispatch_fwd<KG_TRANSE>(c, A, dtype, scores, src_emb, rel_emb, dst_emb, bad); break;
      case KG_TRANSH: rc2 = kg_dispatch_fwd<KG_TRANSH>(c, A, dtype, scores, src_emb, rel_emb, dst_emb, bad); break;
      case KG_TRANSR: rc2 = kg_dispatch_fwd<KG_TRANSR>(c, A, dtype, scores, src_emb, rel_emb, dst_emb, bad); break;
      case KG_TRANSD: rc2 = kg_dispatch_fwd<KG_TRANSD>(c, A, dtype, scores, src_emb, rel_emb, dst_emb, bad); break;
      default: rc2 = kg_dispatch_fwd<KG_DISTMULT>(c, A, dtype, scores, src_emb, rel_emb, dst_emb, bad); break;
    }
    if (rc2) return rc2;
    k_kg_rows<<<(unsigned)A.B, kKgThreads, 0, c->stream>>>(scores, A.B, A.C * A.K, A.margin, rank, rowloss, nullptr, nullptr);
    EU_LAUNCHED();
    return EU_OK;
  });
  if (rc) return rc;
  if (h_bad) {
    set_error("%s: an id lies outside its table's rows", who);
    return EU_ERR_INVALID;
  }
  return EU_OK;
}

}  // namespace eu

using namespace eu;

extern "C" {

int eu_kg_loss(eu_ctx* c, const eu_kg_problem* p, float* scores, int32_t* rank, float* loss, float* src_emb, float* rel_emb,
               float* dst_emb) {
  return kg_forward(c, p, EU_FEAT_F32, scores, rank, loss, src_emb, rel_emb, dst_emb, "eu_kg_loss");
}

int eu_kg_loss_dtype(eu_ctx* c, const eu_kg_problem* p, int32_t table_dtype, float* scores, int32_t* rank, float* loss,
                     float* src_emb, float* rel_emb, float* dst_emb) {
  return kg_forward(c, p, table_dtype, scores, rank, loss, src_emb, rel_emb, dst_emb, "eu_kg_loss_dtype");
}

int eu_kg_loss_backward(eu_ctx* c, const eu_kg_problem* p, const float* grad_loss, const float* scores, float* const* grads) {
  return kg_backward(c, p, EU_FEAT_F32, grad_loss, scores, false, grads, nullptr, nullptr, "eu_kg_loss_backward");
}

int eu_kg_loss_backward_dtype(eu_ctx* c, const eu_kg_problem* p, int32_t table_dtype, const float* grad_loss, const float* scores,
                              float* const* grads) {
  return kg_backward(c, p, table_dtype, grad_loss, scores, false, grads, nullptr, nullptr, "eu_kg_loss_backward_dtype");
}

int eu_kg_loss_backward_sparse(eu_ctx* c, const eu_kg_problem* p, const float* grad_loss, const float* scores, int64_t* const* rows,
                               float* const* values, int64_t* counts) {
  return kg_backward(c, p, EU_FEAT_F32, grad_loss, scores, true, values, rows, counts, "eu_kg_loss_backward_sparse");
}

int eu_kg_loss_backward_sparse_dtype(eu_ctx* c, const eu_kg_problem* p, int32_t table_dtype, const float* grad_loss,
                                     const float* scores, int64_t* const* rows, float* const* values, int64_t* counts) {
  return kg_backward(c, p, table_dtype, grad_loss, scores, true, values, rows, counts, "eu_kg_loss_backward_sparse_dtype");
}

}  // extern "C"
