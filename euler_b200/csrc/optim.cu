// tf_euler's optimizers (tf_euler/python/utils/optimizers.py: sgd = MomentumOptimizer(lr, 0), momentum =
// MomentumOptimizer(lr, 0.9), AdagradOptimizer, AdamOptimizer) on the device, as TF 1.x applies them, in place over a
// variable var f32[N, D] and its slot tables of the same shape.
//
// All arithmetic is f32, each operation one round-to-nearest op in the order written, with no FMA contraction (every op is
// a __f*_rn intrinsic).  rsqrt(a) is 1 / sqrt(a), two roundings.
//
// Sparse gradients (TF's IndexedSlices, summed over duplicate indices first): rows i64[R], sorted and unique, and values
// g f32[R, D].
//   Momentum (sparse_apply_momentum, non-Nesterov), touched rows only:  accum = accum * momentum + g;  var = var - lr * accum
//   Adagrad (sparse_apply_adagrad), touched rows only:  accum = accum + g * g;  var = var - (lr * g) * rsqrt(accum)
//   Adam (AdamOptimizer._apply_sparse_shared), every row of the table:
//     m = m * b1, then on touched rows m = m + g * (1 - b1)
//     v = v * b2, then on touched rows v = v + (g * g) * (1 - b2)
//     var = var - (alpha * m) / (sqrt(v) + eps)
// Dense gradients (apply_momentum, apply_adagrad, ApplyAdam): Momentum and Adagrad as above on every element; Adam
//     m = m + (g - m) * (1 - b1);  v = v + (g * g - v) * (1 - b2);  var = var - (m * alpha) / (sqrt(v) + eps)
// The dense and sparse Adam formulas round differently; both are TF's.  Adam's step scalar
//     alpha = (lr * sqrt(1 - beta2_power)) / (1 - beta1_power)
// is computed in f32 from the device pair powers = (beta1_power, beta2_power), read by every thread, so a step can be captured in a CUDA
// graph.  The powers (TF's non-slot variables, starting at beta1 and beta2) are the caller's: it multiplies each by its beta
// once after every variable of a step is updated (_finish).
//
// Sparse Adam is one pass over the table: each CTA owns kChunk elements' worth of whole rows, issues its var, m, v loads, then
// finds its slice of the sorted gradient rows with one warp-wide 32-way search and maps its rows to their gradient rows in
// shared memory; an untouched row takes the decay-only branch.  It reads and writes var, m and v once and reads each gradient
// row once: 24 N D + 4 R (D + 2) bytes.  Sparse Momentum and Adagrad touch the R rows only; dense forms are element-wise.
// float4 when D % 4 == 0 and every pointer is 16-byte aligned, scalar otherwise; element indices are 64-bit.  No float
// atomics and no host synchronisation.  A row outside [0, N) is never written.
//
// bf16 tables (T = __nv_bfloat16: var and every slot bf16, the gradient f32; the *_dtype entry points).  Each element is
// widened exactly to f32, updated by the same upd / adam_decay in f32, and each value written (var and every slot) is rounded
// to bf16 by sr_st (common.cuh), stochastic rounding.  Its random word is word w (0 var, 1 the first slot, 2 the second) of
// SrKey{seed, step, tensor}'s for the element: element is the flat index r D + col into var, step the device step counter
// (the caller advances it once per step, after every variable, as Adam's powers), tensor the variable's index among the
// caller's.  A step is thus deterministic and can be captured in a CUDA graph.  The 4-wide form
// needs var and the slots 8-byte aligned (one 8-byte load or store per tensor and element group of four).
#include <type_traits>

#include "internal.h"

namespace eu {

constexpr int kOptThreads = 256;
constexpr int kChunk = kOptThreads * 16;   // sparse Adam: elements per CTA pass (16 per thread)

enum { kMomentum = 0, kAdagrad = 1, kAdam = 2 };

struct OptArgs {
  float lr, mom, b1, b2, eps;
  const float* powers;   // Adam: (beta1_power, beta2_power)
};

__device__ __forceinline__ float adam_alpha(const OptArgs& a) {
  const float b1p = __ldg(a.powers), b2p = __ldg(a.powers + 1);
  return __fdiv_rn(__fmul_rn(a.lr, __fsqrt_rn(__fsub_rn(1.f, b2p))), __fsub_rn(1.f, b1p));
}

// one element of a touched (or dense) row; alpha is Adam's step scalar
template <int K, bool SPARSE>
__device__ __forceinline__ void upd(const OptArgs& a, float alpha, float g, float& w, float& s1, float& s2) {
  if (K == kMomentum) {
    s1 = __fadd_rn(__fmul_rn(s1, a.mom), g);
    w = __fsub_rn(w, __fmul_rn(a.lr, s1));
  } else if (K == kAdagrad) {
    s1 = __fadd_rn(s1, __fmul_rn(g, g));
    w = __fsub_rn(w, __fmul_rn(__fmul_rn(a.lr, g), __fdiv_rn(1.f, __fsqrt_rn(s1))));
  } else if (SPARSE) {
    s1 = __fadd_rn(__fmul_rn(s1, a.b1), __fmul_rn(g, __fsub_rn(1.f, a.b1)));
    s2 = __fadd_rn(__fmul_rn(s2, a.b2), __fmul_rn(__fmul_rn(g, g), __fsub_rn(1.f, a.b2)));
    w = __fsub_rn(w, __fdiv_rn(__fmul_rn(alpha, s1), __fadd_rn(__fsqrt_rn(s2), a.eps)));
  } else {
    s1 = __fadd_rn(s1, __fmul_rn(__fsub_rn(g, s1), __fsub_rn(1.f, a.b1)));
    s2 = __fadd_rn(s2, __fmul_rn(__fsub_rn(__fmul_rn(g, g), s2), __fsub_rn(1.f, a.b2)));
    w = __fsub_rn(w, __fdiv_rn(__fmul_rn(s1, alpha), __fadd_rn(__fsqrt_rn(s2), a.eps)));
  }
}

// sparse Adam on a row without gradient: decay m and v, move var
__device__ __forceinline__ void adam_decay(const OptArgs& a, float alpha, float& w, float& m, float& v) {
  m = __fmul_rn(m, a.b1);
  v = __fmul_rn(v, a.b2);
  w = __fsub_rn(w, __fdiv_rn(__fmul_rn(alpha, m), __fadd_rn(__fsqrt_rn(v), a.eps)));
}

template <typename T>
constexpr bool kBf16 = std::is_same<T, __nv_bfloat16>::value;

// VW consecutive elements of a table of T, as f32: one float4 / one 8-byte bf16 access, or one element
template <int VW, typename T = float>
struct Vec {
  float x[VW];
  __device__ __forceinline__ void load(const T* p) {
    if constexpr (VW == 4) {
      const float4 t = rw_ld4(p);
      x[0] = t.x; x[1] = t.y; x[2] = t.z; x[3] = t.w;
    } else {
      x[0] = rw_ld(p);
    }
  }
  // r: the elements' random words (bf16 only)
  __device__ __forceinline__ void store(T* p, const uint32_t (&r)[VW]) const {
    if constexpr (VW == 4) sr_st4(p, make_float4(x[0], x[1], x[2], x[3]), r);
    else sr_st(p, x[0], r[0]);
  }
};

// dense form: element-wise over n = N D elements, VW per thread
template <int K, int VW, typename T>
__global__ void __launch_bounds__(kOptThreads) k_opt_dense(OptArgs a, T* __restrict__ var, T* __restrict__ s1,
                                                           T* __restrict__ s2, const float* __restrict__ grad, int64_t n,
                                                           SrKey sk) {
  const int64_t e = (blockIdx.x * (int64_t)kOptThreads + threadIdx.x) * VW;
  if (e >= n) return;
  const float alpha = K == kAdam ? adam_alpha(a) : 0.f;
  Vec<VW, T> w, x, y;
  Vec<VW> g;
  w.load(var + e);
  x.load(s1 + e);
  if (K == kAdam) y.load(s2 + e);
  g.load(grad + e);
#pragma unroll
  for (int i = 0; i < VW; ++i) upd<K, false>(a, alpha, g.x[i], w.x[i], x.x[i], y.x[i]);
  uint32_t r[3][VW] = {};
  if constexpr (kBf16<T>) sr_words(sk, e, r);
  w.store(var + e, r[0]);
  x.store(s1 + e, r[1]);
  if (K == kAdam) y.store(s2 + e, r[2]);
}

// sparse Momentum / Adagrad: element-wise over the R D gradient elements, VW per thread
template <int K, int VW, typename T>
__global__ void __launch_bounds__(kOptThreads) k_opt_rows(OptArgs a, T* __restrict__ var, T* __restrict__ s1,
                                                          int64_t N, int D, const float* __restrict__ grad,
                                                          const int64_t* __restrict__ rows, int64_t R, SrKey sk) {
  const int64_t q = blockIdx.x * (int64_t)kOptThreads + threadIdx.x, per_row = D / VW;
  if (q >= R * per_row) return;
  const int64_t k = q / per_row, col = (q - k * per_row) * VW, r = __ldg(rows + k);
  if (r < 0 || r >= N) return;
  const int64_t e = r * D + col;
  Vec<VW, T> w, x;
  Vec<VW> g;
  float unused = 0.f;
  w.load(var + e);
  x.load(s1 + e);
  g.load(grad + k * D + col);
#pragma unroll
  for (int i = 0; i < VW; ++i) upd<K, true>(a, 0.f, g.x[i], w.x[i], x.x[i], unused);
  uint32_t rw[3][VW] = {};
  if constexpr (kBf16<T>) sr_words(sk, e, rw);
  w.store(var + e, rw[0]);
  x.store(s1 + e, rw[1]);
}

// the first k in [0, R) with rows[k] >= r0 (R if none), by warp 0: each round the 32 lanes probe 32 evenly spaced rows of the
// remaining range and keep the gap where the answer lies, so a range of R rows takes about log32(R) dependent loads
__device__ int64_t warp_lower_bound(const int64_t* __restrict__ rows, int64_t R, int64_t r0) {
  const int lane = threadIdx.x & 31;
  int64_t lo = 0, hi = R;   // the answer lies in [lo, hi]
  while (lo < hi) {
    const int64_t s = (hi - lo + 31) / 32, idx = lo + lane * s;
    const bool below = idx < hi && __ldg(rows + idx) < r0;
    const int c = __popc(__ballot_sync(0xffffffffu, below));   // rows are sorted: the lanes below r0 are a prefix
    if (c == 0) return lo;
    const int64_t nlo = lo + (c - 1) * s + 1, nhi = lo + c * s;
    lo = nlo;
    hi = nhi < hi ? nhi : hi;
  }
  return lo;
}

// sparse Adam: CTA b owns the rows [b rpc, b rpc + nr) (rpc = rows_per_cta), nr D elements in passes of kChunk
template <int VW, typename T>
__global__ void __launch_bounds__(kOptThreads) k_adam_sparse(OptArgs a, T* __restrict__ var, T* __restrict__ m,
                                                             T* __restrict__ v, int64_t N, int D,
                                                             const float* __restrict__ grad, const int64_t* __restrict__ rows,
                                                             int64_t R, int rows_per_cta, SrKey sk) {
  constexpr int kItems = 16 / VW;   // vectors per thread per pass
  __shared__ int s_slot[kChunk];    // the CTA's row i -> its gradient row - lo, or -1
  __shared__ long long s_lo;
  const int64_t r0 = blockIdx.x * (int64_t)rows_per_cta;
  const int nr = (int)min((int64_t)rows_per_cta, N - r0);
  const int nq = nr * D / VW;   // vectors of the CTA (a vector never straddles two rows)
  T* const vb = var + r0 * D;
  T* const mb = m + r0 * D;
  T* const sb = v + r0 * D;
  const float alpha = adam_alpha(a);
  Vec<VW, T> w[kItems], x[kItems], y[kItems];
  // the first pass's loads go out before the search, so the search's latency hides under them
#pragma unroll
  for (int u = 0; u < kItems; ++u) {
    const int q = threadIdx.x + u * kOptThreads;
    if (q < nq) {
      w[u].load(vb + (int64_t)q * VW);
      x[u].load(mb + (int64_t)q * VW);
      y[u].load(sb + (int64_t)q * VW);
    }
  }
  for (int i = threadIdx.x; i < nr; i += kOptThreads) s_slot[i] = -1;
  if (threadIdx.x < 32) {
    const int64_t lo = warp_lower_bound(rows, R, r0);
    if (threadIdx.x == 0) s_lo = lo;
  }
  __syncthreads();
  const int64_t lo = s_lo;
  for (int64_t k = lo + threadIdx.x; k < R; k += kOptThreads) {
    const int64_t r = __ldg(rows + k);
    if (r >= r0 + nr) break;   // sorted: every later row is past the CTA's rows too
    if (r >= r0) s_slot[r - r0] = (int)(k - lo);
  }
  __syncthreads();
  for (int base = 0; base < nq; base += kItems * kOptThreads) {
    if (base > 0) {
#pragma unroll
      for (int u = 0; u < kItems; ++u) {
        const int q = base + threadIdx.x + u * kOptThreads;
        if (q < nq) {
          w[u].load(vb + (int64_t)q * VW);
          x[u].load(mb + (int64_t)q * VW);
          y[u].load(sb + (int64_t)q * VW);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < kItems; ++u) {
      const int q = base + threadIdx.x + u * kOptThreads;
      if (q >= nq) continue;
      const int e = q * VW, row = e / D, slot = s_slot[row];
      if (slot >= 0) {
        Vec<VW> g;
        g.load(grad + (lo + slot) * (int64_t)D + (e - row * D));
#pragma unroll
        for (int i = 0; i < VW; ++i) upd<kAdam, true>(a, alpha, g.x[i], w[u].x[i], x[u].x[i], y[u].x[i]);
      } else {
#pragma unroll
        for (int i = 0; i < VW; ++i) adam_decay(a, alpha, w[u].x[i], x[u].x[i], y[u].x[i]);
      }
      uint32_t r[3][VW] = {};
      if constexpr (kBf16<T>) sr_words(sk, r0 * D + e, r);
      w[u].store(vb + (int64_t)e, r[0]);
      x[u].store(mb + (int64_t)e, r[1]);
      y[u].store(sb + (int64_t)e, r[2]);
    }
  }
}

static bool a16(const void* p) { return ((uintptr_t)p & 15) == 0; }

// the shared checks of the entry points; *dense is set when R == EU_OPTIM_DENSE
static int opt_check(const char* who, eu_ctx* c, const void* var, const void* s1, const void* s2, bool two_slots, int64_t N,
                     int32_t D, const float* grad, const int64_t* rows, int64_t R, int32_t dtype, const int64_t* step,
                     bool* dense) {
  *dense = R == EU_OPTIM_DENSE;
  const bool any = N > 0;
  if (!c || N < 0 || D < 1 || (R < 0 && !*dense) || (!*dense && R > N) || (any && (!var || !s1 || (two_slots && !s2))) ||
      (*dense && any && !grad) || (!*dense && R > 0 && (!grad || !rows))) {
    set_error("%s: bad argument (N >= 0, D >= 1, R = EU_OPTIM_DENSE or 0 <= R <= N, var and its slots, and grad (and rows "
              "when R > 0))", who);
    return EU_ERR_INVALID;
  }
  if (!dtype_ok(dtype) || (dtype == EU_FEAT_BF16 && !step)) {
    set_error("%s: bad argument (dtype EU_FEAT_F32 or EU_FEAT_BF16, and a bf16 table needs the device step counter)", who);
    return EU_ERR_INVALID;
  }
  return EU_OK;
}

// the 4-wide form: D % 4 == 0, var and the slots aligned to four elements, grad to 16 bytes
static bool opt_vec(int32_t D, int32_t dtype, const void* var, const void* s1, const void* s2, const float* grad) {
  return D % 4 == 0 && aligned4_elems(var, dtype) && aligned4_elems(s1, dtype) && (!s2 || aligned4_elems(s2, dtype)) && a16(grad);
}

template <int K, typename T>
static int launch_dense(eu_ctx* c, const OptArgs& a, const SrKey& sk, T* var, T* s1, T* s2, const float* grad, int64_t n,
                        bool vec) {
  if (n == 0) return EU_OK;
  const int vw = vec ? 4 : 1;
  const unsigned blocks = (unsigned)ceil_div(ceil_div(n, vw), kOptThreads);
  if (vec) k_opt_dense<K, 4><<<blocks, kOptThreads, 0, c->stream>>>(a, var, s1, s2, grad, n, sk);
  else k_opt_dense<K, 1><<<blocks, kOptThreads, 0, c->stream>>>(a, var, s1, s2, grad, n, sk);
  EU_LAUNCHED();
  return EU_OK;
}

template <int K, typename T>
static int launch_rows(eu_ctx* c, const OptArgs& a, const SrKey& sk, T* var, T* s1, int64_t N, int D, const float* grad,
                       const int64_t* rows, int64_t R, bool vec) {
  if (R == 0) return EU_OK;
  const int vw = vec ? 4 : 1;
  const unsigned blocks = (unsigned)ceil_div(R * (D / vw), kOptThreads);
  if (vec) k_opt_rows<K, 4><<<blocks, kOptThreads, 0, c->stream>>>(a, var, s1, N, D, grad, rows, R, sk);
  else k_opt_rows<K, 1><<<blocks, kOptThreads, 0, c->stream>>>(a, var, s1, N, D, grad, rows, R, sk);
  EU_LAUNCHED();
  return EU_OK;
}

// Momentum (K = kMomentum) or Adagrad over a table of T
template <int K, typename T>
static int run_one_slot(eu_ctx* c, const OptArgs& a, const SrKey& sk, void* var, void* accum, int64_t N, int32_t D,
                        const float* grad, const int64_t* rows, int64_t R, bool dense, bool vec) {
  T* w = static_cast<T*>(var);
  T* s1 = static_cast<T*>(accum);
  return dense ? launch_dense<K>(c, a, sk, w, s1, (T*)nullptr, grad, N * D, vec) : launch_rows<K>(c, a, sk, w, s1, N, D, grad, rows, R, vec);
}

template <typename T>
static int run_adam(eu_ctx* c, const OptArgs& a, const SrKey& sk, void* var, void* m, void* v, int64_t N, int32_t D,
                    const float* grad, const int64_t* rows, int64_t R, bool dense, bool vec) {
  T* w = static_cast<T*>(var);
  T* s1 = static_cast<T*>(m);
  T* s2 = static_cast<T*>(v);
  if (dense) return launch_dense<kAdam>(c, a, sk, w, s1, s2, grad, N * D, vec);
  if (N == 0) return EU_OK;
  const int rows_per_cta = D >= kChunk ? 1 : kChunk / D;
  const unsigned blocks = (unsigned)ceil_div(N, rows_per_cta);
  if (vec) k_adam_sparse<4><<<blocks, kOptThreads, 0, c->stream>>>(a, w, s1, s2, N, D, grad, rows, R, rows_per_cta, sk);
  else k_adam_sparse<1><<<blocks, kOptThreads, 0, c->stream>>>(a, w, s1, s2, N, D, grad, rows, R, rows_per_cta, sk);
  EU_LAUNCHED();
  return EU_OK;
}

static int momentum(const char* who, eu_ctx* c, void* var, void* accum, int64_t N, int32_t D, const float* grad,
                    const int64_t* rows, int64_t R, float lr, float mom, int32_t dtype, const SrKey& sk) {
  bool dense;
  int rc;
  if ((rc = opt_check(who, c, var, accum, nullptr, false, N, D, grad, rows, R, dtype, sk.step, &dense))) return rc;
  EU_CUDA(cudaSetDevice(c->g->device));
  const OptArgs a{lr, mom, 0.f, 0.f, 0.f, nullptr};
  const bool vec = opt_vec(D, dtype, var, accum, nullptr, grad);
  EuProfScope ps(c, "optim_momentum", dense ? N : R);
  return with_dtype(dtype, [&](auto t) {
    return run_one_slot<kMomentum, typename decltype(t)::type>(c, a, sk, var, accum, N, D, grad, rows, R, dense, vec);
  });
}

static int adagrad(const char* who, eu_ctx* c, void* var, void* accum, int64_t N, int32_t D, const float* grad,
                   const int64_t* rows, int64_t R, float lr, int32_t dtype, const SrKey& sk) {
  bool dense;
  int rc;
  if ((rc = opt_check(who, c, var, accum, nullptr, false, N, D, grad, rows, R, dtype, sk.step, &dense))) return rc;
  EU_CUDA(cudaSetDevice(c->g->device));
  const OptArgs a{lr, 0.f, 0.f, 0.f, 0.f, nullptr};
  const bool vec = opt_vec(D, dtype, var, accum, nullptr, grad);
  EuProfScope ps(c, "optim_adagrad", dense ? N : R);
  return with_dtype(dtype, [&](auto t) {
    return run_one_slot<kAdagrad, typename decltype(t)::type>(c, a, sk, var, accum, N, D, grad, rows, R, dense, vec);
  });
}

static int adam(const char* who, eu_ctx* c, void* var, void* m, void* v, int64_t N, int32_t D, const float* grad,
                const int64_t* rows, int64_t R, const float* powers, float lr, float beta1, float beta2, float epsilon,
                int32_t dtype, const SrKey& sk) {
  bool dense;
  int rc;
  if ((rc = opt_check(who, c, var, m, v, true, N, D, grad, rows, R, dtype, sk.step, &dense))) return rc;
  if (!powers) {
    set_error("%s: powers (device f32[2]: beta1_power, beta2_power) is needed", who);
    return EU_ERR_INVALID;
  }
  EU_CUDA(cudaSetDevice(c->g->device));
  const OptArgs a{lr, 0.f, beta1, beta2, epsilon, powers};
  const bool vec = opt_vec(D, dtype, var, m, v, grad);
  EuProfScope ps(c, "optim_adam", N);
  return with_dtype(dtype, [&](auto t) {
    return run_adam<typename decltype(t)::type>(c, a, sk, var, m, v, N, D, grad, rows, R, dense, vec);
  });
}

}  // namespace eu

using namespace eu;

extern "C" {

int eu_optim_momentum(eu_ctx* c, float* var, float* accum, int64_t N, int32_t D, const float* grad, const int64_t* rows,
                      int64_t R, float lr, float momentum) {
  return eu::momentum("eu_optim_momentum", c, var, accum, N, D, grad, rows, R, lr, momentum, EU_FEAT_F32, SrKey{0, nullptr, 0});
}

int eu_optim_adagrad(eu_ctx* c, float* var, float* accum, int64_t N, int32_t D, const float* grad, const int64_t* rows,
                     int64_t R, float lr) {
  return eu::adagrad("eu_optim_adagrad", c, var, accum, N, D, grad, rows, R, lr, EU_FEAT_F32, SrKey{0, nullptr, 0});
}

int eu_optim_adam(eu_ctx* c, float* var, float* m, float* v, int64_t N, int32_t D, const float* grad, const int64_t* rows,
                  int64_t R, const float* powers, float lr, float beta1, float beta2, float epsilon) {
  return eu::adam("eu_optim_adam", c, var, m, v, N, D, grad, rows, R, powers, lr, beta1, beta2, epsilon, EU_FEAT_F32,
                  SrKey{0, nullptr, 0});
}

int eu_optim_momentum_dtype(eu_ctx* c, void* var, void* accum, int64_t N, int32_t D, const float* grad, const int64_t* rows,
                            int64_t R, float lr, float momentum, int32_t dtype, uint64_t seed, const int64_t* step,
                            int32_t tensor) {
  return eu::momentum("eu_optim_momentum_dtype", c, var, accum, N, D, grad, rows, R, lr, momentum, dtype,
                      SrKey{seed, step, (uint32_t)tensor});
}

int eu_optim_adagrad_dtype(eu_ctx* c, void* var, void* accum, int64_t N, int32_t D, const float* grad, const int64_t* rows,
                           int64_t R, float lr, int32_t dtype, uint64_t seed, const int64_t* step, int32_t tensor) {
  return eu::adagrad("eu_optim_adagrad_dtype", c, var, accum, N, D, grad, rows, R, lr, dtype, SrKey{seed, step, (uint32_t)tensor});
}

int eu_optim_adam_dtype(eu_ctx* c, void* var, void* m, void* v, int64_t N, int32_t D, const float* grad, const int64_t* rows,
                        int64_t R, const float* powers, float lr, float beta1, float beta2, float epsilon, int32_t dtype,
                        uint64_t seed, const int64_t* step, int32_t tensor) {
  return eu::adam("eu_optim_adam_dtype", c, var, m, v, N, D, grad, rows, R, powers, lr, beta1, beta2, epsilon, dtype,
                  SrKey{seed, step, (uint32_t)tensor});
}

}  // extern "C"
