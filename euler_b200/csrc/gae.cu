// The reconstruction step of the graph auto-encoders, GAE and VGAE, forward and backward: the dot products of each source
// row with its K positive and K negative context rows, the sigmoid cross-entropy mean, the accuracy count and, for the
// variational form, the reparameterised rows and the KL mean.  The inputs are encoder rows, not table ids.
//
// Reference semantics (file:line in the upstream alibaba/euler tree):
//   BaseGraphAutoEncoder.__call__         tf_euler/python/mp_utils/base_gae.py:45-74
//   VariationalGraphAutoEncoder           examples/gae/gae.py:90-160 (embed: the reparameterisation; kl; __call__)
//   acc_score                             tf_euler/python/utils/metrics.py (floor(predict + 0.5) == label, the batch's share)
//
// Three sets of rows s = 0 (src, [B, D]), 1 (pos, [B, K, D]), 2 (negs, [B, K, D]).  Row r of set s is z = mu, or in the
// variational form with noise z = mu + (radius noise) sqrt(exp(log_var)), each element in f32 in that order; without noise
// (VGAE with train=False) z = mu.  Item (b, j) of the launch, j in [-1, 2K), is the src row b's KL (j = -1) or the logit
// x_bj = <z_src[b], z_ctx[b, j]> with ctx j = pos[b, j] for j < K and negs[b, j - K] after.
//   dot: lane l of a group of G lanes (G = the power of two >= ceil(D / 4), at most 32) adds with __fmaf_rn from +0 the columns
//        of its 4-column chunks l, l + G, .., each chunk left to right; then a butterfly over the G lanes, xor distances G/2 .. 1.
//   kl of a row: the f32 elements -0.5 (((lv - exp(lv)) - mu^2) + 1), each lane adding its own in f64 in column order, then
//        the same butterfly in f64.  Item (b, j) owns the KL of ctx j, item (b, -1) that of src b.
//   xent: the f32 term max(x, 0) - x z + log1p(exp(-|x|)) (z = 1 for j < K), kept in f64 per item.
// Then loss = fl32(sum of the 2BK xent terms / 2BK) (+ fl32(sum of the B (2K + 1) row KLs / B D (2K + 1))), each sum one
// k_f64_mean over the items in (b, j) order; correct = #{floor(sigmoid(x) + 0.5) == z}, sigmoid(x) = 1 / (1 + exp(-x)) in f32
// as torch.sigmoid computes it.  No atomics and no host synchronisation: the bits depend on B, K and D only.
//
// Backward, with g the upstream gradient (a device scalar): gx = g / fl(2BK), gk = g / fl(B D (2K + 1)), and per logit
//   c_bj = -gx / (1 + exp(x)) (j < K: (sigmoid(x) - 1) gx)      c_bj = gx / (1 + exp(-x)) (j >= K: sigmoid(x) gx)
//   dz_ctx[b, j] = c_bj z_src[b]      dz_src[b] = sum over j of c_bj z_ctx[b, j] (fma from +0, j order)
//   g_mu = dz (+ gk mu)      g_log_var = dz ((radius noise) 0.5 sqrt(exp(lv))) + gk 0.5 (exp(lv) - 1)
// Every output element is written by one thread: item (b, j) writes ctx j's rows, item (b, -1) src b's.
#include "segment.cuh"

namespace eu {

struct GaeRows {           // one set of rows, each row D floats: mu, and for the variational form log_var and noise
  const float* mu;
  const float* lv;         // null: not variational
  const float* nz;         // null: z = mu
};

struct GaeIn {
  GaeRows s[3];            // src, pos, negs
  float radius;
};

struct GaeGrad {
  float* mu[3];
  float* lv[3];
};

// the chunk [d, d + 4) of row r of set s: mu, log_var (zero when not variational) and z
// set s's pointer of a field, chosen by value: indexing the kernel parameter by a runtime s would copy it to the stack
template <class T>
__device__ __forceinline__ T gae_pick(int s, T p0, T p1, T p2) { return s == 0 ? p0 : (s == 1 ? p1 : p2); }

template <bool VEC, bool VAR>
__device__ __forceinline__ void gae_chunk(const GaeIn& in, int s, int64_t r, int d, int D, float4* mu, float4* lv, float4* z) {
  *mu = row_load4<VEC>(gae_pick(s, in.s[0].mu, in.s[1].mu, in.s[2].mu) + r * D, d, D);
  *z = *mu;
  *lv = make_float4(0.f, 0.f, 0.f, 0.f);
  if (!VAR) return;
  *lv = row_load4<VEC>(gae_pick(s, in.s[0].lv, in.s[1].lv, in.s[2].lv) + r * D, d, D);
  const float* nz = gae_pick(s, in.s[0].nz, in.s[1].nz, in.s[2].nz);
  if (!nz) return;
  const float4 n = row_load4<VEC>(nz + r * D, d, D);
  const float rad = in.radius;
  z->x = __fadd_rn(mu->x, __fmul_rn(__fmul_rn(rad, n.x), sqrtf(expf(lv->x))));
  z->y = __fadd_rn(mu->y, __fmul_rn(__fmul_rn(rad, n.y), sqrtf(expf(lv->y))));
  z->z = __fadd_rn(mu->z, __fmul_rn(__fmul_rn(rad, n.z), sqrtf(expf(lv->z))));
  z->w = __fadd_rn(mu->w, __fmul_rn(__fmul_rn(rad, n.w), sqrtf(expf(lv->w))));
}

__device__ __forceinline__ float gae_kl(float mu, float lv) {
  return __fmul_rn(-0.5f, __fadd_rn(__fsub_rn(__fsub_rn(lv, expf(lv)), __fmul_rn(mu, mu)), 1.f));
}

// acc += the KL elements of the first n columns of a chunk, left to right, in f64
__device__ __forceinline__ double gae_kl4(float4 mu, float4 lv, double acc, int n) {
  acc += (double)gae_kl(mu.x, lv.x);
  if (n > 1) acc += (double)gae_kl(mu.y, lv.y);
  if (n > 2) acc += (double)gae_kl(mu.z, lv.z);
  if (n > 3) acc += (double)gae_kl(mu.w, lv.w);
  return acc;
}

// acc += the dot of the first n columns of two chunks, one __fmaf_rn per column, left to right
__device__ __forceinline__ float gae_fma4(float4 a, float4 b, float acc, int n) {
  acc = __fmaf_rn(a.x, b.x, acc);
  if (n > 1) acc = __fmaf_rn(a.y, b.y, acc);
  if (n > 2) acc = __fmaf_rn(a.z, b.z, acc);
  if (n > 3) acc = __fmaf_rn(a.w, b.w, acc);
  return acc;
}

// the set and row of context j of pair row b
__device__ __forceinline__ int gae_ctx(int64_t b, int K, int j, int64_t* r) {
  *r = b * K + (j < K ? j : j - K);
  return j < K ? 1 : 2;
}

// G lanes per item (b, j), items in (b, j) order with j = -1 first; see the top of the file
template <bool VEC, bool VAR>
__global__ void __launch_bounds__(256) k_gae_fwd(GaeIn in, int64_t B, int K, int D, int G, float* __restrict__ logits,
                                                 double* __restrict__ xterm, double* __restrict__ kterm) {
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t item = tid >> (31 - __clz(G));
  const int sub = (int)(tid & (G - 1));
  const int J = 2 * K;
  if (item >= B * (J + 1)) return;   // group-uniform
  const unsigned gm = group_mask(G);
  const int64_t b = item / (J + 1);
  const int j = (int)(item - b * (J + 1)) - 1;
  if (!VAR && j < 0) return;   // a src item only sums its row's KL
  int64_t cr = b;
  const int cs = j < 0 ? 0 : gae_ctx(b, K, j, &cr);
  float dot = 0.f;
  double kl = 0.0;
  for (int d = sub * 4; d < D; d += G * 4) {
    const int n = D - d < 4 ? D - d : 4;
    float4 mu, lv, zc;
    gae_chunk<VEC, VAR>(in, cs, cr, d, D, &mu, &lv, &zc);
    if (VAR) kl = gae_kl4(mu, lv, kl, n);
    if (j >= 0) {
      float4 smu, slv, zs;
      gae_chunk<VEC, VAR>(in, 0, b, d, D, &smu, &slv, &zs);
      dot = gae_fma4(zs, zc, dot, n);
    }
  }
  for (int o = G >> 1; o > 0; o >>= 1) {
    dot = __fadd_rn(dot, __shfl_xor_sync(gm, dot, o, G));
    if (VAR) kl += __shfl_xor_sync(gm, kl, o, G);
  }
  if (sub != 0) return;
  if (VAR) kterm[item] = kl;
  if (j < 0) return;
  logits[b * J + j] = dot;
  float t = fmaxf(dot, 0.f);
  if (j < K) t = __fsub_rn(t, dot);
  xterm[b * J + j] = (double)__fadd_rn(t, log1pf(expf(-fabsf(dot))));
}

// *correct = #{floor(sigmoid(x) + 0.5) == z} over the N = 2BK logits, *loss = means[0] (+ means[1]); one block of kMeanThreads
__global__ void __launch_bounds__(kMeanThreads) k_gae_finish(const float* __restrict__ logits, int64_t N, int K,
                                                             const float* __restrict__ means, bool var, float* __restrict__ loss,
                                                             int64_t* __restrict__ correct) {
  __shared__ long long sh[kMeanThreads];
  long long cnt = 0;
  for (int64_t e = threadIdx.x; e < N; e += kMeanThreads) {
    const float x = __ldg(logits + e);
    const float p = floorf(__fadd_rn(__fdiv_rn(1.f, __fadd_rn(1.f, expf(-x))), 0.5f));
    cnt += p == ((int)(e % (2 * K)) < K ? 1.f : 0.f);
  }
  sh[threadIdx.x] = cnt;
  __syncthreads();
  for (int s = kMeanThreads / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x != 0) return;
  *correct = sh[0];
  *loss = var ? __fadd_rn(means[0], means[1]) : means[0];
}

// c_bj of the logit x (see the top of the file)
__device__ __forceinline__ float gae_coef(float x, bool positive, float gx) {
  return positive ? __fdiv_rn(-gx, __fadd_rn(1.f, expf(x))) : __fdiv_rn(gx, __fadd_rn(1.f, expf(-x)));
}

// writes the gradients of the chunk [d, d + n) of row r of set s from dz = dL/dz
template <bool VEC, bool VAR>
__device__ __forceinline__ void gae_store(const GaeIn& in, const GaeGrad& out, int s, int64_t r, int d, int D, int n, float4 dz,
                                          float gk) {
  float4 mu, lv, z;
  gae_chunk<VEC, VAR>(in, s, r, d, D, &mu, &lv, &z);
  float gm[4] = {dz.x, dz.y, dz.z, dz.w}, gl[4] = {0.f, 0.f, 0.f, 0.f};
  if (VAR) {
    const float m[4] = {mu.x, mu.y, mu.z, mu.w}, l[4] = {lv.x, lv.y, lv.z, lv.w};
    float nz[4] = {0.f, 0.f, 0.f, 0.f};
    const float* pn = gae_pick(s, in.s[0].nz, in.s[1].nz, in.s[2].nz);
    if (pn) {
      const float4 v = row_load4<VEC>(pn + r * D, d, D);
      nz[0] = v.x; nz[1] = v.y; nz[2] = v.z; nz[3] = v.w;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float e = expf(l[i]);
      const float dzdl = __fmul_rn(__fmul_rn(__fmul_rn(in.radius, nz[i]), 0.5f), sqrtf(e));
      gl[i] = __fadd_rn(__fmul_rn(gm[i], dzdl), __fmul_rn(gk, __fmul_rn(0.5f, __fsub_rn(e, 1.f))));
      gm[i] = __fadd_rn(gm[i], __fmul_rn(gk, m[i]));
    }
  }
  float* om = gae_pick(s, out.mu[0], out.mu[1], out.mu[2]) + r * D + d;
  float* ol = VAR ? gae_pick(s, out.lv[0], out.lv[1], out.lv[2]) + r * D + d : nullptr;
  if (VEC) {
    *reinterpret_cast<float4*>(om) = make_float4(gm[0], gm[1], gm[2], gm[3]);
    if (VAR) *reinterpret_cast<float4*>(ol) = make_float4(gl[0], gl[1], gl[2], gl[3]);
  } else {
    for (int i = 0; i < n; ++i) {
      om[i] = gm[i];
      if (VAR) ol[i] = gl[i];
    }
  }
}

// G lanes per item (b, j) as in k_gae_fwd: item (b, j) writes ctx j's gradients, item (b, -1) src b's
template <bool VEC, bool VAR>
__global__ void __launch_bounds__(256) k_gae_bwd(GaeIn in, GaeGrad out, const float* __restrict__ grad_loss,
                                                 const float* __restrict__ logits, int64_t B, int K, int D, int G, int64_t Nx,
                                                 int64_t Nk) {
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t item = tid >> (31 - __clz(G));
  const int sub = (int)(tid & (G - 1));
  const int J = 2 * K;
  if (item >= B * (J + 1)) return;
  const int64_t b = item / (J + 1);
  const int j = (int)(item - b * (J + 1)) - 1;
  const float g = __ldg(grad_loss);
  const float gx = __fdiv_rn(g, (float)Nx);
  const float gk = VAR ? __fdiv_rn(g, (float)Nk) : 0.f;
  const float* lrow = logits + b * J;
  for (int d = sub * 4; d < D; d += G * 4) {
    const int n = D - d < 4 ? D - d : 4;
    float4 mu, lv, z, dz;
    if (j >= 0) {
      gae_chunk<VEC, VAR>(in, 0, b, d, D, &mu, &lv, &z);
      const float c = gae_coef(__ldg(lrow + j), j < K, gx);
      dz = make_float4(__fmul_rn(c, z.x), __fmul_rn(c, z.y), __fmul_rn(c, z.z), __fmul_rn(c, z.w));
      int64_t cr;
      const int cs = gae_ctx(b, K, j, &cr);
      gae_store<VEC, VAR>(in, out, cs, cr, d, D, n, dz, gk);
    } else {
      dz = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
      for (int jj = 0; jj < J; ++jj) {
        int64_t cr;
        const int cs = gae_ctx(b, K, jj, &cr);
        gae_chunk<VEC, VAR>(in, cs, cr, d, D, &mu, &lv, &z);
        const float c = gae_coef(__ldg(lrow + jj), jj < K, gx);
        dz.x = __fmaf_rn(c, z.x, dz.x); dz.y = __fmaf_rn(c, z.y, dz.y);
        dz.z = __fmaf_rn(c, z.z, dz.z); dz.w = __fmaf_rn(c, z.w, dz.w);
      }
      gae_store<VEC, VAR>(in, out, 0, b, d, D, n, dz, gk);
    }
  }
}

// The inputs of either pass, checked: EU_ERR_INVALID (nothing written) unless B >= 0, K >= 1, D >= 1, the mu sets given,
// log_var all three sets or none, noise all three or none and only with log_var, and radius finite.
static int gae_check(eu_ctx* c, int64_t B, int32_t K, int32_t D, const float* const* mu, const float* const* log_var,
                     const float* const* noise, float radius, GaeIn* in, const char* who) {
  bool ok = c && B >= 0 && K >= 1 && D >= 1 && mu && isfinite(radius) && (!noise || log_var);
  for (int s = 0; ok && s < 3; ++s)
    ok = (B == 0 || mu[s]) && (!log_var || B == 0 || log_var[s]) && (!noise || B == 0 || noise[s]);
  if (!ok) {
    set_error("%s: bad argument (B >= 0, K >= 1, D >= 1, three mu sets, log_var and noise three sets or none, noise only "
              "with log_var, radius finite)", who);
    return EU_ERR_INVALID;
  }
  if (K >= (1 << 29) || B * (2 * (int64_t)K + 1) >= ((int64_t)1 << 34)) {   // 2K and the grid of B (2K + 1) 32-lane groups
    set_error("%s: K below 2^29 and B (2K + 1) below 2^34 are supported", who);
    return EU_ERR_UNSUPPORTED;
  }
  for (int s = 0; s < 3; ++s)
    in->s[s] = GaeRows{mu[s], log_var ? log_var[s] : nullptr, noise ? noise[s] : nullptr};
  in->radius = radius;
  return EU_OK;
}

static bool gae_aligned(const GaeIn& in, int D) {
  if (D % 4) return false;
  for (int s = 0; s < 3; ++s)
    if (!aligned16(in.s[s].mu) || !aligned16(in.s[s].lv) || !aligned16(in.s[s].nz)) return false;
  return true;
}

}  // namespace eu

using namespace eu;

extern "C" {

int eu_gae_loss(eu_ctx* c, int64_t B, int32_t K, int32_t D, const float* const* mu, const float* const* log_var,
                const float* const* noise, float radius, float* logits, float* loss, int64_t* correct) {
  const char* who = "eu_gae_loss";
  GaeIn in;
  int rc = gae_check(c, B, K, D, mu, log_var, noise, radius, &in, who);
  if (rc) return rc;
  if (!loss || !correct) {
    set_error("%s: bad argument (loss and correct are required)", who);
    return EU_ERR_INVALID;
  }
  EU_CUDA(cudaSetDevice(c->g->device));
  const bool var = log_var != nullptr;
  const int J = 2 * K;
  const int64_t Nx = B * J, items = B * (J + 1);
  // means f32[2] (256 B) | xterm f64[Nx] | kterm f64[items] | logits f32[Nx] when the caller keeps none
  const size_t o_x = 256, o_k = o_x + a256(8 * (size_t)Nx), o_l = o_k + a256(var ? 8 * (size_t)items : 0);
  if ((rc = ctx_misc(c, (int64_t)(o_l + (logits ? 0 : a256(4 * (size_t)Nx)))))) return rc;
  char* m = (char*)c->d_misc;
  float* means = (float*)m;
  double* xterm = (double*)(m + o_x);
  double* kterm = (double*)(m + o_k);
  float* lg = logits ? logits : (float*)(m + o_l);
  cudaStream_t s = c->stream;
  EuProfScope ps(c, "gae_fwd", B);
  if (B > 0) {
    const int G = group_lanes(ceil_div(D, 4));
    const unsigned blocks = (unsigned)ceil_div(items * G, 256);
    const bool vec = gae_aligned(in, D);
    if (var && vec) k_gae_fwd<true, true><<<blocks, 256, 0, s>>>(in, B, K, D, G, lg, xterm, kterm);
    else if (var) k_gae_fwd<false, true><<<blocks, 256, 0, s>>>(in, B, K, D, G, lg, xterm, kterm);
    else if (vec) k_gae_fwd<true, false><<<blocks, 256, 0, s>>>(in, B, K, D, G, lg, xterm, kterm);
    else k_gae_fwd<false, false><<<blocks, 256, 0, s>>>(in, B, K, D, G, lg, xterm, kterm);
    EU_LAUNCHED();
  }
  k_f64_mean<<<1, kMeanThreads, 0, s>>>(xterm, Nx, Nx, means);
  EU_LAUNCHED();
  if (var) {
    k_f64_mean<<<1, kMeanThreads, 0, s>>>(kterm, items, items * D, means + 1);
    EU_LAUNCHED();
  }
  k_gae_finish<<<1, kMeanThreads, 0, s>>>(lg, Nx, K, means, var, loss, correct);
  EU_LAUNCHED();
  return EU_OK;
}

int eu_gae_loss_backward(eu_ctx* c, const float* grad_loss, int64_t B, int32_t K, int32_t D, const float* const* mu,
                         const float* const* log_var, const float* const* noise, float radius, const float* logits,
                         float* const* grad_mu, float* const* grad_log_var) {
  const char* who = "eu_gae_loss_backward";
  GaeIn in;
  int rc = gae_check(c, B, K, D, mu, log_var, noise, radius, &in, who);
  if (rc) return rc;
  const bool var = log_var != nullptr;
  bool ok = grad_loss && grad_mu && (B == 0 || logits) && (!var || grad_log_var);
  for (int s = 0; ok && s < 3; ++s) ok = B == 0 || (grad_mu[s] && (!var || grad_log_var[s]));
  if (!ok) {
    set_error("%s: bad argument (grad_loss, logits, three grad_mu sets and, with log_var, three grad_log_var sets)", who);
    return EU_ERR_INVALID;
  }
  if (B == 0) return EU_OK;
  EU_CUDA(cudaSetDevice(c->g->device));
  GaeGrad out;
  for (int s = 0; s < 3; ++s) {
    out.mu[s] = grad_mu[s];
    out.lv[s] = var ? grad_log_var[s] : nullptr;
  }
  bool vec = gae_aligned(in, D);
  for (int s = 0; s < 3; ++s) vec = vec && aligned16(out.mu[s]) && aligned16(out.lv[s]);
  const int J = 2 * K;
  const int64_t items = B * (J + 1);
  const int G = group_lanes(ceil_div(D, 4));
  const unsigned blocks = (unsigned)ceil_div(items * G, 256);
  cudaStream_t s = c->stream;
  EuProfScope ps(c, "gae_bwd", B);
  if (var && vec) k_gae_bwd<true, true><<<blocks, 256, 0, s>>>(in, out, grad_loss, logits, B, K, D, G, B * J, items * D);
  else if (var) k_gae_bwd<false, true><<<blocks, 256, 0, s>>>(in, out, grad_loss, logits, B, K, D, G, B * J, items * D);
  else if (vec) k_gae_bwd<true, false><<<blocks, 256, 0, s>>>(in, out, grad_loss, logits, B, K, D, G, B * J, items * D);
  else k_gae_bwd<false, false><<<blocks, 256, 0, s>>>(in, out, grad_loss, logits, B, K, D, G, B * J, items * D);
  EU_LAUNCHED();
  return EU_OK;
}

}  // extern "C"
