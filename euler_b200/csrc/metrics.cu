// The streaming metrics of tf_euler/python/utils/metrics.py on the device: auc_score (tf.metrics.auc at num_thresholds T,
// trapezoidal ROC), f1_score (tf.metrics.true_positives / false_negatives / false_positives) and acc_score
// (tf.metrics.accuracy).  Each call adds one batch's counts to float32 state vectors the caller owns and writes the value of
// the new state, as the update op of the TF 1.x metric returns it.  The constants follow TF 1.x metrics_impl.py.
//
// AUC.  Threshold i of T is t[0] = fl32(-1e-7), t[T-1] = fl32(1 + 1e-7) and t[i] = fl32(i / (T - 1)) in between, each
// computed in double and rounded once; the table is strictly increasing for every T in [2, 16384] with t[0] < 0 and
// t[T-1] > 1.  A prediction p (in [0, 1]) falls in bucket b(p) = #{i : t[i] < p}, in [1, T-1]; it is positive at threshold
// i iff i < b(p).  k_auc_hist counts each batch's labels per bucket in u32 shared histograms, one per block (positive label:
// any nonzero value, NaN included), added into u64 global ones with integer atomics, so the counts are exact and do not
// depend on the launch.  k_auc_finish turns them into the four per-threshold counts with prefix sums (fn[i] = positives in
// buckets <= i, tp[i] the rest; tn and fp likewise for the negatives), rounds each count once to f32 and adds it to the state
// with one f32 add, then writes the value:
//   rec[i] = (tp + 1e-6) / ((tp + fn) + 1e-6)     fpr[i] = fp / ((fp + tn) + 1e-6)
//   term[i] = (fpr[i] - fpr[i+1]) * ((rec[i] + rec[i+1]) / 2),  i < T - 1
// each op one round-to-nearest f32 op (no contraction).  Lane j of kAucThreads adds term[j], term[j + kAucThreads], .. from +0
// left to right, and the lanes' sums are added by a tree: lane j += lane j + s for s = kAucThreads / 2 .. 1.
// A batch with a prediction outside [0, 1] (NaN included) is not counted: the state is untouched and refused += 1.  The
// value is NaN while refused > 0.
//
// F1 and accuracy.  k_count counts, with integers, tp, fn, fp (labels and floor(p + 0.5) cast to bool: nonzero, NaN included,
// is true) and correct (floor(p + 0.5) == label, NaN never equal); k_count_finish rounds each count once to f32, adds it to
// the state and writes the value.
//
// No call synchronises with the host (once the ctx scratch has grown to T) and no float atomics are used: the state and
// value bits depend on the inputs only, and every call can be captured in a CUDA graph.
#include "internal.h"

namespace eu {

constexpr int kHistThreads = 512;     // k_auc_hist and k_count blocks
constexpr int kHistPerBlock = 4096;   // elements per block before the grid is capped at 4 blocks per SM
constexpr int kAucThreads = 1024;     // the one k_auc_finish block: it fixes the order of the value's sum

__device__ __forceinline__ float f32_nan() { return __int_as_float(0x7fc00000); }

// threshold i of T (see the top of the file)
__device__ __forceinline__ float auc_threshold(int i, int T) {
  if (i == 0) return __double2float_rn(-1e-7);
  if (i == T - 1) return __double2float_rn(1.0 + 1e-7);
  return __double2float_rn(__ddiv_rn((double)i, (double)(T - 1)));
}

// #{i : t[i] < p} for p in [0, 1]: t[0] < 0 <= p ends the first loop and t[T-1] > 1 >= p the second, so the result lies in
// [1, T-1].  The guess floor(p (T - 1)) is within a step or two of it.
__device__ __forceinline__ int auc_bucket(float p, int T) {
  int i = (int)((double)p * (double)(T - 1));
  if (i > T - 2) i = T - 2;
  while (!(auc_threshold(i, T) < p)) --i;
  while (auc_threshold(i + 1, T) < p) ++i;
  return i + 1;
}

// hist u64[2][T + 1] (negative labels, then positive) += this batch's bucket counts; *bad = 1 if a prediction is outside
// [0, 1] or NaN.  Dynamic shared memory: u32[2][T + 1].  A block handles far fewer than 2^32 elements (the grid covers N in
// blocks of at least kHistPerBlock up to the cap), so its u32 counts cannot wrap.
__global__ void __launch_bounds__(kHistThreads) k_auc_hist(const float* __restrict__ labels, const float* __restrict__ pred,
                                                           int64_t N, int T, unsigned long long* __restrict__ hist,
                                                           unsigned* __restrict__ bad) {
  extern __shared__ unsigned sh_hist[];
  const int nb = T + 1;
  for (int k = threadIdx.x; k < 2 * nb; k += blockDim.x) sh_hist[k] = 0u;
  __syncthreads();
  bool out = false;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < N; e += (int64_t)gridDim.x * blockDim.x) {
    const float p = __ldg(pred + e);
    if (!(p >= 0.f && p <= 1.f)) {
      out = true;
      continue;
    }
    atomicAdd(sh_hist + (__ldg(labels + e) != 0.f ? nb : 0) + auc_bucket(p, T), 1u);
  }
  if (out) *bad = 1u;
  __syncthreads();
  for (int k = threadIdx.x; k < 2 * nb; k += blockDim.x)
    if (sh_hist[k]) atomicAdd(hist + k, (unsigned long long)sh_hist[k]);
}

// rec and fpr of threshold i of the state
__device__ __forceinline__ void auc_point(const float* tp, const float* fn, const float* tn, const float* fp, int i, float* rec,
                                          float* fpr) {
  const float eps = 1e-6f;
  *rec = __fdiv_rn(__fadd_rn(tp[i], eps), __fadd_rn(__fadd_rn(tp[i], fn[i]), eps));
  *fpr = __fdiv_rn(fp[i], __fadd_rn(__fadd_rn(fp[i], tn[i]), eps));
}

// one block of kAucThreads: the state += the batch's per-threshold counts (unless *bad), then the value (see the top of the file)
__global__ void __launch_bounds__(kAucThreads) k_auc_finish(const unsigned long long* __restrict__ hist,
                                                            const unsigned* __restrict__ bad, int T, float* tp, float* fn,
                                                            float* tn, float* fp, int64_t* refused, float* value) {
  __shared__ unsigned long long s_neg[kAucThreads], s_pos[kAucThreads];
  __shared__ float part[kAucThreads];
  const int j = threadIdx.x;
  if (*bad) {   // block-uniform
    if (j == 0) {
      *refused += 1;
      *value = f32_nan();
    }
    return;
  }
  // lane j owns the buckets [lo, hi); an inclusive scan of the lanes' sums gives each lane its starting prefix
  const int nb = T + 1, per = (nb + kAucThreads - 1) / kAucThreads;
  const int lo = min(j * per, nb), hi = min(lo + per, nb);
  unsigned long long cn = 0, cp = 0;
  for (int b = lo; b < hi; ++b) {
    cn += hist[b];
    cp += hist[nb + b];
  }
  s_neg[j] = cn;
  s_pos[j] = cp;
  __syncthreads();
  for (int o = 1; o < kAucThreads; o <<= 1) {
    const unsigned long long an = j >= o ? s_neg[j - o] : 0ull, ap = j >= o ? s_pos[j - o] : 0ull;
    __syncthreads();
    s_neg[j] += an;
    s_pos[j] += ap;
    __syncthreads();
  }
  const unsigned long long n_neg = s_neg[kAucThreads - 1], n_pos = s_pos[kAucThreads - 1];
  cn = s_neg[j] - cn;
  cp = s_pos[j] - cp;
  for (int b = lo; b < hi && b < T; ++b) {   // threshold b: buckets 0 .. b are at or below it
    cn += hist[b];
    cp += hist[nb + b];
    fn[b] = __fadd_rn(fn[b], __ull2float_rn(cp));
    tp[b] = __fadd_rn(tp[b], __ull2float_rn(n_pos - cp));
    tn[b] = __fadd_rn(tn[b], __ull2float_rn(cn));
    fp[b] = __fadd_rn(fp[b], __ull2float_rn(n_neg - cn));
  }
  __syncthreads();   // the block's state writes are visible to the whole block
  float acc = 0.f;
  for (int i = j; i < T - 1; i += kAucThreads) {
    float r0, f0, r1, f1;
    auc_point(tp, fn, tn, fp, i, &r0, &f0);
    auc_point(tp, fn, tn, fp, i + 1, &r1, &f1);
    acc = __fadd_rn(acc, __fmul_rn(__fsub_rn(f0, f1), __fdiv_rn(__fadd_rn(r0, r1), 2.f)));
  }
  part[j] = acc;
  __syncthreads();
  for (int s = kAucThreads / 2; s > 0; s >>= 1) {
    if (j < s) part[j] = __fadd_rn(part[j], part[j + s]);
    __syncthreads();
  }
  if (j == 0) *value = *refused > 0 ? f32_nan() : part[0];
}

// counts u64[4] += (tp, fn, fp, correct) of the batch
__global__ void __launch_bounds__(kHistThreads) k_count(const float* __restrict__ labels, const float* __restrict__ pred,
                                                        int64_t N, unsigned long long* __restrict__ counts) {
  __shared__ unsigned long long sh[4][kHistThreads / 32];
  unsigned long long c[4] = {0ull, 0ull, 0ull, 0ull};
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < N; e += (int64_t)gridDim.x * blockDim.x) {
    const float l = __ldg(labels + e);
    const float p = floorf(__fadd_rn(__ldg(pred + e), 0.5f));
    const bool lb = l != 0.f, pb = p != 0.f;
    c[0] += lb && pb;
    c[1] += lb && !pb;
    c[2] += !lb && pb;
    c[3] += p == l;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    for (int o = 16; o > 0; o >>= 1) c[k] += __shfl_xor_sync(0xffffffffu, c[k], o);
    if (lane == 0) sh[k][warp] = c[k];
  }
  __syncthreads();
  if (threadIdx.x >= 4) return;
  unsigned long long t = 0;
  for (int w = 0; w < kHistThreads / 32; ++w) t += sh[threadIdx.x][w];
  if (t) atomicAdd(counts + threadIdx.x, t);
}

// one thread: the state += the batch's counts, then the value.  correct (device, may be null) replaces counts[3], and N is
// then the number of predictions it counts.
__global__ void k_count_finish(int kind, const unsigned long long* __restrict__ counts, const int64_t* __restrict__ correct,
                               int64_t N, float* state, float* value) {
  if (kind == EU_METRIC_F1) {
    const float eps = 1e-7f;
    const float tp = state[0] = __fadd_rn(state[0], __ull2float_rn(counts[0]));
    const float fn = state[1] = __fadd_rn(state[1], __ull2float_rn(counts[1]));
    const float fp = state[2] = __fadd_rn(state[2], __ull2float_rn(counts[2]));
    const float p = __fdiv_rn(tp, __fadd_rn(__fadd_rn(eps, tp), fp));
    const float r = __fdiv_rn(tp, __fadd_rn(__fadd_rn(eps, tp), fn));
    *value = __fdiv_rn(__fmul_rn(__fmul_rn(2.f, p), r), __fadd_rn(__fadd_rn(p, r), eps));
    return;
  }
  const float add = correct ? __ll2float_rn(*correct) : __ull2float_rn(counts[3]);
  const float total = state[0] = __fadd_rn(state[0], add);
  const float count = state[1] = __fadd_rn(state[1], __ll2float_rn(N));
  *value = count > 0.f ? __fdiv_rn(total, count) : 0.f;
}

// the grid of k_auc_hist and k_count over N > 0 elements
static int grid_for(eu_ctx* c, int64_t N, unsigned* blocks) {
  int sms = 0;
  EU_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->g->device));
  const int64_t want = ceil_div(N, kHistPerBlock), cap = 4 * (int64_t)sms;
  *blocks = (unsigned)(want < cap ? want : cap);
  return EU_OK;
}

}  // namespace eu

using namespace eu;

extern "C" {

int eu_metric_auc_update(eu_ctx* c, const float* labels, const float* predictions, int64_t N, int32_t T, float* tp, float* fn,
                         float* tn, float* fp, int64_t* refused, float* value) {
  const char* who = "eu_metric_auc_update";
  if (!c || N < 0 || T < 2 || T > EU_METRIC_AUC_MAX_THRESHOLDS || !tp || !fn || !tn || !fp || !refused || !value ||
      (N > 0 && (!labels || !predictions))) {
    set_error("%s: bad argument (N >= 0, 2 <= T <= %d, labels and predictions when N > 0, four state vectors, refused and "
              "value)", who, EU_METRIC_AUC_MAX_THRESHOLDS);
    return EU_ERR_INVALID;
  }
  EU_CUDA(cudaSetDevice(c->g->device));
  // bad u32 (256 B) | hist u64[2][T + 1]
  const size_t hist_bytes = 2 * (size_t)(T + 1) * sizeof(unsigned long long);
  int rc;
  if ((rc = ctx_misc(c, (int64_t)(256 + hist_bytes)))) return rc;
  char* m = (char*)c->d_misc;
  unsigned* bad = (unsigned*)m;
  unsigned long long* hist = (unsigned long long*)(m + 256);
  cudaStream_t s = c->stream;
  EuProfScope ps(c, "metric_auc", N);
  EU_CUDA(cudaMemsetAsync(m, 0, 256 + hist_bytes, s));
  if (N > 0) {
    unsigned blocks;
    if ((rc = grid_for(c, N, &blocks))) return rc;
    const size_t shb = 2 * (size_t)(T + 1) * sizeof(unsigned);
    if (shb > 48 * 1024) EU_CUDA(cudaFuncSetAttribute(k_auc_hist, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shb));
    k_auc_hist<<<blocks, kHistThreads, shb, s>>>(labels, predictions, N, T, hist, bad);
    EU_LAUNCHED();
  }
  k_auc_finish<<<1, kAucThreads, 0, s>>>(hist, bad, T, tp, fn, tn, fp, refused, value);
  EU_LAUNCHED();
  return EU_OK;
}

int eu_metric_count_update(eu_ctx* c, int32_t kind, const float* labels, const float* predictions, int64_t N,
                           const int64_t* correct, float* state, float* value) {
  const char* who = "eu_metric_count_update";
  const bool data = !correct;
  if (!c || N < 0 || !state || !value || (kind != EU_METRIC_F1 && kind != EU_METRIC_ACC) ||
      (data && N > 0 && (!labels || !predictions)) || (!data && (kind != EU_METRIC_ACC || labels || predictions))) {
    set_error("%s: bad argument (kind EU_METRIC_F1 or EU_METRIC_ACC, N >= 0, state and value, and either labels and "
              "predictions or, for EU_METRIC_ACC only, correct)", who);
    return EU_ERR_INVALID;
  }
  EU_CUDA(cudaSetDevice(c->g->device));
  int rc;
  if ((rc = ctx_misc(c, 256))) return rc;
  unsigned long long* counts = (unsigned long long*)c->d_misc;
  cudaStream_t s = c->stream;
  EuProfScope ps(c, "metric_count", N);
  if (data) {
    EU_CUDA(cudaMemsetAsync(counts, 0, 4 * sizeof(unsigned long long), s));
    if (N > 0) {
      unsigned blocks;
      if ((rc = grid_for(c, N, &blocks))) return rc;
      k_count<<<blocks, kHistThreads, 0, s>>>(labels, predictions, N, counts);
      EU_LAUNCHED();
    }
  }
  k_count_finish<<<1, 1, 0, s>>>(kind, counts, correct, N, state, value);
  EU_LAUNCHED();
  return EU_OK;
}

}  // extern "C"
