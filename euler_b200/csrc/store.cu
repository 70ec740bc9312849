// The per-layer embedding stores of ScalableSageEncoder / ScalableGCNEncoder: the two in-place updates a training step makes
// to a store table and its gradient table, deterministic however often an id repeats.
//
// Reference semantics (file:line in the upstream alibaba/euler tree):
//   _update_store / _optimize_store   tf_euler/python/utils/encoders.py:370-408, 710-748  stores[l][node] = node_embeddings[l]
//                                     (tf.scatter_update); g = gradient_stores[l][node], then those rows zeroed
//   _update_gradient                  the same files  gradient_stores[l][neighbor] += the gradient of the neighbour rows
//                                     (tf.scatter_add)
// With repeated ids tf.scatter_update's winner is unspecified and tf.scatter_add adds through atomics; here both are fixed:
//
// Exchange (store, grad_store, ids [M], rows [M, dim], taken [M, dim]): the ids are planned once by the id-table gradient
// path's plan_rows (segment.cuh), whose stable order lists each distinct id's occurrences in input order.  One lane group
// per distinct id v then, column by column: reads g = grad_store[v], writes taken[i] = g for every occurrence i of v (the
// pre-clear row), store[v] = rows[the LAST occurrence of v] and grad_store[v] = 0.  Each row is owned by one group, so
// there are no races and no atomics.
//
// Accumulate (grad_store, ids [M], grad [M / count, dim], count, pool): grad_store[v] += the sum over the occurrences e of v
// of grad[e / count] (divided by fl(count) as it is read under EU_POOL_MEAN), the gradient of eu_shallow_encode_pool over
// the store.  The sums are the shared path's (sum_distinct_rows, gathered kind): each id's entries in stable order, chunks
// of kSegChunk from +0, the chunk sums in chunk order, into a COO scratch of the distinct ids; k_store_add then adds each
// distinct row into grad_store with one __fadd_rn per element, bounded by the distinct count on the device.
//
// Both calls check the ids (one flag, one read-back) before anything is written; under CUDA-graph capture the check is
// skipped, and an id outside the table is then routed to a virtual row n_rows that is never read or written (its taken
// rows are NaN).  No other host synchronisation.
//
// bf16 stores (T = __nv_bfloat16, the *_dtype entry points: store and grad_store both bf16; rows, taken and grad stay f32).
// Every read widens a stored element exactly to f32; only the writes round.  The exchange's store row is an overwrite, so it
// is rounded to nearest even (feat_st); taken is the gradient row as it was, widened; the cleared row is exact zeros.  The
// accumulation adds the same f32 sum S_v to the widened stored value with the same __fadd_rn and writes it by stochastic
// rounding (sr_st), its random word the first of SrKey{seed, step, tensor}'s for element v dim + f (common.cuh), so an add
// smaller than half an ulp is kept on average.  The 4-wide path needs the bf16 tables aligned to four elements (8 bytes) and
// rows / taken to 16 bytes.
#include <type_traits>

#include "segment.cuh"

namespace eu {

// key[i] = ids[i], or n_rows (flagged) when ids[i] lies outside [0, n_rows); node[i] = i when node is given
__global__ void k_store_keys(const int64_t* __restrict__ ids, int64_t M, int64_t n_rows, int32_t* __restrict__ key,
                             int32_t* __restrict__ node, int* bad) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < M; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t v = __ldg(ids + i);
    const bool ok = v >= 0 && v < n_rows;
    if (!ok) *bad = 1;
    key[i] = (int32_t)(ok ? v : n_rows);
    if (node) node[i] = (int32_t)i;
  }
}

// columns [d, d + 4) of a row of T (fewer at its end), each value rounded to nearest: one 4-wide store (VEC) or up to four
// scalar stores
template <bool VEC, typename T>
__device__ __forceinline__ void row_store4(T* __restrict__ row, int d, int dim, float4 v) {
  if (VEC) {
    rn_st4(row + d, v);
    return;
  }
  row[d] = feat_st<T>(v.x);
  if (d + 1 < dim) row[d + 1] = feat_st<T>(v.y);
  if (d + 2 < dim) row[d + 2] = feat_st<T>(v.z);
  if (d + 3 < dim) row[d + 3] = feat_st<T>(v.w);
}

// G lanes per distinct id p of the plan (segment [start[p], start[p + 1]) of the stable order perm), 4 columns per lane and
// step.  The group reads the gradient row before it clears it; the stores' rows are written but never read here, so the
// loads of grad_store and rows go through the read-write path.  T: the stores' type.
template <bool VEC, typename T>
__global__ void __launch_bounds__(256) k_store_exchange(DistinctPlan P, const int32_t* __restrict__ perm, int64_t n_rows, int dim,
                                                        int G, const float* __restrict__ rows, T* __restrict__ store,
                                                        T* __restrict__ grad_store, float* __restrict__ taken) {
  const int lg = 31 - __clz(G);
  const int sub = (int)(threadIdx.x & (G - 1));
  const int64_t D = __ldg(P.nd);
  const int64_t step = ((int64_t)gridDim.x * blockDim.x) >> lg;
  const float4 nan4 = make_float4(__int_as_float(0x7fc00000), __int_as_float(0x7fc00000), __int_as_float(0x7fc00000),
                                  __int_as_float(0x7fc00000));
  for (int64_t p = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> lg; p < D; p += step) {
    const int64_t v = __ldg(P.key + p);
    const int64_t k0 = __ldg(P.start + p), k1 = __ldg(P.start + p + 1);
    const bool real = v < n_rows;   // false only under capture: the virtual row of the ids outside the table
    T* s = store + v * dim;
    T* gs = grad_store + v * dim;
    const float* last = rows + (int64_t)__ldg(perm + k1 - 1) * dim;
    for (int d = sub * 4; d < dim; d += G * 4) {
      float4 g = nan4;
      if (real) {
        g = row_load4<VEC, T, true>(gs, d, dim);
        row_store4<VEC>(s, d, dim, row_load4<VEC>(last, d, dim));
        row_store4<VEC>(gs, d, dim, make_float4(0.f, 0.f, 0.f, 0.f));
      }
      for (int64_t k = k0; k < k1; ++k) row_store4<VEC>(taken + (int64_t)__ldg(perm + k) * dim, d, dim, g);
    }
  }
}

// grad_store[key[p]] = __fadd_rn(grad_store[key[p]], vals[p]) elementwise, for the distinct ids p < *nd (not the virtual row).
// T = bf16: the stored value is widened, and the sum written by stochastic rounding keyed (seed, *step, tensor, element);
// the f32 kernel never reads the key, which follows its parameters so theirs keep their offsets.
template <typename T>
__global__ void k_store_add(DistinctPlan P, int64_t n_rows, int dim, const float* __restrict__ vals, T* __restrict__ grad_store,
                            unsigned long long seed, const int64_t* __restrict__ step, uint32_t tensor) {
  const int64_t D = __ldg(P.nd);
  const SrKey sk{seed, step, tensor};
  uint32_t s32 = 0;
  if constexpr (!std::is_same<T, float>::value) s32 = (uint32_t)__ldg(step);
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < D * dim; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = t / dim, f = t - p * dim;
    const int64_t v = __ldg(P.key + p);
    if (v < n_rows) {
      const int64_t e = v * dim + f;
      const float x = __fadd_rn(rw_ld(grad_store + e), __ldg(vals + t));
      if constexpr (std::is_same<T, float>::value) grad_store[e] = x;
      else grad_store[e] = sr_st(x, sr_bits(sk, s32, (unsigned long long)e).x);
    }
  }
}

static int store_check(eu_ctx* c, bool ok, int64_t n_rows, int32_t dim, int64_t M, const char* who) {
  if (!c || !ok || n_rows < 1 || dim < 1 || M < 0) {
    set_error("%s: bad argument", who);
    return EU_ERR_INVALID;
  }
  if (n_rows >= ((int64_t)1 << 31) - 1 || M >= ((int64_t)1 << 31) || !entries_fit(M)) {
    set_error("%s: 2^31 or more table rows or ids are not supported", who);
    return EU_ERR_UNSUPPORTED;
  }
  return EU_OK;
}

// The prologue both calls share, in the ctx scratch laid out as
//   flag (256 B) | key [M] | node [M] (with_node) | vals [M, dim] (vals_dim) | the ids' order and distinct-id plan
// the ids' keys (and the entries' identity rows), then, outside capture, the flag read back: an id outside [0, n_rows)
// returns EU_ERR_INVALID before any table is touched.  Then the plan.  *L and *tail (vals) are the caller's.
static int store_plan(eu_ctx* c, const int64_t* ids, int64_t M, int64_t n_rows, int dim, bool with_node, int vals_dim, RowList* L,
                      int32_t** node, float** vals, const char* who) {
  cudaStream_t s = c->stream;
  const size_t o_key = 256, o_node = o_key + a256(4 * (size_t)M), o_vals = o_node + (with_node ? a256(4 * (size_t)M) : 0);
  const size_t o_plan = o_vals + a256(4 * (size_t)M * vals_dim);
  int rc = ctx_misc(c, (int64_t)(o_plan + row_plan_bytes(M, n_rows + 1, dim)));
  if (rc) return rc;
  char* m = (char*)c->d_misc;
  int32_t* flag = (int32_t*)m;
  L->E = M;
  L->n_rows = n_rows + 1;   // the virtual row n_rows of the ids outside the table
  L->key = (int32_t*)(m + o_key);
  *node = with_node ? (int32_t*)(m + o_node) : nullptr;
  *vals = (float*)(m + o_vals);
  EU_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), s));
  k_store_keys<<<stride_grid(M), 256, 0, s>>>(ids, M, n_rows, L->key, *node, flag);
  EU_LAUNCHED();
  cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
  EU_CUDA(cudaStreamIsCapturing(s, &st));
  if (st == cudaStreamCaptureStatusNone) {
    bool bad = false;
    if ((rc = read_back(c, flag, &bad, 0, nullptr, nullptr))) return rc;
    if (bad) {
      set_error("%s: an id lies outside the table's rows [0, %lld)", who, (long long)n_rows);
      return EU_ERR_INVALID;
    }
  }
  return plan_rows(c, m + o_plan, L);
}

static int store_exchange(eu_ctx* c, void* store, void* grad_store, int64_t n_rows, int32_t dim, const int64_t* ids, int64_t M,
                          const float* rows, float* taken, int32_t dtype, const char* who) {
  int rc = store_check(c, store && grad_store && (M == 0 || (ids && rows && taken)), n_rows, dim, M, who);
  if (rc) return rc;
  if ((rc = dtype_check(dtype, who, "store"))) return rc;
  EU_CUDA(cudaSetDevice(c->g->device));
  if (M == 0) return EU_OK;
  RowList L;
  int32_t* node;
  float* vals;
  {
    EuProfScope ps(c, "store_exchange_plan", M);
    if ((rc = store_plan(c, ids, M, n_rows, dim, false, 0, &L, &node, &vals, who))) return rc;
  }
  const bool vec = dim % 4 == 0 && aligned4_elems(store, dtype) && aligned4_elems(grad_store, dtype) && aligned16(rows) &&
                   aligned16(taken);
  const int G = group_lanes(ceil_div(dim, 4));
  EuProfScope ps(c, "store_exchange", M);
  with_dtype(dtype, [&](auto t) {
    using T = typename decltype(t)::type;
    auto k = vec ? k_store_exchange<true, T> : k_store_exchange<false, T>;
    k<<<stride_grid(M * G), 256, 0, c->stream>>>(L.P, L.ord.perm, n_rows, dim, G, rows, (T*)store, (T*)grad_store, taken);
  });
  EU_LAUNCHED();
  return EU_OK;
}

static int store_accumulate(eu_ctx* c, void* grad_store, int64_t n_rows, int32_t dim, const int64_t* ids, int64_t M, int32_t count,
                            int32_t pool, const float* grad, int32_t dtype, uint64_t seed, const int64_t* step, int32_t tensor,
                            const char* who) {
  int rc = store_check(c, grad_store && (M == 0 || (ids && grad)), n_rows, dim, M, who);
  if (rc) return rc;
  if (count < 1 || M % count || (pool != EU_POOL_SUM && pool != EU_POOL_MEAN)) {
    set_error("%s: count = %d must be at least 1 and divide M = %lld, pool must be EU_POOL_SUM or EU_POOL_MEAN", who, (int)count,
              (long long)M);
    return EU_ERR_INVALID;
  }
  if (!dtype_ok(dtype) || (dtype == EU_FEAT_BF16 && !step)) {
    set_error("%s: bad argument (dtype EU_FEAT_F32 or EU_FEAT_BF16, and a bf16 gradient store needs the device step counter)",
              who);
    return EU_ERR_INVALID;
  }
  EU_CUDA(cudaSetDevice(c->g->device));
  if (M == 0) return EU_OK;
  RowList L;
  int32_t* node;
  float* vals;
  {
    EuProfScope ps(c, "store_accumulate_plan", M);
    if ((rc = store_plan(c, ids, M, n_rows, dim, true, dim, &L, &node, &vals, who))) return rc;
  }
  EuProfScope ps(c, "store_accumulate", M);
  RowEntries R;   // the gathered kind: entry e's row is row e / count of grad
  R.n_src = M;
  R.gt = grad;
  R.node = node;
  R.ld = dim;
  R.group = count;
  R.pool_den = pool == EU_POOL_MEAN ? (float)count : 0.f;
  if ((rc = sum_distinct_rows(c, R, L, dim, false, vals, nullptr))) return rc;
  with_dtype(dtype, [&](auto t) {   // an f32 store never reads the key
    using T = typename decltype(t)::type;
    k_store_add<T><<<stride_grid(M * dim), 256, 0, c->stream>>>(L.P, n_rows, dim, vals, (T*)grad_store, seed, step, (uint32_t)tensor);
  });
  EU_LAUNCHED();
  return EU_OK;
}

}  // namespace eu

using namespace eu;

extern "C" {

int eu_store_exchange(eu_ctx* c, float* store, float* grad_store, int64_t n_rows, int32_t dim, const int64_t* ids, int64_t M,
                      const float* rows, float* taken) {
  return store_exchange(c, store, grad_store, n_rows, dim, ids, M, rows, taken, EU_FEAT_F32, "eu_store_exchange");
}

int eu_store_accumulate(eu_ctx* c, float* grad_store, int64_t n_rows, int32_t dim, const int64_t* ids, int64_t M, int32_t count,
                        int32_t pool, const float* grad) {
  return store_accumulate(c, grad_store, n_rows, dim, ids, M, count, pool, grad, EU_FEAT_F32, 0, nullptr, 0, "eu_store_accumulate");
}

int eu_store_exchange_dtype(eu_ctx* c, void* store, void* grad_store, int64_t n_rows, int32_t dim, const int64_t* ids, int64_t M,
                            const float* rows, float* taken, int32_t dtype) {
  return store_exchange(c, store, grad_store, n_rows, dim, ids, M, rows, taken, dtype, "eu_store_exchange_dtype");
}

int eu_store_accumulate_dtype(eu_ctx* c, void* grad_store, int64_t n_rows, int32_t dim, const int64_t* ids, int64_t M,
                              int32_t count, int32_t pool, const float* grad, int32_t dtype, uint64_t seed, const int64_t* step,
                              int32_t tensor) {
  return store_accumulate(c, grad_store, n_rows, dim, ids, M, count, pool, grad, dtype, seed, step, tensor,
                          "eu_store_accumulate_dtype");
}

}  // extern "C"
