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

// columns [d, d + 4) of a row (fewer at its end): one float4 store (VEC) or up to four scalar stores
template <bool VEC>
__device__ __forceinline__ void row_store4(float* __restrict__ row, int d, int dim, float4 v) {
  if (VEC) {
    *reinterpret_cast<float4*>(row + d) = v;
    return;
  }
  row[d] = v.x;
  if (d + 1 < dim) row[d + 1] = v.y;
  if (d + 2 < dim) row[d + 2] = v.z;
  if (d + 3 < dim) row[d + 3] = v.w;
}

// G lanes per distinct id p of the plan (segment [start[p], start[p + 1]) of the stable order perm), 4 columns per lane and
// step.  The group reads the gradient row before it clears it; the stores' rows are written but never read here, so the
// loads of grad_store and rows go through the read-write path.
template <bool VEC>
__global__ void __launch_bounds__(256) k_store_exchange(DistinctPlan P, const int32_t* __restrict__ perm, int64_t n_rows, int dim,
                                                        int G, const float* __restrict__ rows, float* __restrict__ store,
                                                        float* __restrict__ grad_store, float* __restrict__ taken) {
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
    float* s = store + v * dim;
    float* gs = grad_store + v * dim;
    const float* last = rows + (int64_t)__ldg(perm + k1 - 1) * dim;
    for (int d = sub * 4; d < dim; d += G * 4) {
      float4 g = nan4;
      if (real) {
        g = VEC ? *reinterpret_cast<const float4*>(gs + d) : make_float4(gs[d], d + 1 < dim ? gs[d + 1] : 0.f,
                                                                          d + 2 < dim ? gs[d + 2] : 0.f, d + 3 < dim ? gs[d + 3] : 0.f);
        row_store4<VEC>(s, d, dim, row_load4<VEC>(last, d, dim));
        row_store4<VEC>(gs, d, dim, make_float4(0.f, 0.f, 0.f, 0.f));
      }
      for (int64_t k = k0; k < k1; ++k) row_store4<VEC>(taken + (int64_t)__ldg(perm + k) * dim, d, dim, g);
    }
  }
}

// grad_store[key[p]] = __fadd_rn(grad_store[key[p]], vals[p]) elementwise, for the distinct ids p < *nd (not the virtual row)
__global__ void k_store_add(DistinctPlan P, int64_t n_rows, int dim, const float* __restrict__ vals, float* __restrict__ grad_store) {
  const int64_t D = __ldg(P.nd);
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < D * dim; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = t / dim, f = t - p * dim;
    const int64_t v = __ldg(P.key + p);
    if (v < n_rows) grad_store[v * dim + f] = __fadd_rn(grad_store[v * dim + f], __ldg(vals + t));
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

}  // namespace eu

using namespace eu;

extern "C" {

int eu_store_exchange(eu_ctx* c, float* store, float* grad_store, int64_t n_rows, int32_t dim, const int64_t* ids, int64_t M,
                      const float* rows, float* taken) {
  const char* who = "eu_store_exchange";
  int rc = store_check(c, store && grad_store && (M == 0 || (ids && rows && taken)), n_rows, dim, M, who);
  if (rc) return rc;
  EU_CUDA(cudaSetDevice(c->g->device));
  if (M == 0) return EU_OK;
  RowList L;
  int32_t* node;
  float* vals;
  {
    EuProfScope ps(c, "store_exchange_plan", M);
    if ((rc = store_plan(c, ids, M, n_rows, dim, false, 0, &L, &node, &vals, who))) return rc;
  }
  const bool vec = dim % 4 == 0 && aligned16(store) && aligned16(grad_store) && aligned16(rows) && aligned16(taken);
  const int G = group_lanes(ceil_div(dim, 4));
  EuProfScope ps(c, "store_exchange", M);
  auto k = vec ? k_store_exchange<true> : k_store_exchange<false>;
  k<<<stride_grid(M * G), 256, 0, c->stream>>>(L.P, L.ord.perm, n_rows, dim, G, rows, store, grad_store, taken);
  EU_LAUNCHED();
  return EU_OK;
}

int eu_store_accumulate(eu_ctx* c, float* grad_store, int64_t n_rows, int32_t dim, const int64_t* ids, int64_t M, int32_t count,
                        int32_t pool, const float* grad) {
  const char* who = "eu_store_accumulate";
  int rc = store_check(c, grad_store && (M == 0 || (ids && grad)), n_rows, dim, M, who);
  if (rc) return rc;
  if (count < 1 || M % count || (pool != EU_POOL_SUM && pool != EU_POOL_MEAN)) {
    set_error("%s: count = %d must be at least 1 and divide M = %lld, pool must be EU_POOL_SUM or EU_POOL_MEAN", who, (int)count,
              (long long)M);
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
  k_store_add<<<stride_grid(M * dim), 256, 0, c->stream>>>(L.P, n_rows, dim, vals, grad_store);
  EU_LAUNCHED();
  return EU_OK;
}

}  // extern "C"
