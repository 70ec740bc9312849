// Layer-wise neighbor sampling and batch adjacency (SURVEY.md section 8f, next-3): FastGCN / AS-GCN / LGCN style dataflows.
// Reference semantics (file:line relative to /root/reference):
//   tf_euler SampleNeighborLayerwiseWithAdj   tf_euler/kernels/sample_neighbor_layerwise_with_adj_op.cc:54-150
//       query v(nodes).sampleLNB(edge_types, n, m, [weight_func,] default_node): per batch row of n nodes, m neighbors drawn from
//       the UNION of their neighbor lists; adj[b, j, k] = 1 iff out[b, k] is a neighbor of nodes[b, j]
//   API_LOCAL_SAMPLE_L                        euler/core/kernels/local_sample_layer_op.cc:41-140
//       candidates = the batch's full neighbors made unique by (dst, type) with their weights SUMMED in listing order, optional
//       sqrt, CompactWeightedCollection over them (sequential f32 prefix), m draws of one uniform each; an empty / zero-weight
//       candidate set fills default_node
//   API_SPARSE_GET_ADJ / tf_euler SparseGetAdj euler/core/kernels/sparse_get_adj_op.cc:34-90, tf_euler/kernels/sparse_get_adj_op.cc
//       adj[b, j, k] = 1 iff an edge (nodes[b, j], nb[b, k], t) exists for a listed type t
// Parity note: the reference enumerates the candidates in the iteration order of a std::unordered_map<std::string, ...> keyed
// by to_string(dst) + to_string(type) (local_sample_layer_op.cc:77-90) -- an order with no meaning that its own tests do not
// pin (neighbor_ops_test.py:142-181 check membership and adj consistency only).  Here the candidates are ordered by
// (dst, type): the candidate SET, every candidate's summed weight (same additions, same order) and hence the sampling
// DISTRIBUTION are identical; which uniform maps to which candidate differs.  tests/ check exactly that.
#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_sort.cuh>
#include <cub/iterator/counting_input_iterator.cuh>
#include <cub/iterator/transform_input_iterator.cuh>

#include <algorithm>

#include "internal.h"
#include "uq.cuh"

namespace eu {

__global__ void k_lw_iota(long long* a, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) a[i] = i;
}
__global__ void k_lw_gather_type(const long long* __restrict__ idx, const int32_t* __restrict__ t, int64_t n, int32_t* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = t[idx[i]];
}
__global__ void k_lw_gather_id(const long long* __restrict__ idx, const unsigned long long* __restrict__ ids, int64_t n,
                               unsigned long long* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = ids[idx[i]];
}
// segment b = the listing entries of batch row b: [ptr[b*n], ptr[(b+1)*n])
struct BatchSeg {
  const long long* ptr; long long n;
  __host__ __device__ long long operator()(long long b) const { return ptr[b * n]; }
};

// One thread per batch row walks its (dst, type)-sorted entries: unique candidates, weights summed in listing order (the
// sorts are stable), optional sqrt, sequential f32 prefix (CompactWeightedCollection::Init, compact_weighted_collection.h:82-97)
// written in place over the entry arrays.  cand_n[b] = candidates, cand_total[b] = their prefix end.
__global__ void k_lw_candidates(const long long* __restrict__ ptr, int64_t batch, int32_t n, const long long* __restrict__ order,
                                const unsigned long long* __restrict__ ids, const float* __restrict__ w, const int32_t* __restrict__ t,
                                int32_t weight_func, unsigned long long* __restrict__ c_id, int32_t* __restrict__ c_t,
                                float* __restrict__ c_cum, int32_t* __restrict__ cand_n, float* __restrict__ cand_total) {
  const int64_t b = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (b >= batch) return;
  const long long lo = ptr[b * n], hi = ptr[(b + 1) * (int64_t)n];
  long long o = lo;       // candidates of this batch row are compacted to [lo, lo + cand_n)
  float run = 0.f;
  long long k = lo;
  while (k < hi) {
    const long long e0 = order[k];
    const unsigned long long id = ids[e0];
    const int32_t ty = t[e0];
    float sum = w[e0];
    long long k2 = k + 1;
    while (k2 < hi) {
      const long long e = order[k2];
      if (ids[e] != id || t[e] != ty) break;
      sum = __fadd_rn(sum, w[e]);
      ++k2;
    }
    if (weight_func == 1) sum = sqrtf(sum);          // local_sample_layer_op.cc:93-101 (float sqrt)
    run = __fadd_rn(run, sum);
    c_id[o] = id; c_t[o] = ty; c_cum[o] = run;
    ++o;
    k = k2;
  }
  cand_n[b] = (int32_t)(o - lo);
  cand_total[b] = run;
}

// serial prefix over the batch rows: how many uniforms the rows before b consumed (count each, only rows that sample)
__global__ void k_lw_positions(const int32_t* __restrict__ cand_n, const float* __restrict__ cand_total, int64_t batch, int32_t count,
                               unsigned long long* __restrict__ pos, EuRngState* rng, bool minstd) {
  if (blockIdx.x || threadIdx.x) return;
  unsigned long long run = 0;
  for (int64_t b = 0; b < batch; ++b) {
    pos[b] = run;
    if (cand_n[b] > 0 && cand_total[b] != 0.f) run += (unsigned long long)count;
  }
  pos[batch] = run;
  if (minstd) { rng->x_prev = rng->x; rng->x = modmul(rng->x, modpow_a(2ull * run)); rng->draws += run; }
  rng->calls += 1;
}

__global__ void k_lw_sample(const long long* __restrict__ ptr, int64_t batch, int32_t n, int32_t count, long long default_node,
                            const unsigned long long* __restrict__ c_id, const float* __restrict__ c_cum, const int32_t* __restrict__ cand_n,
                            const float* __restrict__ cand_total, const unsigned long long* __restrict__ pos, const EuRngState* rng,
                            bool philox, unsigned long long key, long long* __restrict__ out) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= batch * (int64_t)count) return;
  const int64_t b = i / count;
  const int32_t j = (int32_t)(i - b * count);
  const int32_t nc = cand_n[b];
  const float total = cand_total[b];
  if (nc == 0 || total == 0.f) { out[i] = default_node; return; }
  double u, u2;
  if (philox) philox_uniform2((unsigned long long)b, (uint32_t)j, (uint32_t)rng->calls, key ^ 0x4C57ull, u, u2);
  else { uint32_t x = modmul(rng->x_prev, modpow_a(2ull * (pos[b] + (unsigned long long)j))); u = minstd_uniform(x); }
  const float* cum = c_cum + ptr[b * n];
  const int32_t k = upper_bound_clamped(cum, 0, nc - 1, gt_threshold(pick_r(u, 0.f, total)));
  out[i] = (long long)c_id[ptr[b * n] + k];
}

// adj[b, j, k] = 1 iff nb[b, k] appears among the listed neighbors of nodes[b, j]; the listing slice of (b, j) is searched
// linearly (unsorted lists are legal)
__global__ void k_lw_adj(const long long* __restrict__ ptr, int64_t batch, int32_t n, int32_t m, const unsigned long long* __restrict__ ids,
                         const long long* __restrict__ nb, float* __restrict__ adj) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= batch * (int64_t)n * m) return;
  const int64_t bj = i / m;
  const int64_t b = bj / n;
  const int32_t k = (int32_t)(i - bj * m);
  const unsigned long long want = (unsigned long long)nb[b * m + k];
  float v = 0.f;
  for (long long e = ptr[bj]; e < ptr[bj + 1]; ++e)
    if (ids[e] == want) { v = 1.f; break; }
  adj[i] = v;
}

// ---- sparse batch adjacency (eu_sparse_get_adj_coo, section 3.5 of DESIGN.md) ----
// Row i = b * N + j of the listing, entry e.  sk / sv: each batch row's nb ids sorted, with their positions k.

// segment b of the sorted nb = [b * m, (b + 1) * m)
struct StrideSeg {
  long long m;
  __host__ __device__ long long operator()(long long b) const { return b * m; }
};

__global__ void k_adj_kiota(int32_t* __restrict__ v, int64_t n, int32_t m) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) v[p] = (int32_t)(p % m);
}

// the last i in [0, rows) with ptr[i] <= e (rows before it may be empty)
__device__ __forceinline__ int32_t adj_row_of(const long long* __restrict__ ptr, int32_t rows, long long e) {
  int32_t lo = 0, hi = rows - 1;
  while (lo < hi) {
    const int32_t mid = (int32_t)(((int64_t)lo + hi + 1) >> 1);
    if (ptr[mid] <= e) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// One thread per listed entry, so a hub row is spread over as many threads as it has entries: the entry's id is looked up
// in its batch row's sorted nb (the range [lo, lo + span) of equal ids), and every hit enters the first-occurrence table
// under key (row, lo) -- an id listed several times by one row (multi-edges, repeated types) keeps its first entry only.
__global__ void __launch_bounds__(256) k_adj_probe(const long long* __restrict__ ptr, int32_t rows, int32_t N, int32_t M,
                                                   const unsigned long long* __restrict__ ids, int64_t total,
                                                   const unsigned long long* __restrict__ sk, const long long* __restrict__ nb,
                                                   HashSlot* tab, unsigned long long mask, int32_t* __restrict__ row_of,
                                                   int32_t* __restrict__ lo_of, int32_t* __restrict__ span_of,
                                                   int32_t* __restrict__ has_last) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= total) return;
  const int32_t i = adj_row_of(ptr, rows, e);
  const int32_t b = i / N;
  const unsigned long long id = ids[e];
  const int32_t s0 = b * M, s1 = s0 + M;
  int32_t lo = s0, hi = s1;
  while (lo < hi) { const int32_t mid = (lo + hi) >> 1; if (sk[mid] < id) lo = mid + 1; else hi = mid; }
  int32_t up = lo;
  hi = s1;
  while (up < hi) { const int32_t mid = (up + hi) >> 1; if (sk[mid] <= id) up = mid + 1; else hi = mid; }
  row_of[e] = i;
  lo_of[e] = lo;
  span_of[e] = up - lo;
  if (up > lo) {
    uq_insert_warp(tab, mask, (unsigned long long)i * (unsigned long long)M + (unsigned long long)(lo - s0), (unsigned long long)e);
    // (b, N-1, M-1) is an entry: no filler for this batch row
    if (i - b * N == N - 1 &&id == (unsigned long long)nb[(int64_t)b * M + M - 1]) has_last[b] = 1;
  }
}

// cnt[e] = the entries e contributes (its span if it is the first entry of its row listing that id, else 0); cnt[total] = 0
__global__ void k_adj_keep(int64_t total, int32_t M, const int32_t* __restrict__ row_of, const int32_t* __restrict__ lo_of,
                           const int32_t* __restrict__ span_of, const HashSlot* tab, unsigned long long mask, int32_t N,
                           long long* __restrict__ cnt) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e > total) return;
  long long c = 0;
  if (e < total && span_of[e] > 0) {
    const int32_t i = row_of[e], s0 = i / N * M;
    if (uq_first(tab, mask, (unsigned long long)i * (unsigned long long)M + (unsigned long long)(lo_of[e] - s0)) == (unsigned long long)e)
      c = span_of[e];
  }
  cnt[e] = c;
}

// fl[b] = 1 iff batch row b gets the filler (b, N-1, M-1) = 0; fl[batch] = 0
__global__ void k_adj_fillers(const int32_t* __restrict__ has_last, int64_t batch, long long* __restrict__ fl) {
  const int64_t b = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (b <= batch) fl[b] = b < batch && !has_last[b] ? 1 : 0;
}

// rowptr[i] = the entries before row i: the kept hits of the listing before it plus the fillers of earlier batch rows
__global__ void k_adj_rowptr(int64_t rows, int32_t N, const long long* __restrict__ ptr, const long long* __restrict__ scan_e,
                             const long long* __restrict__ scan_f, long long* __restrict__ rowptr) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i <= rows) rowptr[i] = scan_e[ptr[i]] + scan_f[i / N];
}

// One thread per kept (row, k) pair, so a hit of many positions (an id repeated in nb) is spread too: hit slot h is found
// by binary search in the scanned counts, its k read from the sorted positions.  Rows are final here, k still in id order.
__global__ void __launch_bounds__(256) k_adj_expand(int64_t total, int32_t N, const long long* __restrict__ scan_e,
                                                    const long long* __restrict__ scan_f, const int32_t* __restrict__ row_of,
                                                    const int32_t* __restrict__ lo_of, const int32_t* __restrict__ sv,
                                                    long long* __restrict__ out_idx, long long* __restrict__ out_val,
                                                    int32_t* __restrict__ kbuf) {
  const long long hits = scan_e[total];
  for (long long h = blockIdx.x * (long long)blockDim.x + threadIdx.x; h < hits; h += (long long)gridDim.x * blockDim.x) {
    int64_t lo = 0, hi = total - 1;          // the last e with scan_e[e] <= h (its count is > 0)
    while (lo < hi) {
      const int64_t mid = (lo + hi + 1) >> 1;
      if (scan_e[mid] <= h) lo = mid; else hi = mid - 1;
    }
    const int32_t i = row_of[lo], b = i / N;
    const long long o = h + scan_f[b];
    out_idx[3 * o] = b;
    out_idx[3 * o + 1] = i - (long long)b * N;
    out_val[o] = 1;
    kbuf[o] = sv[lo_of[lo] + (int32_t)(h - scan_e[lo])];
  }
}

// the filler of batch row b closes row (b, N-1): M-1 is the largest k and absent from that row
__global__ void k_adj_filler(const int32_t* __restrict__ has_last, int64_t batch, int32_t N, int32_t M,
                             const long long* __restrict__ rowptr, long long* __restrict__ out_idx, long long* __restrict__ out_val,
                             int32_t* __restrict__ kbuf) {
  const int64_t b = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (b >= batch || has_last[b]) return;
  const long long o = rowptr[(b + 1) * N] - 1;
  out_idx[3 * o] = b;
  out_idx[3 * o + 1] = N - 1;
  out_val[o] = 0;
  kbuf[o] = M - 1;
}

__global__ void k_adj_col(int64_t nnz, const int32_t* __restrict__ k, long long* __restrict__ out_idx) {
  for (int64_t o = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; o < nnz; o += (int64_t)gridDim.x * blockDim.x) out_idx[3 * o + 2] = k[o];
}

}  // namespace eu

using namespace eu;

// Shared front end: the full listing of batch * n nodes into scratch (synchronises once to size it).
struct LwListing {
  long long* ptr = nullptr; unsigned long long* ids = nullptr; float* w = nullptr; int32_t* t = nullptr; long long total = 0;
  void free_all() { cudaFree(ptr); cudaFree(ids); cudaFree(w); cudaFree(t); }
};
static int lw_listing(eu_ctx* c, const int64_t* nodes, int64_t rows, const int32_t* etypes, int32_t K, LwListing* L) {
  cudaStream_t s = c->stream;
  EU_CUDA(cudaMalloc(&L->ptr, 8 * (size_t)(rows + 1)));
  int rc = eu_get_full_neighbor(c, nodes, rows, etypes, K, 0, (int64_t*)L->ptr, nullptr, nullptr, nullptr);
  if (rc) return rc;
  EU_CUDA(cudaMemcpyAsync(&L->total, L->ptr + rows, 8, cudaMemcpyDeviceToHost, s));
  EU_CUDA(cudaStreamSynchronize(s));
  if (L->total >= ((long long)1 << 31)) { set_error("layerwise: more than 2^31 listed neighbors"); return EU_ERR_UNSUPPORTED; }
  const size_t nn = (size_t)std::max<long long>(L->total, 1);
  EU_CUDA(cudaMalloc(&L->ids, 8 * nn));
  EU_CUDA(cudaMalloc(&L->w, 4 * nn));
  EU_CUDA(cudaMalloc(&L->t, 4 * nn));
  if (L->total > 0) rc = eu_get_full_neighbor(c, nodes, rows, etypes, K, L->total, (int64_t*)L->ptr, (int64_t*)L->ids, L->w, L->t);
  return rc;
}

extern "C" int eu_sample_neighbor_layerwise(eu_ctx* c, const int64_t* nodes, int64_t batch, int32_t n, const int32_t* etypes, int32_t K,
                                            int32_t count, int64_t default_node, int32_t weight_func, int64_t* out_nb, float* out_adj) {
  if (!c || batch < 0 || n < 1 || count < 0 || weight_func < 0 || weight_func > 1 || (batch > 0 && (!nodes || (count > 0 && !out_nb)))) {
    set_error("eu_sample_neighbor_layerwise: bad argument");
    return EU_ERR_INVALID;
  }
  EU_CUDA(cudaSetDevice(c->g->device));
  if (batch == 0 || count == 0) return EU_OK;
  if (batch >= ((int64_t)1 << 31)) { set_error("eu_sample_neighbor_layerwise: more than 2^31 batch rows"); return EU_ERR_UNSUPPORTED; }
  cudaStream_t s = c->stream;
  LwListing L;
  int rc = lw_listing(c, nodes, batch * n, etypes, K, &L);
  char* buf = nullptr;
  if (!rc) {
    const size_t nn = (size_t)std::max<long long>(L.total, 1);
    BatchSeg f{L.ptr, (long long)n};
    cub::CountingInputIterator<long long> cnt(0);
    cub::TransformInputIterator<long long, BatchSeg, cub::CountingInputIterator<long long>> seg(cnt, f);
    size_t tmp1 = 0, tmp2 = 0;
    cub::DeviceSegmentedSort::StableSortPairs((void*)nullptr, tmp1, (const int32_t*)nullptr, (int32_t*)nullptr, (const long long*)nullptr,
                                              (long long*)nullptr, (int)nn, (int)batch, seg, seg + 1, s);
    cub::DeviceSegmentedSort::StableSortPairs((void*)nullptr, tmp2, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                              (const long long*)nullptr, (long long*)nullptr, (int)nn, (int)batch, seg, seg + 1, s);
    const size_t tmp = (std::max(tmp1, tmp2) + 255) & ~(size_t)255;
    // idx_a 8 | idx_b 8 | key64_a 8 | key64_b 8 | key32_a 4 | key32_b 4 | c_id 8 | c_cum 4 | c_t 4 | per batch: cand_n 4, total 4, pos 8(+1)
    const size_t per = 8 + 8 + 8 + 8 + 4 + 4 + 8 + 4 + 4;
    const size_t bytes = per * nn + 16 * (size_t)(batch + 2) + 4096 + tmp;
    if (cudaMalloc(&buf, bytes) != cudaSuccess) { set_error("eu_sample_neighbor_layerwise: cudaMalloc(%zu) failed", bytes); rc = EU_ERR_CUDA; }
    if (!rc) {
      char* p = buf;
      auto take = [&](size_t b) { char* q = p; p += (b + 255) & ~(size_t)255; return q; };
      long long* idx_a = (long long*)take(8 * nn); long long* idx_b = (long long*)take(8 * nn);
      unsigned long long* k64_a = (unsigned long long*)take(8 * nn); unsigned long long* k64_b = (unsigned long long*)take(8 * nn);
      int32_t* k32_a = (int32_t*)take(4 * nn); int32_t* k32_b = (int32_t*)take(4 * nn);
      unsigned long long* c_id = (unsigned long long*)take(8 * nn); float* c_cum = (float*)take(4 * nn); int32_t* c_t = (int32_t*)take(4 * nn);
      int32_t* cand_n = (int32_t*)take(4 * (size_t)batch); float* cand_total = (float*)take(4 * (size_t)batch);
      unsigned long long* pos = (unsigned long long*)take(8 * (size_t)(batch + 1));
      void* cubtmp = take(tmp);
      const long long* order = idx_a;
      if (L.total > 0) {
        // stable sort by type, then stable sort by neighbor id: entries ordered by (dst, type), equal keys in listing order
        k_lw_iota<<<kSMs * 4, 256, 0, s>>>(idx_a, L.total);
        cudaMemcpyAsync(k32_a, L.t, 4 * nn, cudaMemcpyDeviceToDevice, s);
        cudaError_t e = cub::DeviceSegmentedSort::StableSortPairs(cubtmp, tmp1, (const int32_t*)k32_a, k32_b, (const long long*)idx_a, idx_b,
                                                                  (int)L.total, (int)batch, seg, seg + 1, s);
        k_lw_gather_id<<<kSMs * 4, 256, 0, s>>>(idx_b, L.ids, L.total, k64_a);
        if (e == cudaSuccess)
          e = cub::DeviceSegmentedSort::StableSortPairs(cubtmp, tmp2, (const unsigned long long*)k64_a, k64_b, (const long long*)idx_b, idx_a,
                                                        (int)L.total, (int)batch, seg, seg + 1, s);
        g_launches += 4;
        if (e != cudaSuccess) { set_error("eu_sample_neighbor_layerwise: %s", cudaGetErrorString(e)); rc = EU_ERR_CUDA; }
      }
      if (!rc) {
        k_lw_candidates<<<(unsigned)ceil_div(batch, 128), 128, 0, s>>>(L.ptr, batch, n, order, L.ids, L.w, L.t, weight_func, c_id, c_t, c_cum,
                                                                      cand_n, cand_total);
        k_lw_positions<<<1, 32, 0, s>>>(cand_n, cand_total, batch, count, pos, c->d_rng, c->rng == EU_RNG_MINSTD);
        k_lw_sample<<<(unsigned)ceil_div(batch * (int64_t)count, 256), 256, 0, s>>>(L.ptr, batch, n, count, (long long)default_node, c_id, c_cum,
                                                                                   cand_n, cand_total, pos, c->d_rng, c->rng == EU_RNG_PHILOX,
                                                                                   c->seed, (long long*)out_nb);
        g_launches += 3;
        if (out_adj) {
          k_lw_adj<<<(unsigned)ceil_div(batch * (int64_t)n * count, 256), 256, 0, s>>>(L.ptr, batch, n, count, L.ids, (const long long*)out_nb, out_adj);
          g_launches++;
        }
        if (cudaStreamSynchronize(s) != cudaSuccess) { set_error("eu_sample_neighbor_layerwise: %s", cudaGetErrorString(cudaGetLastError())); rc = EU_ERR_CUDA; }
      }
    }
  }
  cudaFree(buf);
  L.free_all();
  return rc;
}

// tf_euler.sparse_get_adj: dense 0/1 view [batch, N, M] of the reference's SparseTensor
extern "C" int eu_sparse_get_adj(eu_ctx* c, const int64_t* nodes, const int64_t* nb_nodes, int64_t batch, int32_t N, int32_t M,
                                 const int32_t* etypes, int32_t K, float* out_adj) {
  if (!c || batch < 0 || N < 1 || M < 1 || (batch > 0 && (!nodes || !nb_nodes || !out_adj))) { set_error("eu_sparse_get_adj: bad argument"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  if (batch == 0) return EU_OK;
  LwListing L;
  int rc = lw_listing(c, nodes, batch * N, etypes, K, &L);
  if (!rc) {
    k_lw_adj<<<(unsigned)ceil_div(batch * (int64_t)N * M, 256), 256, 0, c->stream>>>(L.ptr, batch, N, M, L.ids, (const long long*)nb_nodes, out_adj);
    g_launches++;
    if (cudaStreamSynchronize(c->stream) != cudaSuccess) { set_error("eu_sparse_get_adj: %s", cudaGetErrorString(cudaGetLastError())); rc = EU_ERR_CUDA; }
  }
  L.free_all();
  return rc;
}

// tf_euler.sparse_get_adj as the reference's SparseTensor (tf_euler/kernels/sparse_get_adj_op.cc:84-117); DESIGN.md section 3.5.
// Everything after the listing is O(listed entries + entries + M log M) per batch row: no pass over the N * M pairs.
static int adj_coo(eu_ctx* c, const int64_t* nb_nodes, int64_t batch, int32_t N, int32_t M, int64_t cap, const LwListing& L,
                   int64_t* out_ptr, int64_t* out_indices, int64_t* out_values) {
  cudaStream_t s = c->stream;
  const int64_t rows = batch * N, nbs = batch * M, E = L.total;
  const int64_t tcap = uq_table_cap(E);
  cub::CountingInputIterator<long long> cnt_it(0);
  cub::TransformInputIterator<long long, StrideSeg, cub::CountingInputIterator<long long>> seg(cnt_it, StrideSeg{(long long)M});
  size_t t_nb = 0, t_se = 0, t_sf = 0, t_sort = 0;
  cub::DeviceSegmentedSort::SortPairs((void*)nullptr, t_nb, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                      (const int32_t*)nullptr, (int32_t*)nullptr, (int)nbs, (int)batch, seg, seg + 1, s);
  cub::DeviceScan::ExclusiveSum((void*)nullptr, t_se, (const long long*)nullptr, (long long*)nullptr, (int)(E + 1), s);
  cub::DeviceScan::ExclusiveSum((void*)nullptr, t_sf, (const long long*)nullptr, (long long*)nullptr, (int)(batch + 1), s);
  if (cap > 0)
    cub::DeviceSegmentedSort::SortKeys((void*)nullptr, t_sort, (const int32_t*)nullptr, (int32_t*)nullptr, (int)cap, (int)rows,
                                       (const long long*)out_ptr, (const long long*)out_ptr + 1, s);
  const size_t tmp = std::max(std::max(t_nb, t_se), std::max(t_sf, t_sort));
  auto a256 = [](size_t b) { return (b + 255) & ~(size_t)255; };
  const size_t e1 = (size_t)std::max<int64_t>(E, 1);
  // table | sorted nb ids | positions in / sorted | per entry: row, lo, span, count, scan | per batch row: has_last, filler,
  // scan | [per entry of the output: k, sorted k] | cub temp
  const size_t o_tab = 0, o_sk = o_tab + a256(16 * (size_t)(tcap + 1)), o_kio = o_sk + a256(8 * (size_t)nbs),
               o_sv = o_kio + a256(4 * (size_t)nbs), o_row = o_sv + a256(4 * (size_t)nbs), o_lo = o_row + a256(4 * e1),
               o_span = o_lo + a256(4 * e1), o_cnt = o_span + a256(4 * e1), o_se = o_cnt + a256(8 * (size_t)(E + 1)),
               o_has = o_se + a256(8 * (size_t)(E + 1)), o_fl = o_has + a256(4 * (size_t)batch),
               o_sf = o_fl + a256(8 * (size_t)(batch + 1)), o_k = o_sf + a256(8 * (size_t)(batch + 1)),
               o_k2 = o_k + a256(4 * (size_t)cap), o_tmp = o_k2 + a256(4 * (size_t)cap), total = o_tmp + a256(tmp);
  int rc = ctx_misc(c, (int64_t)total);
  if (rc) return rc;
  char* m = (char*)c->d_misc;
  HashSlot* tab = (HashSlot*)(m + o_tab);
  unsigned long long* sk = (unsigned long long*)(m + o_sk);
  int32_t *kio = (int32_t*)(m + o_kio), *sv = (int32_t*)(m + o_sv), *row = (int32_t*)(m + o_row), *lo = (int32_t*)(m + o_lo),
          *span = (int32_t*)(m + o_span), *has_last = (int32_t*)(m + o_has), *kbuf = (int32_t*)(m + o_k), *kbuf2 = (int32_t*)(m + o_k2);
  long long *cnt = (long long*)(m + o_cnt), *scan_e = (long long*)(m + o_se), *fl = (long long*)(m + o_fl), *scan_f = (long long*)(m + o_sf);
  const unsigned long long mask = (unsigned long long)tcap - 1;
  const unsigned cap_blocks = kSMs * 8;

  k_uq_clear<<<(unsigned)std::min<int64_t>(ceil_div(tcap + 1, 256), cap_blocks), 256, 0, s>>>(tab, tcap + 1);
  EU_LAUNCHED();
  k_adj_kiota<<<(unsigned)std::min<int64_t>(ceil_div(nbs, 256), cap_blocks), 256, 0, s>>>(kio, nbs, M);
  EU_LAUNCHED();
  EU_CUDA(cub::DeviceSegmentedSort::SortPairs(m + o_tmp, t_nb, (const unsigned long long*)nb_nodes, sk, (const int32_t*)kio, sv,
                                              (int)nbs, (int)batch, seg, seg + 1, s));
  EU_LAUNCHED();
  EU_CUDA(cudaMemsetAsync(has_last, 0, 4 * (size_t)batch, s));
  if (E > 0) {
    k_adj_probe<<<(unsigned)ceil_div(E, 256), 256, 0, s>>>(L.ptr, (int32_t)rows, N, M, L.ids, E, sk, (const long long*)nb_nodes, tab,
                                                           mask, row, lo, span, has_last);
    EU_LAUNCHED();
  }
  k_adj_keep<<<(unsigned)ceil_div(E + 1, 256), 256, 0, s>>>(E, M, row, lo, span, tab, mask, N, cnt);
  EU_LAUNCHED();
  k_adj_fillers<<<(unsigned)ceil_div(batch + 1, 256), 256, 0, s>>>(has_last, batch, fl);
  EU_LAUNCHED();
  EU_CUDA(cub::DeviceScan::ExclusiveSum(m + o_tmp, t_se, (const long long*)cnt, scan_e, (int)(E + 1), s));
  EU_LAUNCHED();
  EU_CUDA(cub::DeviceScan::ExclusiveSum(m + o_tmp, t_sf, (const long long*)fl, scan_f, (int)(batch + 1), s));
  EU_LAUNCHED();
  k_adj_rowptr<<<(unsigned)ceil_div(rows + 1, 256), 256, 0, s>>>(rows, N, L.ptr, scan_e, scan_f, (long long*)out_ptr);
  EU_LAUNCHED();
  if (cap == 0) return EU_OK;

  long long nnz = 0;
  EU_CUDA(cudaMemcpyAsync(&nnz, out_ptr + rows, 8, cudaMemcpyDeviceToHost, s));
  EU_CUDA(cudaStreamSynchronize(s));
  if (nnz != cap) {
    set_error("eu_sparse_get_adj_coo: cap %lld is not the entry count %lld (call with cap = 0 first)", (long long)cap, nnz);
    return EU_ERR_INVALID;
  }
  long long* idx = (long long*)out_indices;
  k_adj_expand<<<(unsigned)std::min<int64_t>(ceil_div(cap, 256), cap_blocks), 256, 0, s>>>(E, N, scan_e, scan_f, row, lo, sv, idx,
                                                                                            (long long*)out_values, kbuf);
  EU_LAUNCHED();
  k_adj_filler<<<(unsigned)ceil_div(batch, 256), 256, 0, s>>>(has_last, batch, N, M, (const long long*)out_ptr, idx,
                                                              (long long*)out_values, kbuf);
  EU_LAUNCHED();
  EU_CUDA(cub::DeviceSegmentedSort::SortKeys(m + o_tmp, t_sort, (const int32_t*)kbuf, kbuf2, (int)cap, (int)rows,
                                             (const long long*)out_ptr, (const long long*)out_ptr + 1, s));
  EU_LAUNCHED();
  k_adj_col<<<(unsigned)std::min<int64_t>(ceil_div(cap, 256), cap_blocks), 256, 0, s>>>(cap, kbuf2, idx);
  EU_LAUNCHED();
  return EU_OK;
}

extern "C" int eu_sparse_get_adj_coo(eu_ctx* c, const int64_t* nodes, const int64_t* nb_nodes, int64_t batch, int32_t N, int32_t M,
                                     const int32_t* etypes, int32_t K, int64_t cap, int64_t* out_ptr, int64_t* out_indices,
                                     int64_t* out_values) {
  if (!c || batch < 0 || N < 0 || M < 0 || cap < 0 || !out_ptr || (batch > 0 && N > 0 && !nodes) || (batch > 0 && M > 0 && !nb_nodes) ||
      (cap > 0 && (!out_indices || !out_values))) {
    set_error("eu_sparse_get_adj_coo: bad argument");
    return EU_ERR_INVALID;
  }
  EU_CUDA(cudaSetDevice(c->g->device));
  const int64_t rows = batch * (int64_t)N;
  if (rows >= ((int64_t)1 << 31) || batch * (int64_t)M >= ((int64_t)1 << 31) || cap >= ((int64_t)1 << 31)) {
    set_error("eu_sparse_get_adj_coo: 2^31 or more node rows, neighbor slots or entries are not supported");
    return EU_ERR_UNSUPPORTED;
  }
  if (rows == 0 || M == 0) {            // no (b, j, k) position at all: no entry and no filler
    if (cap > 0) { set_error("eu_sparse_get_adj_coo: cap %lld is not the entry count 0", (long long)cap); return EU_ERR_INVALID; }
    EU_CUDA(cudaMemsetAsync(out_ptr, 0, 8 * (size_t)(rows + 1), c->stream));
    return EU_OK;
  }
  LwListing L;
  int rc = lw_listing(c, nodes, rows, etypes, K, &L);
  if (!rc) rc = adj_coo(c, nb_nodes, batch, N, M, cap, L, out_ptr, out_indices, out_values);
  if (!rc && cudaStreamSynchronize(c->stream) != cudaSuccess) {
    set_error("eu_sparse_get_adj_coo: %s", cudaGetErrorString(cudaGetLastError()));
    rc = EU_ERR_CUDA;
  }
  L.free_all();
  return rc;
}
