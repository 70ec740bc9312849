// The neighbour mean over a CSR adjacency, forward and backward: what the dense-combining sparse aggregators of GCNEncoder
// and GenieEncoder ('gcn', 'mean') compute from get_multi_hop_neighbor's (indptr, cols) of a hop.
//
// Reference semantics (file:line in the upstream alibaba/euler tree):
//   GCNAggregator / MeanAggregator   tf_euler/python/utils/sparse_aggregators.py:37-84  adj = _sparse_ones_like(adj);
//                                    degree = sparse_reduce_sum(adj, 1); sparse_tensor_dense_matmul(adj, neigh) /
//                                    maximum(degree, 1e-7)
//
// Forward, for row i with entries [indptr[i], indptr[i+1]) and deg_i of them:
//   S_i   = the neighbour rows x[cols[k]] summed in chunks of kSegChunk entries counted from the row's first one, each chunk
//           left to right from +0, the chunk sums of a row of several chunks added in chunk order from +0 (k_seg_combine)
//   out_i = __fdiv_rn(S_i, max(fl(deg_i), 1e-7f))   (a row without entries gives a zero row)
// A group of G lanes per chunk, 4 columns per lane and step, kAdjUnroll rows loaded ahead of the ordered adds; float4 loads
// when D % 4 == 0 and x / out are 16-byte aligned, scalar otherwise: the same adds, so the bits do not depend on the path.
// A chunk of a one-chunk row writes the output row, divided; the chunks of a longer row write chunk sums, which
// k_seg_combine adds into the output row and k_adj_divide divides.  A hub row is spread over as many groups as it has
// chunks.  The rows are the CSR's own, so nothing is sorted and nothing is read back: no host synchronisation, and the
// scratch (the rows' chunk offsets and (n + nnz / 256) * D floats of chunk sums) only grows with the sizes.
//
// Backward, grad_x[j] = sum over column j's entries k in row order of gs[row_k], gs_i = __fdiv_rn(grad_out_i, max(fl(deg_i),
// 1e-7f)): the transposed sum is an id-table gradient, so it goes through the path of segment.cuh that the embedding,
// skip-gram and KG backward passes share (plan_rows on cols as keys, sum_distinct_rows with the gathered entry kind reading
// row row_k of gs), whose order fixes the bits: each column's entries in stable row order, chunks of kSegChunk from +0, the
// chunk sums in chunk order.  No atomics and no host synchronisation either.
#include "segment.cuh"

namespace eu {

constexpr int kAdjUnroll = 8;   // neighbour rows in flight per lane ahead of the ordered adds

__device__ __forceinline__ float adj_den(int64_t deg) { return fmaxf((float)deg, 1e-7f); }

// start[i] = indptr[i] as int32 (every offset is below 2^31), for i in [0, n]
__global__ void k_adj_starts(const int64_t* __restrict__ indptr, int64_t n, int32_t* __restrict__ start) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i <= n; i += (int64_t)gridDim.x * blockDim.x)
    start[i] = (int32_t)__ldg(indptr + i);
}

// G lanes per chunk of kSegChunk entries: the chunk's neighbour rows summed left to right from +0
template <bool VEC>
__global__ void __launch_bounds__(256) k_adj_chunks(const float* __restrict__ x, const int64_t* __restrict__ cols,
                                                    const int32_t* __restrict__ start, const int32_t* __restrict__ chunk_off,
                                                    int64_t n, int dim, int G, float* __restrict__ partial, float* __restrict__ out) {
  const int lg = 31 - __clz(G);
  const int sub = (int)(threadIdx.x & (G - 1));
  const int64_t nch_all = __ldg(chunk_off + n);
  const int64_t step = ((int64_t)gridDim.x * blockDim.x) >> lg;
  constexpr int U = VEC ? kAdjUnroll : kAdjUnroll / 2;
  for (int64_t c = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> lg; c < nch_all; c += step) {
    const int64_t i = key_upper_bound(chunk_off, n + 1, c) - 1;   // the row of chunk c (rows without chunks are skipped)
    const int64_t c0 = __ldg(chunk_off + i), nch = __ldg(chunk_off + i + 1) - c0;
    const int64_t r0 = __ldg(start + i), r1 = __ldg(start + i + 1);
    const int64_t b = r0 + (c - c0) * kSegChunk, e = min(b + kSegChunk, r1);
    float* o = nch == 1 ? out + i * dim : partial + c * dim;
    const float den = adj_den(r1 - r0);
    for (int d = sub * 4; d < dim; d += G * 4) {
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int64_t k0 = b; k0 < e; k0 += U) {
        float4 v[U];
#pragma unroll
        for (int q = 0; q < U; ++q)
          if (k0 + q < e) v[q] = row_load4<VEC>(x + __ldg(cols + k0 + q) * dim, d, dim);
#pragma unroll
        for (int q = 0; q < U; ++q) {
          if (k0 + q < e) {
            acc.x = __fadd_rn(acc.x, v[q].x); acc.y = __fadd_rn(acc.y, v[q].y);
            acc.z = __fadd_rn(acc.z, v[q].z); acc.w = __fadd_rn(acc.w, v[q].w);
          }
        }
      }
      if (nch == 1) {
        acc.x = __fdiv_rn(acc.x, den); acc.y = __fdiv_rn(acc.y, den);
        acc.z = __fdiv_rn(acc.z, den); acc.w = __fdiv_rn(acc.w, den);
      }
      if (VEC) {
        *reinterpret_cast<float4*>(o + d) = acc;
      } else {
        o[d] = acc.x;
        if (d + 1 < dim) o[d + 1] = acc.y;
        if (d + 2 < dim) o[d + 2] = acc.z;
        if (d + 3 < dim) o[d + 3] = acc.w;
      }
    }
  }
}

// out[i, f] /= max(fl(deg_i), 1e-7) for the rows of several chunks (k_seg_combine wrote their sums)
__global__ void k_adj_divide(const int32_t* __restrict__ start, const int32_t* __restrict__ chunk_off, int64_t n, int dim,
                             float* __restrict__ out) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n * dim; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / dim;
    if (__ldg(chunk_off + i + 1) - __ldg(chunk_off + i) > 1) out[t] = __fdiv_rn(out[t], adj_den(__ldg(start + i + 1) - __ldg(start + i)));
  }
}

// gs[i, :] = grad_out[i, :] / max(fl(deg_i), 1e-7)
__global__ void k_adj_scale_grad(const float* __restrict__ g, const int64_t* __restrict__ indptr, int64_t n, int dim,
                                 float* __restrict__ gs) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n * dim; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / dim;
    gs[t] = __fdiv_rn(__ldg(g + t), adj_den(__ldg(indptr + i + 1) - __ldg(indptr + i)));
  }
}

// per entry k: key[k] = cols[k] (the gradient row), row[k] = the adjacency row holding k (the row of gs it reads)
__global__ void k_adj_entries(const int64_t* __restrict__ indptr, const int64_t* __restrict__ cols, int64_t n, int64_t nnz,
                              int32_t* __restrict__ key, int32_t* __restrict__ row) {
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < nnz; k += (int64_t)gridDim.x * blockDim.x) {
    int64_t lo = 0, hi = n;   // the last i with indptr[i] <= k
    while (lo < hi) {
      const int64_t mid = (lo + hi + 1) >> 1;
      if (__ldg(indptr + mid) <= k) lo = mid; else hi = mid - 1;
    }
    key[k] = (int32_t)__ldg(cols + k);
    row[k] = (int32_t)lo;
  }
}

// ok: the caller's pointers that the sizes need are there
static int adj_check(eu_ctx* c, bool ok, int64_t n, int64_t nnz, int64_t m, int32_t dim, const char* who) {
  if (!c || !ok || n < 0 || nnz < 0 || m < 0 || dim < 1 || (nnz > 0 && (n == 0 || m == 0))) {
    set_error("%s: bad argument", who);
    return EU_ERR_INVALID;
  }
  if (n >= ((int64_t)1 << 31) || nnz >= ((int64_t)1 << 31) || m >= ((int64_t)1 << 31) || !entries_fit(nnz)) {
    set_error("%s: 2^31 or more rows or entries are not supported", who);
    return EU_ERR_UNSUPPORTED;
  }
  return EU_OK;
}

}  // namespace eu

using namespace eu;

extern "C" {

int eu_adjacency_mean(eu_ctx* c, const float* x_neigh, int64_t m, const int64_t* indptr, const int64_t* cols, int64_t n,
                      int64_t nnz, int32_t dim, float* out) {
  const bool ok = (nnz == 0 || (x_neigh && cols)) && (n == 0 || (indptr && out));
  int rc = adj_check(c, ok, n, nnz, m, dim, "eu_adjacency_mean");
  if (rc) return rc;
  EU_CUDA(cudaSetDevice(c->g->device));
  if (n == 0) return EU_OK;
  cudaStream_t s = c->stream;
  // start | nc | chunk_off [n + 1] each | scan temp | chunk sums [n + nnz / kSegChunk, dim]
  const size_t n1 = a256(4 * (size_t)(n + 1)), scan = seg_scan_bytes(n);
  const int64_t slots = n + nnz / kSegChunk;
  const size_t o_part = 3 * n1 + a256(scan);
  if ((rc = ctx_misc(c, (int64_t)(o_part + 4 * (size_t)slots * dim)))) return rc;
  char* buf = (char*)c->d_misc;
  int32_t* start = (int32_t*)buf;
  int32_t* nc = (int32_t*)(buf + n1);
  int32_t* chunk_off = (int32_t*)(buf + 2 * n1);
  float* partial = (float*)(buf + o_part);
  k_adj_starts<<<stride_grid(n + 1), 256, 0, s>>>(indptr, n, start);
  EU_LAUNCHED();
  if ((rc = seg_chunk_offsets(c, start, n, kSegChunk, nc, buf + 3 * n1, scan, chunk_off))) return rc;
  const bool vec = dim % 4 == 0 && aligned16(x_neigh) && aligned16(out);
  const int G = group_lanes(ceil_div(dim, 4));
  {
    EuProfScope ps(c, "adj_mean_chunks", nnz);
    const unsigned blocks = stride_grid(slots * G);   // >= one group per chunk, up to the grid cap
    if (vec) k_adj_chunks<true><<<blocks, 256, 0, s>>>(x_neigh, cols, start, chunk_off, n, dim, G, partial, out);
    else k_adj_chunks<false><<<blocks, 256, 0, s>>>(x_neigh, cols, start, chunk_off, n, dim, G, partial, out);
    EU_LAUNCHED();
  }
  EuProfScope ps(c, "adj_mean_combine", n);
  k_seg_combine<<<(unsigned)ceil_div(n * dim, 256), 256, 0, s>>>(chunk_off, partial, n, dim, out);
  EU_LAUNCHED();
  k_adj_divide<<<stride_grid(n * dim), 256, 0, s>>>(start, chunk_off, n, dim, out);
  EU_LAUNCHED();
  return EU_OK;
}

int eu_adjacency_mean_backward(eu_ctx* c, const float* grad_out, const int64_t* indptr, const int64_t* cols, int64_t n,
                               int64_t nnz, int64_t m, int32_t dim, float* grad_x) {
  const char* who = "eu_adjacency_mean_backward";
  const bool ok = (nnz == 0 || cols) && (n == 0 || (indptr && grad_out)) && (m == 0 || grad_x);
  int rc = adj_check(c, ok, n, nnz, m, dim, who);
  if (rc) return rc;
  EU_CUDA(cudaSetDevice(c->g->device));
  cudaStream_t s = c->stream;
  if (m > 0) EU_CUDA(cudaMemsetAsync(grad_x, 0, 4 * (size_t)m * dim, s));
  if (nnz == 0) return EU_OK;
  // gs [n, dim] | key [nnz] | row [nnz] | the entries' order and distinct-column plan
  const size_t o_key = a256(4 * (size_t)n * dim), o_row = o_key + a256(4 * (size_t)nnz), o_plan = o_row + a256(4 * (size_t)nnz);
  if ((rc = ctx_misc(c, (int64_t)(o_plan + row_plan_bytes(nnz, m, dim))))) return rc;
  char* buf = (char*)c->d_misc;
  float* gs = (float*)buf;
  RowList L;
  L.E = nnz;
  L.n_rows = m;
  L.key = (int32_t*)(buf + o_key);
  int32_t* row = (int32_t*)(buf + o_row);
  {
    EuProfScope ps(c, "adj_mean_bwd_entries", nnz);
    k_adj_scale_grad<<<stride_grid(n * dim), 256, 0, s>>>(grad_out, indptr, n, dim, gs);
    EU_LAUNCHED();
    k_adj_entries<<<stride_grid(nnz), 256, 0, s>>>(indptr, cols, n, nnz, L.key, row);
    EU_LAUNCHED();
  }
  {
    EuProfScope ps(c, "adj_mean_bwd_order", nnz);
    if ((rc = plan_rows(c, buf + o_plan, &L))) return rc;
  }
  EuProfScope ps(c, "adj_mean_bwd_sums", nnz);
  RowEntries R;   // the gathered kind: entry k's row is row row[k] of gs
  R.n_src = nnz;
  R.gt = gs;
  R.node = row;
  R.ld = dim;
  return sum_distinct_rows(c, R, L, dim, true, grad_x, nullptr);
}

}  // extern "C"
