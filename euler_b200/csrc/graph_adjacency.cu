// The adjacency of the resident graph itself, with graph rows as columns: what layer-by-layer inference of the
// full-neighbourhood encoders (GCNEncoder.infer, GenieEncoder.infer) aggregates over, one pass per layer over the graph's
// edges instead of one L-hop neighbourhood per minibatch.
//
// Row i of the output lists engine row r0 + i (or rows[r0 + i]) as get_full_neighbor lists that row's node (neighbor.cu:
// the requested edge types in the order given, repeats repeat, multi-edges kept), each neighbour id replaced by its engine
// row (lookup_row: arithmetic for synthetic and sharded layouts, the htab probe otherwise).  A listed id that is not a node
// gets column n + k, k numbering such ids in first-occurrence order over the call's listing; the call returns them.
//
// Launches, no host synchronisation inside (the caller reads nnz and the absent-entry count between its two calls):
//   k_gadj_len -> cub scan          per-row lengths from grp_ptr, and offsets
//   k_gadj_entries<false>           (first call) the listed entries whose id is not a node, counted
//   k_gadj_entries<true>            (second call) every entry's column and weight, written once; entries are spread over the
//                                   threads by entry, not by row, so a hub row of ~10^5 entries does not serialise on one
//                                   lane group, and a warp writes 32 consecutive entries (coalesced).  Absent ids go to a
//                                   first-occurrence table (uq.cuh) and a list
//   [radix sort -> k_extra_first -> cub scan -> k_extra_emit]   only when some id is absent: the list in entry order, the
//                                   first occurrences numbered, every absent entry's column n + k
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "internal.h"
#include "segment.cuh"
#include "uq.cuh"

namespace eu {

static constexpr int kGadjThreads = 256;
static constexpr int kGadjPerThread = 4;
static constexpr int kGadjTile = kGadjThreads * kGadjPerThread;   // entries per CTA tile

__device__ __forceinline__ int64_t gadj_row(const DevGraph& g, const int64_t* __restrict__ rows, int64_t r0, int64_t i) {
  const int64_t r = rows ? rows[r0 + i] : r0 + i;
  return r >= 0 && r < g.n ? r : -1;
}

__global__ void k_gadj_len(DevGraph g, const int64_t* __restrict__ rows, int64_t r0, int64_t R, ETList et,
                           long long* __restrict__ out_ptr /* [R+1]; [0] = 0, [i+1] = len(i) */) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i == 0) out_ptr[0] = 0;
  if (i >= R) return;
  const int64_t r = gadj_row(g, rows, r0, i);
  long long len = 0;
  if (r >= 0) {
    const int64_t* gp = g.grp_ptr + r * g.T;
    for (int32_t k = 0; k < et.K; ++k) {
      const int32_t t = et.v[k];
      if (t >= 0 && t < g.T) len += gp[t + 1] - gp[t];
    }
  }
  out_ptr[i + 1] = len;
}

// Every listed entry e < ptr[R] (and < cap): FILL = false counts those whose id is not a node into *n_absent; FILL = true
// writes cols[e] (the row, or -1 for now) and w[e], and lists the absent ones as (entry, id) pairs and in the table.
template <bool FILL>
__global__ void __launch_bounds__(kGadjThreads) k_gadj_entries(DevGraph g, const int64_t* __restrict__ rows, int64_t r0, int64_t R,
                                                               ETList et, const long long* __restrict__ ptr, int64_t cap,
                                                               long long* __restrict__ cols, float* __restrict__ w,
                                                               unsigned long long* __restrict__ n_absent, HashSlot* tab,
                                                               unsigned long long mask, long long* __restrict__ lst_e,
                                                               unsigned long long* __restrict__ lst_id, int64_t lst_cap) {
  __shared__ int64_t s_lo, s_hi;
  const int64_t E = min((int64_t)ptr[R], cap);
  unsigned long long absent = 0;
  for (int64_t base = blockIdx.x * (int64_t)kGadjTile; base < E; base += (int64_t)gridDim.x * kGadjTile) {
    if (threadIdx.x == 0) {      // the tile's rows: every entry below searches only these
      s_lo = hop_row_of(ptr, 0, R - 1, base);
      s_hi = hop_row_of(ptr, s_lo, R - 1, min(base + kGadjTile, E) - 1);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kGadjPerThread; ++k) {
      const int64_t e = base + k * kGadjThreads + threadIdx.x;   // a warp holds 32 consecutive entries
      if (e >= E) continue;
      const int64_t i = hop_row_of(ptr, s_lo, s_hi, e);
      const int64_t r = gadj_row(g, rows, r0, i);   // >= 0: only rows of the graph have entries
      const int64_t* gp = g.grp_ptr + r * g.T;
      int64_t j = e - ptr[i], src = -1;
      for (int32_t q = 0; q < et.K; ++q) {      // the listing order: the requested types in turn, repeats repeat
        const int32_t tq = et.v[q];
        if (tq < 0 || tq >= g.T) continue;
        const int64_t len = gp[tq + 1] - gp[tq];
        if (j < len) { src = gp[tq] + j; break; }
        j -= len;
      }
      const unsigned long long id = g.nbr[src];
      const int64_t c = lookup_row(g, id);
      if (!FILL) {
        absent += c < 0;
        continue;
      }
      cols[e] = c;
      if (w) w[e] = __fsub_rn(g.cum_w[src], src == gp[0] ? 0.f : g.cum_w[src - 1]);
      if (c < 0) {
        const unsigned long long s = atomicAdd(n_absent, 1ull);
        if ((int64_t)s < lst_cap) { lst_e[s] = e; lst_id[s] = id; }
        uq_insert(tab, mask, id, (unsigned long long)e);
      }
    }
    __syncthreads();
  }
  if (!FILL && absent) atomicAdd(n_absent, absent);
}

// flag[i] = the absent entry se[i] is its id's first occurrence
__global__ void k_extra_first(const HashSlot* tab, unsigned long long mask, const long long* __restrict__ se,
                              const unsigned long long* __restrict__ sid, int64_t A, int32_t* __restrict__ flag) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < A) flag[i] = uq_first(tab, mask, sid[i]) == (unsigned long long)se[i] ? 1 : 0;
}

// cols[se[i]] = n + k of its id (k = pos of the id's first occurrence in the sorted list); first occurrences write the id
__global__ void k_extra_emit(const HashSlot* tab, unsigned long long mask, const long long* __restrict__ se,
                             const unsigned long long* __restrict__ sid, int64_t A, const int32_t* __restrict__ flag,
                             const int32_t* __restrict__ pos, int64_t n, long long* __restrict__ cols,
                             long long* __restrict__ extra, long long* __restrict__ n_extra) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= A) return;
  const long long f = (long long)uq_first(tab, mask, sid[i]);
  int64_t lo = 0, hi = A - 1;   // se is ascending and holds f
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (se[mid] < f) lo = mid + 1; else hi = mid;
  }
  cols[se[i]] = n + pos[lo];
  if (flag[i]) extra[pos[i]] = (long long)sid[i];
  if (i == A - 1) *n_extra = (long long)pos[i] + flag[i];
}

__global__ void k_node_rows(DevGraph g, const unsigned long long* __restrict__ nodes, int64_t B, long long* __restrict__ out) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < B) out[i] = lookup_row(g, nodes[i]);
}

}  // namespace eu

using namespace eu;

extern "C" {

int eu_graph_node_ids(eu_ctx* c, int64_t* out) {
  if (!c || (c->g->d.n > 0 && !out)) { set_error("eu_graph_node_ids: bad argument"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  if (c->g->d.n > 0) EU_CUDA(cudaMemcpyAsync(out, c->g->d.ids, 8 * (size_t)c->g->d.n, cudaMemcpyDeviceToDevice, c->stream));
  return EU_OK;
}

int eu_graph_node_rows(eu_ctx* c, const int64_t* nodes, int64_t B, int64_t* out) {
  if (!c || B < 0 || (B > 0 && (!nodes || !out))) { set_error("eu_graph_node_rows: bad argument"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  if (B == 0) return EU_OK;
  k_node_rows<<<(unsigned)ceil_div(B, 256), 256, 0, c->stream>>>(c->g->d, (const unsigned long long*)nodes, B, (long long*)out);
  EU_LAUNCHED();
  return EU_OK;
}

int eu_graph_adjacency(eu_ctx* c, const int32_t* etypes, int32_t K, const int64_t* rows, int64_t r0, int64_t r1, int64_t cap,
                       int64_t extra_cap, int64_t* out_ptr, int64_t* out_cols, float* out_w, int64_t* out_extra,
                       int64_t* counts) {
  if (!c || K < 0 || K > EU_MAX_ETYPES || (K > 0 && !etypes) || r0 < 0 || r1 < r0 || (!rows && r1 > c->g->d.n) ||
      cap < 0 || extra_cap < 0 || (extra_cap > 0 && cap == 0) || !out_ptr || !counts || (cap > 0 && !out_cols) ||
      (extra_cap > 0 && !out_extra)) {
    set_error("eu_graph_adjacency: bad argument");
    return EU_ERR_INVALID;
  }
  if (extra_cap >= ((int64_t)1 << 31) || r1 - r0 >= ((int64_t)1 << 31)) {
    set_error("eu_graph_adjacency: 2^31 or more rows or absent entries are not supported");
    return EU_ERR_UNSUPPORTED;
  }
  EU_CUDA(cudaSetDevice(c->g->device));
  const DevGraph& d = c->g->d;
  const int64_t R = r1 - r0;
  ETList et{};
  et.K = K;
  for (int32_t k = 0; k < K; ++k) et.v[k] = etypes[k];
  cudaStream_t s = c->stream;
  const bool fill = cap > 0;
  const int64_t A = extra_cap, tcap = uq_table_cap(A);
  size_t len_tmp = 0, sort_tmp = 0, flag_tmp = 0;
  cub::DeviceScan::InclusiveSum((void*)nullptr, len_tmp, (long long*)nullptr, (long long*)nullptr, (int)(R + 1), s);
  if (A > 0) {
    cub::DeviceRadixSort::SortPairs((void*)nullptr, sort_tmp, (const long long*)nullptr, (long long*)nullptr,
                                    (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)A, 0,
                                    radix_bits((unsigned long long)cap), s);
    cub::DeviceScan::ExclusiveSum((void*)nullptr, flag_tmp, (int32_t*)nullptr, (int32_t*)nullptr, (int)A, s);
  }
  // scratch: scan temp | absent count | [table | list (e, id) | sorted (e, id) | flag | pos | sort temp | flag scan temp]
  const size_t o_cnt = a256(len_tmp), o_tab = o_cnt + 256, o_le = o_tab + (A ? a256(16 * (size_t)(tcap + 1)) : 0),
               o_li = o_le + a256(8 * (size_t)A), o_se = o_li + a256(8 * (size_t)A), o_si = o_se + a256(8 * (size_t)A),
               o_flag = o_si + a256(8 * (size_t)A), o_pos = o_flag + a256(4 * (size_t)A), o_sort = o_pos + a256(4 * (size_t)A),
               o_fscan = o_sort + a256(sort_tmp), total = o_fscan + a256(flag_tmp);
  int rc = ctx_misc(c, (int64_t)total);
  if (rc) return rc;
  char* m = (char*)c->d_misc;
  unsigned long long* n_absent = (unsigned long long*)(m + o_cnt);
  HashSlot* tab = (HashSlot*)(m + o_tab);
  long long *le = (long long*)(m + o_le), *se = (long long*)(m + o_se);
  unsigned long long *li = (unsigned long long*)(m + o_li), *si = (unsigned long long*)(m + o_si);
  int32_t *flag = (int32_t*)(m + o_flag), *pos = (int32_t*)(m + o_pos);
  long long* ptr = (long long*)out_ptr;
  { EuProfScope ps(c, "k_gadj_len", R);
    k_gadj_len<<<(unsigned)ceil_div(std::max<int64_t>(R, 1), 256), 256, 0, s>>>(d, rows, r0, R, et, ptr); }
  EU_LAUNCHED();
  EU_CUDA(cub::DeviceScan::InclusiveSum(m, len_tmp, ptr, ptr, (int)(R + 1), s));
  EU_LAUNCHED();
  EU_CUDA(cudaMemsetAsync(n_absent, 0, 8, s));
  if (A > 0) {
    k_uq_clear<<<(unsigned)std::min<int64_t>(ceil_div(tcap + 1, 256), kSMs * 8), 256, 0, s>>>(tab, tcap + 1);
    EU_LAUNCHED();
  }
  if (R > 0) {
    EuProfScope ps(c, fill ? "k_gadj_fill" : "k_gadj_count", R);
    const unsigned blocks = fill ? (unsigned)std::max<int64_t>(1, std::min<int64_t>(ceil_div(cap, kGadjTile), kSMs * 8)) : kSMs * 8;
    if (fill)
      k_gadj_entries<true><<<blocks, kGadjThreads, 0, s>>>(d, rows, r0, R, et, ptr, cap, (long long*)out_cols, out_w, n_absent,
                                                            tab, (unsigned long long)tcap - 1, le, li, A);
    else
      k_gadj_entries<false><<<blocks, kGadjThreads, 0, s>>>(d, rows, r0, R, et, ptr, INT64_MAX, nullptr, nullptr, n_absent,
                                                             nullptr, 0, nullptr, nullptr, 0);
    EU_LAUNCHED();
  }
  if (!fill) {   // counts[0] = the absent entries
    EU_CUDA(cudaMemcpyAsync(counts, n_absent, 8, cudaMemcpyDeviceToDevice, s));
    return EU_OK;
  }
  if (A == 0) {
    EU_CUDA(cudaMemsetAsync(counts + 1, 0, 8, s));
    return EU_OK;
  }
  EuProfScope ps(c, "gadj_extras", A);
  EU_CUDA(cub::DeviceRadixSort::SortPairs(m + o_sort, sort_tmp, (const long long*)le, se, (const unsigned long long*)li, si, (int)A,
                                          0, radix_bits((unsigned long long)cap), s));
  EU_LAUNCHED();
  const unsigned nb = (unsigned)ceil_div(A, 256);
  k_extra_first<<<nb, 256, 0, s>>>(tab, (unsigned long long)tcap - 1, se, si, A, flag);
  EU_LAUNCHED();
  EU_CUDA(cub::DeviceScan::ExclusiveSum(m + o_fscan, flag_tmp, flag, pos, (int)A, s));
  EU_LAUNCHED();
  k_extra_emit<<<nb, 256, 0, s>>>(tab, (unsigned long long)tcap - 1, se, si, A, flag, pos, d.n, (long long*)out_cols,
                                  (long long*)out_extra, (long long*)counts + 1);
  EU_LAUNCHED();
  return EU_OK;
}

}  // extern "C"
