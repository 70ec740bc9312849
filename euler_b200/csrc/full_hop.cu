// One full-neighbor hop of the full-neighborhood minibatch constructions, fused on the device:
//   GCNDataFlow       tf_euler/python/dataflow/gcn_dataflow.py:34-48 + UniqueDataFlow.produce_subgraph
//                     (neighbor_dataflow.py:84-110): unique(concat(listing, frontier)), edges [rows (+ self loops), inverse]
//   RelationDataFlow  relation_dataflow.py:31-71: the same unique, no self loops, the listed edge types alongside
//   get_multi_hop_neighbor  tf_euler/python/euler_ops/neighbor_ops.py:209-242: unique(listing) only, adjacency entries
//                     (row, col) -> weight in sparse_reorder order (by row, then col; equal pairs in listing order)
// where the listing is get_full_neighbor's (neighbor.cu) and unique is tf.unique (first-occurrence order, unique.cu).
//
// Launches (no host sync; the caller reads the listing total and the unique count, the two shapes TF needs as well):
//   k_full_len -> cub scan                       per-node lengths and offsets (eu_get_full_neighbor with cap = 0)
//   k_uq_clear -> k_hop_fill                     every listed entry written once (id, row, weight, type) and entered into
//                                                the first-occurrence table under its index in the VIRTUAL concatenation
//                                                [listing, frontier]: entry e -> e, frontier node i -> E + i.  The
//                                                concatenation itself is never written.  Balanced by entries, not nodes:
//                                                a hub row is spread over as many threads as it has entries.
//   k_hop_first -> cub scan -> k_hop_emit        first-occurrence flags, their scan, then the new frontier, each entry's
//                                                column and the frontier's positions straight into their final layout
//   [cub segmented stable sort]                  EU_HOP_SORT: each row's entries by column
#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_sort.cuh>

#include "internal.h"
#include "uq.cuh"

namespace eu {

static constexpr int kHopThreads = 256;
static constexpr int kHopPerThread = 4;
static constexpr int kHopTile = kHopThreads * kHopPerThread;   // entries per CTA tile

// V = E (+ n when the frontier is appended) virtual items; items [0, E) are the listing, [E, V) the frontier
__global__ void __launch_bounds__(kHopThreads) k_hop_fill(DevGraph g, const unsigned long long* __restrict__ nodes, int64_t n,
                                                          ETList et, const long long* __restrict__ ptr, int64_t E, int64_t V,
                                                          HashSlot* tab, unsigned long long mask, unsigned long long* __restrict__ vals,
                                                          long long* __restrict__ out_rows, float* __restrict__ out_w,
                                                          int32_t* __restrict__ out_t) {
  __shared__ int64_t s_lo, s_hi;
  for (int64_t base = blockIdx.x * (int64_t)kHopTile; base < V; base += (int64_t)gridDim.x * kHopTile) {
    if (threadIdx.x == 0 && base < E) {      // the tile's rows: every entry below searches only these
      s_lo = hop_row_of(ptr, 0, n - 1, base);
      s_hi = hop_row_of(ptr, s_lo, n - 1, min(base + kHopTile, E) - 1);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kHopPerThread; ++k) {
      const int64_t e = base + k * kHopThreads + threadIdx.x;   // a warp holds 32 consecutive items
      if (e >= V) continue;
      unsigned long long id;
      if (e < E) {
        const int64_t i = hop_row_of(ptr, s_lo, s_hi, e);
        const int64_t row = lookup_row(g, nodes[i]);
        int64_t j = e - ptr[i], src = -1;
        int32_t t = -1;
        if (row >= 0) {
          const int64_t* gp = g.grp_ptr + row * g.T;
          for (int32_t q = 0; q < et.K; ++q) {      // the listing order: the requested types in turn, repeats repeat
            const int32_t tq = et.v[q];
            if (tq < 0 || tq >= g.T) continue;
            const int64_t len = gp[tq + 1] - gp[tq];
            if (j < len) { src = gp[tq] + j; t = tq; break; }
            j -= len;
          }
          id = src >= 0 ? g.nbr[src] : 0ull;       // src < 0 only when cap disagrees with the listing (outside the contract)
          if (out_w) out_w[e] = src < 0 ? 0.f : __fsub_rn(g.cum_w[src], src == gp[0] ? 0.f : g.cum_w[src - 1]);
        } else {
          id = 0ull;
          if (out_w) out_w[e] = 0.f;
        }
        vals[e] = id;
        if (out_rows) out_rows[e] = i;
        if (out_t) out_t[e] = t;
      } else {
        id = nodes[e - E];
      }
      uq_insert_warp(tab, mask, id, (unsigned long long)e);
    }
    __syncthreads();
  }
}

__global__ void k_hop_first(const HashSlot* tab, unsigned long long mask, const unsigned long long* __restrict__ vals,
                            const unsigned long long* __restrict__ nodes, int64_t E, int64_t V, int32_t* __restrict__ first,
                            int32_t* __restrict__ flag) {
  const int64_t v = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (v >= V) return;
  const int32_t f = (int32_t)uq_first(tab, mask, v < E ? vals[v] : nodes[v - E]);
  first[v] = f;
  flag[v] = f == (int32_t)v ? 1 : 0;
}

// cols: [E] entry columns (+ [n] self-loop columns after them when self_loops); rows gets the self loops' rows
__global__ void k_hop_emit(const unsigned long long* __restrict__ vals, const unsigned long long* __restrict__ nodes, int64_t E,
                           int64_t V, const int32_t* __restrict__ first, const int32_t* __restrict__ flag,
                           const int32_t* __restrict__ pos, unsigned long long* __restrict__ uniq, long long* __restrict__ cols,
                           long long* __restrict__ res, bool self_loops, long long* __restrict__ rows, long long* __restrict__ n_unique) {
  const int64_t v = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (v >= V) return;
  if (flag[v]) uniq[pos[v]] = v < E ? vals[v] : nodes[v - E];
  const long long inv = pos[first[v]];
  if (v < E) {
    cols[v] = inv;
  } else {
    const int64_t k = v - E;
    if (res) res[k] = inv;
    if (self_loops) {
      cols[v] = inv;
      if (rows) rows[v] = k;
    }
  }
  if (v == V - 1) *n_unique = (long long)pos[v] + flag[v];
}

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

}  // namespace eu

using namespace eu;

extern "C" int eu_full_neighbor_hop(eu_ctx* c, const int64_t* nodes, int64_t n, const int32_t* etypes, int32_t K, int32_t flags,
                                    int64_t cap, int64_t* out_ptr, int64_t* out_uniq, int64_t* n_unique, int64_t* out_rows,
                                    int64_t* out_cols, float* out_w, int32_t* out_t, int64_t* out_res) {
  const bool append = flags & EU_HOP_APPEND_FRONTIER, self_loops = flags & EU_HOP_SELF_LOOPS, sort = flags & EU_HOP_SORT;
  const bool lengths_only = cap == 0 && !out_uniq;
  const int64_t E = cap, V = E + (append ? n : 0), W = E + (self_loops ? n : 0);
  if (!c || n < 0 || cap < 0 || (flags & ~(EU_HOP_APPEND_FRONTIER | EU_HOP_SELF_LOOPS | EU_HOP_SORT)) ||
      (self_loops && (!append || sort)) || (sort && out_t) || (!append && out_res) || !out_ptr ||
      (!lengths_only && V > 0 && (!out_uniq || !n_unique)) || (!lengths_only && W > 0 && !out_cols)) {
    set_error("eu_full_neighbor_hop: bad argument");
    return EU_ERR_INVALID;
  }
  // lengths and offsets (validates nodes / etypes / K and selects the device)
  int rc = eu_get_full_neighbor(c, nodes, n, etypes, K, 0, out_ptr, nullptr, nullptr, nullptr);
  if (rc || lengths_only) return rc;
  if (V >= ((int64_t)1 << 31) || n >= ((int64_t)1 << 31)) {
    set_error("eu_full_neighbor_hop: the hop lists %lld entries%s; 2^31 or more are not supported (tf.unique's int32 index)",
              (long long)E, append ? " plus the frontier" : "");
    return EU_ERR_UNSUPPORTED;
  }
  cudaStream_t s = c->stream;
  if (V == 0) {
    if (n_unique) EU_CUDA(cudaMemsetAsync(n_unique, 0, sizeof(int64_t), s));
    return EU_OK;
  }
  ETList et{};
  et.K = K;
  for (int32_t k = 0; k < K; ++k) et.v[k] = etypes[k];
  const int64_t tcap = uq_table_cap(V);
  size_t scan_tmp = 0, sort_tmp = 0;
  cub::DeviceScan::ExclusiveSum((void*)nullptr, scan_tmp, (int32_t*)nullptr, (int32_t*)nullptr, (int)V, s);
  if (sort && E > 0) {
    if (out_w)
      cub::DeviceSegmentedSort::StableSortPairs((void*)nullptr, sort_tmp, (const long long*)nullptr, (long long*)nullptr,
                                                (const float*)nullptr, (float*)nullptr, (int)E, (int)n, (const long long*)out_ptr,
                                                (const long long*)out_ptr + 1, s);
    else
      cub::DeviceSegmentedSort::StableSortKeys((void*)nullptr, sort_tmp, (const long long*)nullptr, (long long*)nullptr, (int)E,
                                               (int)n, (const long long*)out_ptr, (const long long*)out_ptr + 1, s);
  }
  // scratch: table | listed ids | first | flag | pos | scan temp [| sort keys | sort weights | sort temp]
  const size_t o_tab = 0, o_vals = o_tab + align256(16 * (size_t)(tcap + 1)), o_first = o_vals + align256(8 * (size_t)E),
               o_flag = o_first + align256(4 * (size_t)V), o_pos = o_flag + align256(4 * (size_t)V),
               o_scan = o_pos + align256(4 * (size_t)V), o_keys = o_scan + align256(scan_tmp),
               o_sw = o_keys + (sort ? align256(8 * (size_t)E) : 0), o_sort = o_sw + (sort ? align256(4 * (size_t)E) : 0),
               total = o_sort + (sort ? align256(sort_tmp) : 0);
  if ((rc = ctx_misc(c, (int64_t)total))) return rc;
  char* m = (char*)c->d_misc;
  HashSlot* tab = (HashSlot*)(m + o_tab);
  unsigned long long* vals = (unsigned long long*)(m + o_vals);
  int32_t *first = (int32_t*)(m + o_first), *flag = (int32_t*)(m + o_flag), *pos = (int32_t*)(m + o_pos);
  long long* cols = sort ? (long long*)(m + o_keys) : (long long*)out_cols;       // sorted: listing-order columns are sort keys
  float* w = sort && out_w ? (float*)(m + o_sw) : out_w;
  const unsigned long long mask = (unsigned long long)tcap - 1;
  const auto* d_nodes = (const unsigned long long*)nodes;
  { EuProfScope ps(c, "k_hop_fill", V);
    k_uq_clear<<<(unsigned)std::min<int64_t>(ceil_div(tcap + 1, 256), kSMs * 8), 256, 0, s>>>(tab, tcap + 1);
    EU_LAUNCHED();
    const unsigned blocks = (unsigned)std::min<int64_t>(ceil_div(V, kHopTile), kSMs * 8);
    k_hop_fill<<<blocks, kHopThreads, 0, s>>>(c->g->d, d_nodes, n, et, (const long long*)out_ptr, E, V, tab, mask, vals,
                                              (long long*)out_rows, w, out_t); }
  EU_LAUNCHED();
  const unsigned nb = (unsigned)ceil_div(V, 256);
  { EuProfScope ps(c, "k_hop_first", V);
    k_hop_first<<<nb, 256, 0, s>>>(tab, mask, vals, d_nodes, E, V, first, flag); }
  EU_LAUNCHED();
  EU_CUDA(cub::DeviceScan::ExclusiveSum(m + o_scan, scan_tmp, flag, pos, (int)V, s));
  EU_LAUNCHED();
  { EuProfScope ps(c, "k_hop_emit", V);
    k_hop_emit<<<nb, 256, 0, s>>>(vals, d_nodes, E, V, first, flag, pos, (unsigned long long*)out_uniq, cols, (long long*)out_res,
                                  self_loops, (long long*)out_rows, (long long*)n_unique); }
  EU_LAUNCHED();
  if (sort && E > 0) {
    EuProfScope ps(c, "hop_segmented_sort", E);
    if (out_w)
      EU_CUDA(cub::DeviceSegmentedSort::StableSortPairs(m + o_sort, sort_tmp, (const long long*)cols, (long long*)out_cols,
                                                        (const float*)w, out_w, (int)E, (int)n, (const long long*)out_ptr,
                                                        (const long long*)out_ptr + 1, s));
    else
      EU_CUDA(cub::DeviceSegmentedSort::StableSortKeys(m + o_sort, sort_tmp, (const long long*)cols, (long long*)out_cols, (int)E,
                                                       (int)n, (const long long*)out_ptr, (const long long*)out_ptr + 1, s));
    EU_LAUNCHED();
  }
  return EU_OK;
}
