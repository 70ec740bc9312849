// Edge orders and fixed-order segment sums shared by the fused aggregations (gat.cu, relation.cu, dna.cu), the mp scatter and
// the id-table gradients (embedding.cu, skipgram.cu, kg.cu).
//
// An edge order walks the edges sorted by an int32 index (the target, the source, a relation), stably: edges with equal
// index keep their order, so a sum over a segment in order gives the bits of the same sum over the stably sorted list.  A
// fixed-order segment sum cuts each segment into chunks of kSegChunk positions counted from its first one; each chunk is
// summed left to right and a segment of several chunks adds its chunk sums in chunk order.  The bits then depend on the
// segment's own sequence only, never on the launch configuration or on other segments, and a hub is spread over many CTAs.
#pragma once
#include <algorithm>

#include "internal.h"

namespace eu {

constexpr int kSegChunk = 256;   // positions per chunk of a fixed-order segment sum: it fixes the bits of those sums

// ---------------------------------------------------------------------------- device helpers
// the first position k in [0, n) with a[k] >= key (a non-decreasing), or n
__device__ __forceinline__ int64_t key_lower_bound(const int32_t* __restrict__ a, int64_t n, int64_t key) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if ((int64_t)__ldg(a + mid) < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// the first position k in [0, n) with a[k] > key (a non-decreasing), or n
__device__ __forceinline__ int64_t key_upper_bound(const int32_t* __restrict__ a, int64_t n, int64_t key) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if ((int64_t)__ldg(a + mid) <= key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// the edge at position k of an order (perm: position -> edge, null = the identity)
__device__ __forceinline__ int64_t edge_at(const int32_t* __restrict__ perm, int64_t k) { return perm ? (int64_t)__ldg(perm + k) : k; }

// the mask of the G-lane group this lane belongs to (G a power of two)
__device__ __forceinline__ unsigned group_mask(int G) {
  if (G == 32) return 0xffffffffu;
  const int lane = threadIdx.x & 31;
  return ((1u << G) - 1u) << (lane & ~(G - 1));
}

// ---------------------------------------------------------------------------- host helpers
inline bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

// lanes of a group over n items per row (n = columns, or float4s of columns): a power of two >= n, at most 32
inline int group_lanes(int64_t n) {
  int g = 1;
  while (g < 32 && g < n) g <<= 1;
  return g;
}

// the radix-sort bits of the keys [0, n)
inline int radix_bits(unsigned long long n) {
  int b = 1;
  while (b < 64 && (1ull << b) < n) ++b;
  return b;
}

// the grid of a grid-stride loop over n items, 256 threads per CTA
inline unsigned stride_grid(int64_t n) { return (unsigned)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, 256), kSMs * 8)); }

// ---------------------------------------------------------------------------- edge orders
__global__ void k_check_sorted(const int32_t* __restrict__ idx, int64_t E, int* unsorted);   // *unsorted = 1 if idx decreases

struct EdgeOrder {                 // the order of the edges by `idx` (int32[E] in [0, n)), stable
  const int32_t* key = nullptr;    // idx itself when it is already non-decreasing
  const int32_t* perm = nullptr;   // null then
};

size_t order_bytes(int64_t E, int64_t n);   // the scratch order_by needs
// the stable order of the edges by idx (a radix sort), in `buf` (order_bytes(E, n) bytes)
int order_by(eu_ctx* c, const int32_t* idx, int64_t E, int64_t n, char* buf, EdgeOrder* o);

// The prologue of an entry point that walks the edges by target: the order by dst, and the ctx scratch laid out as
//   flag (256 B) | head (head_bytes) | [the dst order when dst is unsorted] | tail (tail_bytes)
// The scratch is sized once the sortedness flag is read back (one stream synchronisation when E >= 2), so a sorted dst holds
// no sort scratch; a growth reallocates, and nothing but the flag has been written by then.  An unsorted dst is sorted
// inside the profile scope `sort_scope` (none when null).
struct TargetOrder {
  EdgeOrder ord;
  char* head = nullptr;
  char* tail = nullptr;
};
int order_targets(eu_ctx* c, const int32_t* dst, int64_t E, int64_t n_dst, size_t head_bytes, size_t tail_bytes,
                  const char* sort_scope, TargetOrder* t);

// ---------------------------------------------------------------------------- chunked segments
// Segment s of an order is the positions [start[s], start[s + 1]); its chunk c - chunk_off[s] covers K positions from
// start[s] + (c - chunk_off[s]) * K.

// start[s] = the first position of segment s in the sorted keys `key` [P], for s in [0, n]
__global__ void k_seg_starts(const int32_t* __restrict__ key, int64_t P, int64_t n, int32_t* __restrict__ start);
// out[s, f] = the chunk sums partial[c, f] of a segment of several chunks, added in chunk order from +0; one thread per (s, f)
__global__ void k_seg_combine(const int32_t* __restrict__ chunk_off, const float* __restrict__ partial, int64_t n, int F,
                              float* __restrict__ out);

size_t seg_scan_bytes(int64_t n);   // the scan scratch of seg_chunk_offsets over n segments
// chunk_off [n + 1] = each segment's first chunk of K positions, and at n the number of chunks; nc [n + 1] and tmp (tmp_bytes
// >= seg_scan_bytes(n)) are scratch
int seg_chunk_offsets(eu_ctx* c, const int32_t* start, int64_t n, int K, int32_t* nc, void* tmp, size_t tmp_bytes,
                      int32_t* chunk_off);

// The n segments of an edge order of E positions cut into chunks of kSegChunk, in a scratch of seg_plan_bytes(E, n, width)
// bytes: start [n + 1] | nc [n + 1] | chunk_off [n + 1] | scan temp | partial chunk sums [slots, width]
struct SegPlan {
  int64_t n = 0, slots = 0;   // slots = n + E / kSegChunk >= the chunks: sum over segments of ceil(len / K) <= n + E / K
  int32_t *start = nullptr, *chunk_off = nullptr;
  float* partial = nullptr;
};
size_t seg_plan_bytes(int64_t E, int64_t n, int64_t width);
// the segment starts and chunk offsets of the order o of E > 0 edges over n segments, in buf
int plan_segments(eu_ctx* c, const EdgeOrder& o, int64_t E, int64_t n, char* buf, SegPlan* S);

// The segments of the DISTINCT keys of an order of E > 0 positions, for keys drawn from a range too large to plan over (an
// embedding table's rows): segment s < D is the s-th distinct key, D (<= E) stays on the device, so planning needs no host
// synchronisation and its scratch is O(E) whatever the key range.  Arrays of E + 1 entries cover the worst case D = E:
// segments s >= D are empty (start[s] = E, no chunks).  Chunk sums of the segments of several chunks go to
// partial[part_off[s] + (c - chunk_off[s])]: fewer than 2E / kSegChunk + 1 rows, since such a segment of len positions has
// ceil(len / K) < 2 len / K chunks.  Scratch of distinct_plan_bytes(E, width) bytes:
//   sid [E] | key, start, nc, chunk_off, part_off [E + 1] each | scan temp | partial [part_rows, width]
struct DistinctPlan {
  int64_t E = 0, part_rows = 0;
  const int32_t* nd = nullptr;   // device: D
  int32_t *key = nullptr, *start = nullptr, *chunk_off = nullptr, *part_off = nullptr;
  float* partial = nullptr;
};
size_t distinct_plan_bytes(int64_t E, int64_t width);
int plan_distinct(eu_ctx* c, const EdgeOrder& o, int64_t E, char* buf, DistinctPlan* P);

// ---------------------------------------------------------------------------- id-table rows summed per distinct id
// Every backward pass that trains id tables (embedding.cu's SparseEmbedding and ShallowEncoder, skipgram.cu, kg.cu) reduces its
// table gradients this one way, which fixes their bits: the op's own key kernel lists one int32 key (a table row) per entry;
// plan_rows orders the entries stably by key and plans the distinct rows; sum_distinct_rows sums each 256-entry chunk from +0
// and adds a row's chunk sums in chunk order, into a dense table or a coalesced COO; read_back then reads the bad-id flag and
// the distinct counts in one synchronisation.  Deterministic, no atomics, O(entries) scratch whatever the table's rows.

// a list of E entries and their chunks is indexed by int32 positions: E + E / kSegChunk + 1 < 2^31
inline bool entries_fit(int64_t E) { return E + E / kSegChunk + 1 < ((int64_t)1 << 31); }

struct RowList {                   // E entries over a table of n_rows rows
  int64_t E = 0, n_rows = 0;
  int32_t* key = nullptr;          // [E]: each entry's row, written by the caller
  EdgeOrder ord;
  DistinctPlan P;
};
// the scratch plan_rows needs for a list of E entries with width columns of chunk sums (its keys are the caller's); 0 when E = 0
size_t row_plan_bytes(int64_t E, int64_t n_rows, int64_t width);
// L's stable order by key and its distinct-row plan, in buf (row_plan_bytes), once L->key is written; nothing when E = 0
int plan_rows(eu_ctx* c, char* buf, RowList* L);

// the columns [d, d + 4) of a row of f32 or bf16 (T) widened to f32 (fewer than 4 at the row's end): one 4-wide load (VEC:
// 16 bytes of f32, 8 of bf16, so row + d is aligned to four elements) or up to four scalar loads, through the read-only
// cache, or (RW) plain loads of a row the kernel writes
template <bool VEC, typename T, bool RW = false>
__device__ __forceinline__ float4 row_load4(const T* __restrict__ row, int d, int dim) {
  if (VEC) return RW ? rw_ld4(row + d) : feat_ld4<T>(row + d);
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  v.x = RW ? rw_ld(row + d) : feat_ld<T>(row + d);
  if (d + 1 < dim) v.y = RW ? rw_ld(row + d + 1) : feat_ld<T>(row + d + 1);
  if (d + 2 < dim) v.z = RW ? rw_ld(row + d + 2) : feat_ld<T>(row + d + 2);
  if (d + 3 < dim) v.w = RW ? rw_ld(row + d + 3) : feat_ld<T>(row + d + 3);
  return v;
}

// the row of id v, or row 0 (flagged) when v lies outside [0, n_rows)
__device__ __forceinline__ int64_t row_of(int64_t v, int64_t n_rows, int* bad) {
  if (v >= 0 && v < n_rows) return v;
  *bad = 1;
  return 0;
}

// The values of an entry list ordered by row.  Entries e < n_src are stored rows gt[e, :], or, when node is given (the
// gathered kind: every entry stored), rows gt[r * ld, :] with r = node[e] / group, each element divided by pool_den first
// unless that is 0.  Entries e >= n_src have coef[t] * target[src_b, :], t = e - n_src, b = t / J (computed while they are
// summed; target is f32 or bf16, target_dtype, widened as it is read).  A list of stored rows only has n_src = its length.
struct RowEntries {
  int64_t n_src = 0;
  const float* gt = nullptr;
  const int32_t* node = nullptr;
  int ld = 0;
  int group = 1;
  float pool_den = 0.f;
  int J = 1;
  const float* coef = nullptr;
  const int64_t* src = nullptr;
  const void* target = nullptr;
  int64_t n_rows = 0;
  int target_dtype = EU_FEAT_F32;   // last: the other members keep their offsets
};

// The sums per distinct row of list L's entries S (nothing when L.E = 0): each 256-entry chunk adds its entries left to
// right from +0 as acc = fma(w, row, acc) (w = 1 for a stored row, so a plain add), a row of several chunks adds its chunk
// sums in chunk order from +0.  by_key: into the dense table out (rows not in the list untouched); else into COO values out,
// with the rows' ids in rows (may be null).  No atomics: the bits depend on each row's entry sequence only.
int sum_distinct_rows(eu_ctx* c, const RowEntries& S, const RowList& L, int dim, bool by_key, float* out, int64_t* rows);

// One stream synchronisation over a header of 1 + n int32 of device scratch: *bad = (hdr[0] != 0), the bad-id flag (bad
// null: no flag), and counts[i] = *nd[i], the distinct rows of a plan's list, for i < n <= kReadBackMax (a null nd[i], a list
// never planned, reads 0).  The counts are first copied to hdr[1 + i] on the device (unless nd[i] is that slot already), so
// the header comes back in one copy.
constexpr int kReadBackMax = EU_SHALLOW_MAX_SLOTS + 1;
int read_back(eu_ctx* c, int32_t* hdr, bool* bad, int n, const int32_t* const* nd, int64_t* counts);

// *loss = fl32((sum of rowloss[0, B)) / N): thread t adds rowloss[t], rowloss[t + 1024], ... in f64, then a shared-memory tree
// (strides 512 .. 1).  One block of kMeanThreads; N = 0 gives NaN, as a mean of nothing.
constexpr int kMeanThreads = 1024;
__global__ void k_f64_mean(const double* __restrict__ rowloss, int64_t B, int64_t N, float* __restrict__ loss);

// The forward tail of a loss over B rows (skipgram.cu, kg.cu), in the ctx scratch flag (256 B) | rowloss f64[B]: when B > 0,
// rows(flag, rowloss) launches the op's kernels, which write each row's loss and set *flag on an id outside its table; then
// *loss = the k_f64_mean of the rows over N, and *bad = the flag, read back in the call's one synchronisation.
template <class Rows>
int mean_loss(eu_ctx* c, int64_t B, int64_t N, float* loss, bool* bad, Rows rows) {
  int rc = ctx_misc(c, 256 + (int64_t)a256(8 * (size_t)B));
  if (rc) return rc;
  int32_t* flag = (int32_t*)c->d_misc;
  double* rowloss = (double*)((char*)c->d_misc + 256);
  EU_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), c->stream));
  if (B > 0 && (rc = rows(flag, rowloss))) return rc;
  k_f64_mean<<<1, kMeanThreads, 0, c->stream>>>(rowloss, B, N, loss);
  EU_LAUNCHED();
  return read_back(c, flag, bad, 0, nullptr, nullptr);
}

}  // namespace eu
