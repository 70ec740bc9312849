// SparseEmbedding's lookup from node ids, forward and backward: the uint64 ("sparse") slot of each node, turned into one
// f32 row by an embedding table, with no host round trip and no intermediate COO.  And ShallowEncoder's whole input row (an
// id embedding, dense feature slots and several such lookups, concatenated or added) in one pass over the nodes; and those
// rows pooled (sum or mean) over fixed segments of nodes without being written, what SageEncoder's first layer needs of the
// deepest hop of a fanout (k_shallow_pool; its backward is the shared one, reading gradient row node / count).
//
// Reference semantics (file:line in the upstream alibaba/euler tree):
//   SparseEmbedding.call      tf_euler/python/utils/layers.py:152-169  tf.nn.embedding_lookup_sparse(table, sp_ids, None,
//                                                                       combiner), default combiner 'sum'
//   its input                 tf_euler/kernels/get_sparse_feature_op.cc:52-130  the node's values of the slot in stored
//                             order; a node without values (absent id, empty or unknown slot) gets one entry, the default
//   ShallowEncoder.call       tf_euler/python/utils/encoders.py:134-171  [Embedding(ids), get_dense_feature, SparseEmbedding
//                             per slot], then concat or add_n
//
// Forward, for node i with bag v_0 .. v_{n-1} (n >= 1):
//   acc = table[v_0]; acc = __fadd_rn(acc, table[v_k]) for k = 1 .. n-1   (from the first row, not from +0)
//   out_i = acc (sum), __fdiv_rn(acc, fl(n)) (mean), __fdiv_rn(acc, __fsqrt_rn(fl(n))) (sqrtn)
// A group of G lanes per node: the bag's values are loaded G at a time, one per lane, and broadcast by shuffle; kEmbUnroll
// table rows are loaded ahead of the ordered adds (emb_bag_sum, which both forward kernels call).  4-wide loads when
// dim % 4 == 0, the table is aligned to four elements (16 bytes of f32, 8 of bf16) and out to 16 bytes, scalar otherwise:
// the same adds in the same order, so the bits do not depend on the alignment.  No scratch, no synchronisation: the
// forward is capturable in a CUDA graph.
//
// Tables are f32 or bf16 (E; all tables of one problem share it).  Only the forward kernels read a table, through feat_ld /
// feat_ld4, which widen bf16 to f32 exactly; every other step is the f32 one, so a bf16 call gives the f32 call's bits on
// the widened tables.  The backward never dereferences a table: emb_backward, k_emb_lengths, k_emb_entries,
// k_emb_scale_grad and segment.cuh's distinct-row sums read grad_out, the graph's bags, n_rows and dim only, so one
// backward serves both dtypes.
//
// Backward, grad_table[v] = sum over the entries (i, k) with v_k = v of s_i(g_i), where s_i is the identity (sum),
// __fdiv_rn(., fl(n_i)) (mean) or __fdiv_rn(., __fsqrt_rn(fl(n_i))) (sqrtn), elementwise.  The entries of every table are
// listed again from the graph in one pass over the nodes (k_emb_entries: each entry's value and node), then go through the
// id-table gradient path of segment.cuh that the skip-gram and KG losses share: ordered stably by value and planned
// (plan_rows), summed per distinct value in fixed chunks of kSegChunk entries (sum_distinct_rows, reading each entry's
// gradient row in place, row node / group of grad_out): deterministic, no atomics, and a hot value (the default fills every
// empty slot) is spread over many CTAs.  The sums go to a dense table (rows no entry touches are zero) or to a coalesced COO
// of the rows touched.
#include <cub/device/device_scan.cuh>

#include "segment.cuh"

namespace eu {

constexpr int kEmbUnroll = 8;   // table rows in flight per lane ahead of the ordered adds

// the combiner's divisor of a bag of n entries: fl(n) (mean), sqrtf(fl(n)) (sqrtn); sum divides by nothing
__device__ __forceinline__ float emb_den(int64_t n, int comb) { return comb == EU_COMBINE_SQRTN ? __fsqrt_rn((float)n) : (float)n; }

// the columns one lane handles per step: 4 (float4) or 1
template <bool VEC> struct EmbVec;
template <> struct EmbVec<true> {
  using T = float4;
  static constexpr int W = 4;
  static __device__ __forceinline__ T zero(float z) { return make_float4(z, z, z, z); }
  template <typename E> static __device__ __forceinline__ T load(const E* p) { return feat_ld4<E>(p); }
  static __device__ __forceinline__ T load_rw(const float* p) { return *reinterpret_cast<const float4*>(p); }   // written by this kernel
  static __device__ __forceinline__ void store(float* p, T v) { *reinterpret_cast<float4*>(p) = v; }
  static __device__ __forceinline__ T add(T a, T b) {
    return make_float4(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z), __fadd_rn(a.w, b.w));
  }
  static __device__ __forceinline__ T div(T a, float den) {
    return make_float4(__fdiv_rn(a.x, den), __fdiv_rn(a.y, den), __fdiv_rn(a.z, den), __fdiv_rn(a.w, den));
  }
};
template <> struct EmbVec<false> {
  using T = float;
  static constexpr int W = 1;
  static __device__ __forceinline__ T zero(float z) { return z; }
  template <typename E> static __device__ __forceinline__ T load(const E* p) { return feat_ld<E>(p); }
  static __device__ __forceinline__ T load_rw(const float* p) { return *p; }
  static __device__ __forceinline__ void store(float* p, T v) { *p = v; }
  static __device__ __forceinline__ T add(T a, T b) { return __fadd_rn(a, b); }
  static __device__ __forceinline__ T div(T a, float den) { return __fdiv_rn(a, den); }
};

// This lane's columns [d, d + W) of the sum of the bag [b, e) of the uint64 values (empty: the one entry dflt), whole-group
// call (every lane of the group takes part in the shuffles; act: d < dim, an inactive lane loads nothing).  The sum starts
// from the bag's first row (its bits, -0.0 and NaN payloads included) and adds the others left to right.
template <bool VEC, typename E>
__device__ __forceinline__ typename EmbVec<VEC>::T emb_bag_tile(const DevGraph& g, int64_t b, int64_t e, unsigned long long dflt,
                                                                const E* __restrict__ table, int dim, int d, bool act, int G,
                                                                int sub, unsigned gm) {
  using V = EmbVec<VEC>;
  const bool empty = e == b;
  const int64_t n = empty ? 1 : e - b;
  typename V::T acc = V::zero(0.f);
  for (int64_t k0 = 0; k0 < n; k0 += G) {
    const unsigned long long mine = k0 + sub < n ? (empty ? dflt : __ldg(g.u64_val + b + k0 + sub)) : 0ull;
    const int cnt = n - k0 < G ? (int)(n - k0) : G;
    for (int j0 = 0; j0 < cnt; j0 += kEmbUnroll) {
      typename V::T x[kEmbUnroll];
#pragma unroll
      for (int q = 0; q < kEmbUnroll; ++q) {
        const unsigned long long v = __shfl_sync(gm, mine, (j0 + q) & (G - 1), G);
        x[q] = act && j0 + q < cnt ? V::load(table + (int64_t)v * dim + d) : V::zero(0.f);
      }
#pragma unroll
      for (int q = 0; q < kEmbUnroll; ++q)
        if (j0 + q < cnt) acc = k0 + j0 + q == 0 ? x[q] : V::add(acc, x[q]);
    }
  }
  return acc;
}

// The bag sum of graph row `row` (-1: absent) in slot fid, before the combiner's division: G lanes (this one is `sub`, the
// group's mask gm), W columns per lane and step, blocks of G * W columns with a group-uniform trip count (emb_bag_tile).
// *n = the bag's entries (1 for the default); it is set before the first sink(d, acc) call, which hands over the lane's
// columns [d, d + W) of the sum, for d < dim only.
template <bool VEC, typename E, typename Sink>
__device__ __forceinline__ void emb_bag_sum(const DevGraph& g, int64_t row, int32_t fid, unsigned long long dflt,
                                            const E* __restrict__ table, int dim, int G, int sub, unsigned gm, int64_t* n_out,
                                            Sink sink) {
  using V = EmbVec<VEC>;
  int64_t b, e;
  ragged_slice(g.u64_ptr, g.n_u64_slots, row, fid, &b, &e);
  *n_out = e == b ? 1 : e - b;
  for (int d0 = 0; d0 < dim; d0 += G * V::W) {
    const int d = d0 + sub * V::W;
    const typename V::T acc = emb_bag_tile<VEC, E>(g, b, e, dflt, table, dim, d, d < dim, G, sub, gm);
    if (d < dim) sink(d, acc);
  }
}

// G lanes per node r (a power of two)
template <bool VEC, typename E>
__global__ void __launch_bounds__(256, 1) k_emb_fwd(DevGraph g, const unsigned long long* __restrict__ nodes, int64_t M, int32_t fid,
                                                 unsigned long long dflt, const E* __restrict__ table, int dim, int G, int comb,
                                                 float* __restrict__ out) {
  using V = EmbVec<VEC>;
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t r = tid >> (31 - __clz(G));
  const int sub = (int)(tid & (G - 1));
  if (r >= M) return;   // group-uniform
  const unsigned gm = group_mask(G);
  float* o = out + r * (int64_t)dim;
  int64_t n;
  emb_bag_sum<VEC, E>(g, lookup_row(g, __ldg(nodes + r)), fid, dflt, table, dim, G, sub, gm, &n,
                   [&](int d, typename V::T acc) { V::store(o + d, acc); });
  if (comb == EU_COMBINE_SUM) return;
  // mean / sqrtn: one division per column, in a pass of its own over the row this group just wrote (L1-resident), so that
  // nothing of the bag loop is live across the division's slow-path subroutine
  __syncwarp(gm);
  const float den = emb_den(n, comb);
  for (int d = sub; d < dim; d += G) o[d] = __fdiv_rn(o[d], den);
}

// ---------------------------------------------------------------------------- ShallowEncoder's row
struct ShallowDev {   // eu_shallow_problem, resolved for the device: column offsets, and which slots take float4 loads
  const unsigned long long* nodes;
  int64_t M;
  int W, add;                      // out's width; EU_SHALLOW_ADD
  const void* id_table;            // every table of the problem: f32, or bf16 (the kernels' E)
  int64_t n_id_rows;
  int id_dim;
  int n_dense, dense_w;            // dense_w: dense_out's width (ADD)
  int32_t dense_fid[EU_SHALLOW_MAX_SLOTS];
  int dense_dim[EU_SHALLOW_MAX_SLOTS], dense_off[EU_SHALLOW_MAX_SLOTS];
  int n_sparse;
  unsigned vec_mask;               // bit s: slot s's table and out columns take 4-wide loads and float4 stores
  int32_t sp_fid[EU_SHALLOW_MAX_SLOTS];
  int sp_dim[EU_SHALLOW_MAX_SLOTS], sp_comb[EU_SHALLOW_MAX_SLOTS], sp_off[EU_SHALLOW_MAX_SLOTS];
  unsigned long long sp_dflt[EU_SHALLOW_MAX_SLOTS];
  const void* sp_table[EU_SHALLOW_MAX_SLOTS];
  float* out;
  float* dense_out;
};

// slot s of node row `row` into o (its first column): stored (CONCAT, or the first term of ADD) or added to what o holds
template <bool VEC, typename E>
__device__ __forceinline__ void shallow_slot(const DevGraph& g, const ShallowDev& p, int s, int64_t row, float* o, bool first, int G,
                                             int sub, unsigned gm) {
  using V = EmbVec<VEC>;
  const int comb = p.sp_comb[s];
  int64_t n;
  emb_bag_sum<VEC, E>(g, row, p.sp_fid[s], p.sp_dflt[s], static_cast<const E*>(p.sp_table[s]), p.sp_dim[s], G, sub, gm, &n, [&](int d, typename V::T acc) {
    if (comb != EU_COMBINE_SUM) acc = V::div(acc, emb_den(n, comb));
    V::store(o + d, first ? acc : V::add(V::load_rw(o + d), acc));
  });
}

// G lanes per node r: the id columns, the dense slots (k_feature's rule: the stored columns, zeros past them, zeros for an
// absent node or an unknown slot), then the sparse slots.  The group syncs between parts: a part may map columns to lanes
// differently from the one before it, and ADD reads what the previous part wrote.  T: the dense table's storage type and P its
// placement, E the id and sparse tables' storage type.
template <typename T, typename E, int P>
__global__ void __launch_bounds__(256) k_shallow_fwd(DevGraph g, ShallowDev p, int G) {
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t r = tid >> (31 - __clz(G));
  const int sub = (int)(tid & (G - 1));
  if (r >= p.M) return;   // group-uniform
  const unsigned gm = group_mask(G);
  const unsigned long long id = __ldg(p.nodes + r);
  float* o = p.out + r * (int64_t)p.W;
  if (p.id_table) {
    const bool ok = (long long)id >= 0 && (long long)id < p.n_id_rows;   // false only under capture (the check is skipped)
    const E* t = static_cast<const E*>(p.id_table) + (ok ? (int64_t)id : 0) * p.id_dim;
    for (int d = sub; d < p.id_dim; d += G) o[d] = ok ? feat_ld<E>(t + d) : __int_as_float(0x7fc00000);
  }
  const int64_t row = lookup_row(g, id);
  float* od = p.add ? p.dense_out + r * (int64_t)p.dense_w : o;
  for (int j = 0; j < p.n_dense; ++j) {
    const int32_t fid = p.dense_fid[j];
    const bool have = fid >= 0 && fid < g.n_slots && row >= 0;
    const int sdim = have ? g.slot_dim[fid] : 0;
    const T* f = feat_row_if<T, P>(g, have, row, have ? g.slot_off[fid] : 0);
    float* oj = od + p.dense_off[j];
    for (int d = sub; d < p.dense_dim[j]; d += G) oj[d] = d < sdim ? feat_ld(f + d) : 0.f;
  }
  for (int s = 0; s < p.n_sparse; ++s) {
    __syncwarp(gm);
    const bool first = !p.add || (s == 0 && !p.id_table);
    float* os = o + p.sp_off[s];
    if (p.vec_mask >> s & 1) shallow_slot<true, E>(g, p, s, row, os, first, G, sub, gm);
    else shallow_slot<false, E>(g, p, s, row, os, first, G, sub, gm);
  }
}

// ---------------------------------------------------------------------------- ShallowEncoder's rows, pooled per segment
// One pooled column: load(0), then load(j) added left to right for j = 1 .. count - 1, kEmbUnroll loads ahead of the adds
template <typename Load>
__device__ __forceinline__ float pool_column(int count, Load load) {
  float acc = 0.f;
  for (int j0 = 0; j0 < count; j0 += kEmbUnroll) {
    float x[kEmbUnroll];
#pragma unroll
    for (int q = 0; q < kEmbUnroll; ++q)
      if (j0 + q < count) x[q] = load(j0 + q);
#pragma unroll
    for (int q = 0; q < kEmbUnroll; ++q)
      if (j0 + q < count) acc = j0 + q == 0 ? x[q] : __fadd_rn(acc, x[q]);
  }
  return acc;
}

// slot s of the segment's nodes (their graph rows in `rows`), pooled into o (the slot's first column of the output row):
// per tile of G * W columns, each node's bag sum and combiner division (shallow_slot's), added across the nodes in registers
template <bool VEC, typename E>
__device__ __forceinline__ void shallow_pool_slot(const DevGraph& g, const ShallowDev& p, int s, const int64_t* rows, int count,
                                                  float pool_den, float* o, int G, int sub, unsigned gm) {
  using V = EmbVec<VEC>;
  const int comb = p.sp_comb[s], dim = p.sp_dim[s];
  for (int d0 = 0; d0 < dim; d0 += G * V::W) {
    const int d = d0 + sub * V::W;
    typename V::T acc = V::zero(0.f);
    for (int j = 0; j < count; ++j) {
      int64_t b, e;
      ragged_slice(g.u64_ptr, g.n_u64_slots, rows[j], p.sp_fid[s], &b, &e);
      typename V::T x = emb_bag_tile<VEC, E>(g, b, e, p.sp_dflt[s], static_cast<const E*>(p.sp_table[s]), dim, d, d < dim, G, sub, gm);
      if (comb != EU_COMBINE_SUM) x = V::div(x, emb_den(e == b ? 1 : e - b, comb));
      acc = j == 0 ? x : V::add(acc, x);
    }
    if (pool_den != 0.f) acc = V::div(acc, pool_den);
    if (d < dim) V::store(o + d, acc);
  }
}

// G lanes per output row r, the pool of the `count` ShallowEncoder rows (CONCAT) of nodes[r * count ..]: k_shallow_fwd's
// parts and rules, each column summed over the segment's nodes in a register, in node order, and divided once by pool_den
// (fl(count); 0: the sum).  The group looks every node's graph row up once, into its `count` slots of shared memory.
template <typename T, typename E, int P>
__global__ void __launch_bounds__(256, 2) k_shallow_pool(DevGraph g, ShallowDev p, int count, float pool_den, int G) {
  extern __shared__ int64_t pool_rows[];
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t r = tid >> (31 - __clz(G));
  const int sub = (int)(tid & (G - 1));
  if (r >= p.M / count) return;   // group-uniform
  const unsigned gm = group_mask(G);
  const unsigned long long* nodes = p.nodes + r * count;
  int64_t* rows = pool_rows + (threadIdx.x >> (31 - __clz(G))) * (int64_t)count;
  for (int j = sub; j < count; j += G) rows[j] = lookup_row(g, __ldg(nodes + j));
  __syncwarp(gm);
  float* o = p.out + r * (int64_t)p.W;
  auto finish = [&](float acc) { return pool_den != 0.f ? __fdiv_rn(acc, pool_den) : acc; };
  for (int d = sub; d < p.id_dim; d += G)
    o[d] = finish(pool_column(count, [&](int j) {
      const long long id = (long long)__ldg(nodes + j);
      const bool ok = id >= 0 && id < p.n_id_rows;   // false only under capture (the check is skipped)
      return ok ? feat_ld<E>(static_cast<const E*>(p.id_table) + id * p.id_dim + d) : __int_as_float(0x7fc00000);
    }));
  for (int k = 0; k < p.n_dense; ++k) {
    const int32_t fid = p.dense_fid[k];
    const bool known = fid >= 0 && fid < g.n_slots;
    const int sdim = known ? g.slot_dim[fid] : 0;
    const int32_t soff = known ? g.slot_off[fid] : 0;
    float* oj = o + p.dense_off[k];
    for (int d = sub; d < p.dense_dim[k]; d += G)
      oj[d] = finish(pool_column(count, [&](int j) { return d < sdim && rows[j] >= 0 ? feat_ld(feat_row<T, P>(g, rows[j], g.feat_dim, soff) + d) : 0.f; }));
  }
  for (int s = 0; s < p.n_sparse; ++s) {
    if (p.vec_mask >> s & 1) shallow_pool_slot<true, E>(g, p, s, rows, count, pool_den, o + p.sp_off[s], G, sub, gm);
    else shallow_pool_slot<false, E>(g, p, s, rows, count, pool_den, o + p.sp_off[s], G, sub, gm);
  }
}

// *bad = 1 when an id lies outside [0, n_rows)
__global__ void k_id_range(const int64_t* __restrict__ ids, int64_t M, int64_t n_rows, int* bad) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < M; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t v = __ldg(ids + i);
    if (v < 0 || v >= n_rows) *bad = 1;
  }
}

// ---------------------------------------------------------------------------- backward
// The tables of one backward pass: the uint64 slots s < S (their bags), then optionally the id table (the node ids).  Each
// one's gradient rows are grad_out[i, col .. col + dim) with row stride ld.
struct EmbTables {
  int S = 0;
  int32_t fid[EU_SHALLOW_MAX_SLOTS] = {};
  unsigned long long dflt[EU_SHALLOW_MAX_SLOTS] = {};
  int comb[EU_SHALLOW_MAX_SLOTS] = {};
  bool has_id = false;
  int64_t n_rows[EU_SHALLOW_MAX_SLOTS + 1] = {}, col[EU_SHALLOW_MAX_SLOTS + 1] = {};
  int dim[EU_SHALLOW_MAX_SLOTS + 1] = {};
};
struct EmbSlots {   // the device copy of the slots' ids and defaults
  int32_t fid[EU_SHALLOW_MAX_SLOTS];
  unsigned long long dflt[EU_SHALLOW_MAX_SLOTS];
};

// len[s * (M + 1) + i + 1] = the entries of node i in slot s (1 for the default), len[s * (M + 1)] = 0: one inclusive scan over
// all S (M + 1) then gives slot s's entries of node i at [ptr[s (M + 1) + i], ptr[s (M + 1) + i + 1]), the slots one after another
__global__ void k_emb_lengths(DevGraph g, const unsigned long long* __restrict__ nodes, int64_t M, EmbSlots sl, int S,
                              long long* __restrict__ len) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < M; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = lookup_row(g, __ldg(nodes + i));
    for (int s = 0; s < S; ++s) {
      int64_t b, e;
      ragged_slice(g.u64_ptr, g.n_u64_slots, row, sl.fid[s], &b, &e);
      len[s * (M + 1) + i + 1] = e == b ? 1 : e - b;
      if (i == 0) len[s * (M + 1)] = 0;
    }
  }
}

// One warp per node i: the key (the row) and the node of each of its entries in every slot, and its id entry at id_base + i
// (id_base < 0: no id table)
__global__ void __launch_bounds__(256) k_emb_entries(DevGraph g, const unsigned long long* __restrict__ nodes, int64_t M, EmbSlots sl,
                                                     int S, const int64_t* __restrict__ ptr, int64_t id_base, int32_t* __restrict__ key,
                                                     int32_t* __restrict__ node) {
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; i < M; i += nwarps) {
    const unsigned long long id = __ldg(nodes + i);
    const int64_t row = lookup_row(g, id);
    if (id_base >= 0 && lane == 0) { key[id_base + i] = (int32_t)id; node[id_base + i] = (int32_t)i; }
    for (int s = 0; s < S; ++s) {
      int64_t b, e;
      ragged_slice(g.u64_ptr, g.n_u64_slots, row, sl.fid[s], &b, &e);
      const int64_t o = __ldg(ptr + s * (M + 1) + i);
      if (e == b) {
        if (lane == 0) { key[o] = (int32_t)sl.dflt[s]; node[o] = (int32_t)i; }
        continue;
      }
      for (int64_t k = lane; k < e - b; k += 32) {
        key[o + k] = (int32_t)__ldg(g.u64_val + b + k);
        node[o + k] = (int32_t)i;
      }
    }
  }
}

// How the nodes share gradient rows: node i reads row i / group of grad_out, divided first by pool_den (one __fdiv_rn per
// element read) unless that is 0.  {1, 0}: a row per node, as it is -- the ops that do not pool.
struct GradRows {
  int group = 1;
  float pool_den = 0.f;
};

// gs[i, d] = g[(i / group) * ld + d] (pooled: / pool_den) / den(n_i) (one __fdiv_rn), n_i = ptr[i + 1] - ptr[i]: the scaled
// gradient of the mean and sqrtn combiners, once per node and column rather than once per entry
__global__ void k_emb_scale_grad(const float* __restrict__ g, int64_t ld, GradRows gr, const int64_t* __restrict__ ptr, int64_t M, int dim,
                                 int comb, float* __restrict__ gs) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < M * dim; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / dim;
    float x = __ldg(g + (i / gr.group) * ld + (t - i * dim));
    if (gr.pool_den != 0.f) x = __fdiv_rn(x, gr.pool_den);
    gs[t] = __fdiv_rn(x, emb_den(__ldg(ptr + i + 1) - __ldg(ptr + i), comb));
  }
}

// The checks of one uint64 slot and its table.  Every value of slot fid and the default must index the table: the slot's
// largest value is kept on the graph, so this costs no device work.
static int emb_slot_check(const eu_graph* g, int32_t fid, int64_t default_value, int64_t n_rows, const char* who) {
  if (default_value < 0 || default_value >= n_rows) {
    set_error("%s: default_value %lld lies outside the table's rows [0, %lld)", who, (long long)default_value, (long long)n_rows);
    return EU_ERR_INVALID;
  }
  if (fid >= 0 && fid < (int32_t)g->u64_slot_max.size() && g->u64_slot_max[fid] >= (uint64_t)n_rows) {
    set_error("%s: slot %d holds the value %llu, outside the table's rows [0, %lld)", who, (int)fid,
              (unsigned long long)g->u64_slot_max[fid], (long long)n_rows);
    return EU_ERR_INVALID;
  }
  return EU_OK;
}

// The checks the passes of the single-slot op share; ok: the pass's own table / output pointers are given.
static int emb_check(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int64_t default_value, bool ok, int64_t n_rows,
                     int32_t dim, int32_t combiner, const void* out, const char* who) {
  if (!c || M < 0 || n_rows < 1 || dim < 1 || combiner < EU_COMBINE_SUM || combiner > EU_COMBINE_SQRTN || (M > 0 && (!nodes || !out)) ||
      !ok) {
    set_error("%s: bad argument", who);
    return EU_ERR_INVALID;
  }
  if (M >= ((int64_t)1 << 31) || n_rows >= ((int64_t)1 << 31)) {
    set_error("%s: 2^31 or more nodes or table rows are not supported", who);
    return EU_ERR_UNSUPPORTED;
  }
  return emb_slot_check(c->g, fid, default_value, n_rows, who);
}

// *bad_host = whether an id of ids [M] lies outside [0, n_rows): one kernel and one synchronisation
static int id_range_check(eu_ctx* c, const int64_t* ids, int64_t M, int64_t n_rows, bool* bad_host) {
  int rc = ctx_misc(c, 256);
  if (rc) return rc;
  int* bad = (int*)c->d_misc;
  EU_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), c->stream));
  k_id_range<<<stride_grid(M), 256, 0, c->stream>>>(ids, M, n_rows, bad);
  EU_LAUNCHED();
  int h = 0;
  EU_CUDA(cudaMemcpyAsync(&h, bad, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  EU_CUDA(cudaStreamSynchronize(c->stream));
  *bad_host = h != 0;
  return EU_OK;
}

// The gradients of the tables T over the nodes [M] (checked by the caller), from grad_out with row stride ld, node i's row
// being row i / gr.group of it (GradRows).  Dense
// (rows == null): grads[t] f32[n_rows_t, dim_t], zeroed first.  Sparse: the COO rows[t] / grads[t] with counts[t] (host).
// Table t < S is slot t, table S the id table.
static int emb_backward(eu_ctx* c, const EmbTables& T, const int64_t* nodes, int64_t M, const float* grad_out, int64_t ld, GradRows gr,
                        float* const* grads, int64_t* const* rows, int64_t* counts, const char* who) {
  EU_CUDA(cudaSetDevice(c->g->device));
  cudaStream_t s = c->stream;
  const bool sparse = rows != nullptr;
  const int S = T.S, NT = S + (T.has_id ? 1 : 0);
  if (!sparse)
    for (int t = 0; t < NT; ++t) EU_CUDA(cudaMemsetAsync(grads[t], 0, 4 * (size_t)T.n_rows[t] * T.dim[t], s));
  if (sparse)
    for (int t = 0; t < NT; ++t) counts[t] = 0;
  if (M == 0) return EU_OK;
  EmbSlots sl;
  for (int k = 0; k < S; ++k) { sl.fid[k] = T.fid[k]; sl.dflt[k] = T.dflt[k]; }
  // flag, the distinct counts (256 B) | ptr [S (M + 1)] | scan temp | then, once the entry counts are known:
  // key [E] | node [E] | scaled gradients [M, dim] | one table's order and plan (reused table after table)
  const int64_t NP = (int64_t)S * (M + 1);
  const size_t o_ptr = 256, o_tmp = o_ptr + a256(8 * (size_t)NP), tmp = S ? ragged_scan_bytes(NP - 1) : 0, o_key = o_tmp + a256(tmp);
  auto entry_ptr = [&]() -> int {
    if (!S) return EU_OK;
    k_emb_lengths<<<stride_grid(M), 256, 0, s>>>(c->g->d, (const unsigned long long*)nodes, M, sl, S, (long long*)((char*)c->d_misc + o_ptr));
    EU_LAUNCHED();
    long long* p = (long long*)((char*)c->d_misc + o_ptr);
    size_t t = tmp;
    EU_CUDA(cub::DeviceScan::InclusiveSum((char*)c->d_misc + o_tmp, t, p, p, (int)NP, s));
    EU_LAUNCHED();
    return EU_OK;
  };
  int rc = ctx_misc(c, (int64_t)o_key);
  if (rc) return rc;
  int* bad = (int*)c->d_misc;
  EU_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), s));
  if (T.has_id) {
    k_id_range<<<stride_grid(M), 256, 0, s>>>(nodes, M, T.n_rows[S], bad);
    EU_LAUNCHED();
  }
  if ((rc = entry_ptr())) return rc;
  int64_t h_end[EU_SHALLOW_MAX_SLOTS] = {};
  int h_bad = 0;
  EU_CUDA(cudaMemcpyAsync(&h_bad, bad, sizeof(int), cudaMemcpyDeviceToHost, s));
  for (int k = 0; k < S; ++k)
    EU_CUDA(cudaMemcpyAsync(h_end + k, (int64_t*)((char*)c->d_misc + o_ptr) + k * (M + 1) + M, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
  EU_CUDA(cudaStreamSynchronize(s));
  if (h_bad) {
    set_error("%s: a node id lies outside the id table's rows [0, %lld)", who, (long long)T.n_rows[S]);
    return EU_ERR_INVALID;
  }
  int64_t base[EU_SHALLOW_MAX_SLOTS + 1], E_t[EU_SHALLOW_MAX_SLOTS + 1];
  for (int k = 0; k < S; ++k) { base[k] = k ? h_end[k - 1] : 0; E_t[k] = h_end[k] - base[k]; }
  const int64_t E = (S ? h_end[S - 1] : 0) + (T.has_id ? M : 0);
  if (T.has_id) { base[S] = E - M; E_t[S] = M; }
  if (!entries_fit(E)) {
    set_error("%s: 2^31 or more entries are not supported", who);
    return EU_ERR_UNSUPPORTED;
  }
  int scaled_dim = 0;
  size_t region = 0;
  for (int t = 0; t < NT; ++t) {
    if (t < S && T.comb[t] != EU_COMBINE_SUM) scaled_dim = std::max(scaled_dim, T.dim[t]);
    region = std::max(region, row_plan_bytes(E_t[t], T.n_rows[t], T.dim[t]));
  }
  const size_t o_node = o_key + a256(4 * (size_t)E), o_gs = o_node + a256(4 * (size_t)E), o_reg = o_gs + a256(4 * (size_t)M * scaled_dim);
  const size_t total = o_reg + region;
  if ((int64_t)total > c->misc_bytes) {   // the growth reallocates: the offsets again (no read-back needed)
    if ((rc = ctx_misc(c, (int64_t)total))) return rc;
    if ((rc = entry_ptr())) return rc;
  }
  char* m = (char*)c->d_misc;
  int32_t* hdr = (int32_t*)m;   // read_back's header: the (spent) flag, then each table's distinct count
  const int64_t* ptr = (const int64_t*)(m + o_ptr);
  int32_t* key = (int32_t*)(m + o_key);
  int32_t* node = (int32_t*)(m + o_node);
  {
    EuProfScope ps(c, "emb_bwd_entries", E);
    k_emb_entries<<<stride_grid(M * 32), 256, 0, s>>>(c->g->d, (const unsigned long long*)nodes, M, sl, S, ptr, T.has_id ? base[S] : -1,
                                                      key, node);
    EU_LAUNCHED();
  }
  const int32_t* nd[kReadBackMax];   // each table's count, copied to its header slot before the plan's scratch is reused
  for (int t = 0; t < NT; ++t) {
    const int dim = T.dim[t];
    RowList L;
    L.E = E_t[t];
    L.n_rows = T.n_rows[t];
    L.key = key + base[t];
    {
      EuProfScope ps(c, "emb_bwd_order", L.E);
      if ((rc = plan_rows(c, m + o_reg, &L))) return rc;
    }
    EuProfScope ps(c, "emb_bwd_sums", L.E);
    RowEntries R;   // the gathered kind: entry e's row is grad_out's row node[e] / group, from the table's column
    R.n_src = L.E;
    R.gt = grad_out + T.col[t];
    R.ld = (int)ld;   // a row of at most EU_SHALLOW_MAX_WIDTH columns
    R.node = node + base[t];
    R.group = gr.group;
    R.pool_den = gr.pool_den;
    if (t < S && T.comb[t] != EU_COMBINE_SUM) {   // a row per node, the pool's division done
      float* scaled = (float*)(m + o_gs);
      k_emb_scale_grad<<<stride_grid(M * dim), 256, 0, s>>>(R.gt, ld, gr, ptr + t * (M + 1), M, dim, T.comb[t], scaled);
      EU_LAUNCHED();
      R.gt = scaled;
      R.ld = dim;
      R.group = 1;
      R.pool_den = 0.f;
    }
    if ((rc = sum_distinct_rows(c, R, L, dim, !sparse, grads[t], sparse ? rows[t] : nullptr))) return rc;
    nd[t] = hdr + 1 + t;
    if (sparse) EU_CUDA(cudaMemcpyAsync(hdr + 1 + t, L.P.nd, sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
  }
  return sparse ? read_back(c, hdr, nullptr, NT, nd, counts) : EU_OK;
}

// The single-slot op as a one-table backward pass
static int single_backward(eu_ctx* c, const float* grad_out, const int64_t* nodes, int64_t M, int32_t fid, int64_t default_value,
                           int64_t n_rows, int32_t dim, int32_t combiner, float* out, int64_t* rows, int64_t* n, const char* who) {
  EmbTables T;
  T.S = 1;
  T.fid[0] = fid;
  T.dflt[0] = (unsigned long long)default_value;
  T.comb[0] = combiner;
  T.n_rows[0] = n_rows;
  T.dim[0] = dim;
  float* g[1] = {out};
  int64_t* r[1] = {rows};
  return emb_backward(c, T, nodes, M, grad_out, dim, GradRows(), g, rows ? r : nullptr, n, who);
}

// The checks of a shallow problem, and its device form (out / dense_out filled in by the caller).  *T: its backward tables.
static int shallow_resolve(eu_ctx* c, const eu_shallow_problem* p, ShallowDev* d, EmbTables* T, const char* who) {
  if (!c || !p || p->M < 0 || (p->M > 0 && !p->nodes) || (p->combiner != EU_SHALLOW_CONCAT && p->combiner != EU_SHALLOW_ADD) ||
      p->n_dense < 0 || p->n_sparse < 0 || (p->id_table && (p->n_id_rows < 1 || p->id_dim < 1))) {
    set_error("%s: bad argument", who);
    return EU_ERR_INVALID;
  }
  if (p->n_dense > EU_SHALLOW_MAX_SLOTS || p->n_sparse > EU_SHALLOW_MAX_SLOTS) {
    set_error("%s: at most %d dense and %d sparse slots are supported", who, EU_SHALLOW_MAX_SLOTS, EU_SHALLOW_MAX_SLOTS);
    return EU_ERR_UNSUPPORTED;
  }
  *d = ShallowDev();
  *T = EmbTables();
  const bool add = p->combiner == EU_SHALLOW_ADD;
  int64_t w = p->id_table ? p->id_dim : 0, dw = 0, emb_dim = p->id_table ? p->id_dim : -1;
  d->n_dense = p->n_dense;
  for (int j = 0; j < p->n_dense; ++j) {
    if (p->dense[j].dim < 0) {
      set_error("%s: dense slot %d has dim %d", who, j, (int)p->dense[j].dim);
      return EU_ERR_INVALID;
    }
    d->dense_fid[j] = p->dense[j].fid;
    d->dense_dim[j] = p->dense[j].dim;
    d->dense_off[j] = (int)std::min<int64_t>(add ? dw : w, EU_SHALLOW_MAX_WIDTH + 1);
    (add ? dw : w) += p->dense[j].dim;
  }
  d->n_sparse = T->S = p->n_sparse;
  for (int k = 0; k < p->n_sparse; ++k) {
    const eu_shallow_sparse& q = p->sparse[k];
    if (!q.table || q.n_rows < 1 || q.dim < 1 || q.combiner < EU_COMBINE_SUM || q.combiner > EU_COMBINE_SQRTN) {
      set_error("%s: sparse slot %d: bad argument", who, k);
      return EU_ERR_INVALID;
    }
    if (add && emb_dim >= 0 && q.dim != emb_dim) {
      set_error("%s: 'add' needs one dim for every embedding, got %lld and %d", who, (long long)emb_dim, (int)q.dim);
      return EU_ERR_INVALID;
    }
    emb_dim = q.dim;
    if (q.n_rows >= ((int64_t)1 << 31)) {
      set_error("%s: tables of 2^31 or more rows are not supported", who);
      return EU_ERR_UNSUPPORTED;
    }
    int rc = emb_slot_check(c->g, q.fid, q.default_value, q.n_rows, who);
    if (rc) return rc;
    d->sp_fid[k] = T->fid[k] = q.fid;
    d->sp_dflt[k] = T->dflt[k] = (unsigned long long)q.default_value;
    d->sp_comb[k] = T->comb[k] = q.combiner;
    d->sp_dim[k] = T->dim[k] = q.dim;
    d->sp_table[k] = q.table;
    d->sp_off[k] = (int)std::min<int64_t>(add ? 0 : w, EU_SHALLOW_MAX_WIDTH + 1);
    T->n_rows[k] = q.n_rows;
    T->col[k] = d->sp_off[k];
    if (!add) w += q.dim;
  }
  if (add) w = std::max<int64_t>(emb_dim, 0);
  if (w > EU_SHALLOW_MAX_WIDTH || dw > EU_SHALLOW_MAX_WIDTH) {
    set_error("%s: rows of more than %d columns are not supported", who, EU_SHALLOW_MAX_WIDTH);
    return EU_ERR_UNSUPPORTED;
  }
  if (p->M >= ((int64_t)1 << 31) || p->n_id_rows >= ((int64_t)1 << 31)) {
    set_error("%s: 2^31 or more nodes or table rows are not supported", who);
    return EU_ERR_UNSUPPORTED;
  }
  d->nodes = (const unsigned long long*)p->nodes;
  d->M = p->M;
  d->W = (int)w;
  d->add = add;
  d->id_table = p->id_table;
  d->n_id_rows = p->n_id_rows;
  d->id_dim = p->id_table ? p->id_dim : 0;
  d->dense_w = (int)dw;
  T->has_id = p->id_table != nullptr;
  if (T->has_id) {
    T->n_rows[T->S] = p->n_id_rows;
    T->dim[T->S] = p->id_dim;
    T->col[T->S] = 0;
  }
  return EU_OK;
}

// The pooled op's own checks, after shallow_resolve's; *gr: how its backward reads grad_out f32[M / count, W]
static int pool_check(const eu_shallow_problem* p, int32_t count, int32_t pool, GradRows* gr, const char* who) {
  if (count < 1 || p->M % count || (pool != EU_POOL_SUM && pool != EU_POOL_MEAN)) {
    set_error("%s: count = %d must be at least 1 and divide M = %lld, pool must be EU_POOL_SUM or EU_POOL_MEAN", who, (int)count,
              (long long)p->M);
    return EU_ERR_INVALID;
  }
  if (p->combiner != EU_SHALLOW_CONCAT) {
    set_error("%s: only EU_SHALLOW_CONCAT rows are pooled", who);
    return EU_ERR_UNSUPPORTED;
  }
  if (count > EU_SHALLOW_POOL_MAX_COUNT) {
    set_error("%s: segments of more than %d nodes are not supported", who, EU_SHALLOW_POOL_MAX_COUNT);
    return EU_ERR_UNSUPPORTED;
  }
  gr->group = count;
  gr->pool_den = pool == EU_POOL_MEAN ? (float)count : 0.f;
  return EU_OK;
}

// outside capture: every id must index the id table before anything is written
static int shallow_id_check(eu_ctx* c, const eu_shallow_problem* p, const char* who) {
  if (!p->id_table) return EU_OK;
  cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
  EU_CUDA(cudaStreamIsCapturing(c->stream, &st));
  if (st != cudaStreamCaptureStatusNone) return EU_OK;
  bool bad = false;
  int rc = id_range_check(c, p->nodes, p->M, p->n_id_rows, &bad);
  if (rc) return rc;
  if (bad) {
    set_error("%s: a node id lies outside the id table's rows [0, %lld)", who, (long long)p->n_id_rows);
    return EU_ERR_INVALID;
  }
  return EU_OK;
}

// the lane group of a row whose widest part has `widest` columns, and the slots that take 4-wide loads and float4 stores (a
// table aligned to four elements of table_dtype, the output to 16 bytes)
static int shallow_lanes(ShallowDev* d, const float* out, int table_dtype) {
  int widest = d->id_dim;
  for (int j = 0; j < d->n_dense; ++j) widest = std::max(widest, d->dense_dim[j]);
  for (int k = 0; k < d->n_sparse; ++k) {
    widest = std::max(widest, d->sp_dim[k]);
    if (d->sp_dim[k] % 4 == 0 && aligned4_elems(d->sp_table[k], table_dtype) && aligned16(out) && d->W % 4 == 0 && d->sp_off[k] % 4 == 0)
      d->vec_mask |= 1u << k;
  }
  return group_lanes(ceil_div(widest, 4));
}

// eu_shallow_encode_backward and its pooled form (gr)
static int shallow_backward(eu_ctx* c, const eu_shallow_problem* p, const ShallowDev& d, const EmbTables& T, GradRows gr,
                            const float* grad_out, float* const* grads, const char* who) {
  const int NT = T.S + (T.has_id ? 1 : 0);
  bool ok = grads && (p->M == 0 || d.W == 0 || grad_out);
  for (int t = 0; ok && t < NT; ++t) ok = grads[t == T.S ? 0 : t + 1] != nullptr;
  if (!ok) {
    set_error("%s: bad argument (grad_out and a gradient per table are required)", who);
    return EU_ERR_INVALID;
  }
  float* g[EU_SHALLOW_MAX_SLOTS + 1];   // the ABI's order (id, slots) to the backward's (slots, id)
  for (int t = 0; t < NT; ++t) g[t] = grads[t == T.S ? 0 : t + 1];
  return emb_backward(c, T, p->nodes, p->M, grad_out, d.W, gr, g, nullptr, nullptr, who);
}

// eu_shallow_encode_backward_sparse and its pooled form (gr)
static int shallow_backward_sparse(eu_ctx* c, const eu_shallow_problem* p, const ShallowDev& d, const EmbTables& T, GradRows gr,
                                   const float* grad_out, int64_t* const* rows, float* const* values, int64_t* counts, const char* who) {
  const int NT = T.S + (T.has_id ? 1 : 0);
  bool ok = rows && values && counts && (p->M == 0 || d.W == 0 || grad_out);
  for (int t = 0; ok && t < NT && p->M > 0; ++t) ok = rows[t == T.S ? 0 : t + 1] && values[t == T.S ? 0 : t + 1];
  if (!ok) {
    set_error("%s: bad argument (grad_out and rows, values and counts per table are required)", who);
    return EU_ERR_INVALID;
  }
  float* v[EU_SHALLOW_MAX_SLOTS + 1];
  int64_t* r[EU_SHALLOW_MAX_SLOTS + 1];
  int64_t n[EU_SHALLOW_MAX_SLOTS + 1] = {};
  for (int t = 0; t < NT; ++t) {
    v[t] = values[t == T.S ? 0 : t + 1];
    r[t] = rows[t == T.S ? 0 : t + 1];
  }
  int rc = emb_backward(c, T, p->nodes, p->M, grad_out, d.W, gr, v, r, n, who);
  if (rc) return rc;
  for (int t = 0; t < NT; ++t) counts[t == T.S ? 0 : t + 1] = n[t];
  if (!T.has_id) counts[0] = 0;
  return EU_OK;
}

// eu_sparse_embedding_lookup(_dtype)
static int emb_lookup(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int64_t default_value, const void* table, int64_t n_rows,
                      int32_t dim, int32_t combiner, int32_t table_dtype, float* out, const char* who) {
  int rc = dtype_check(table_dtype, who, "table");
  if (rc || (rc = emb_check(c, nodes, M, fid, default_value, table != nullptr, n_rows, dim, combiner, out, who))) return rc;
  EU_CUDA(cudaSetDevice(c->g->device));
  if (M == 0) return EU_OK;
  const bool vec = dim % 4 == 0 && aligned4_elems(table, table_dtype) && aligned16(out);
  const int G = group_lanes(ceil_div(dim, vec ? 4 : 1));
  const unsigned blocks = (unsigned)ceil_div(M * G, 256);
  const auto* nd = (const unsigned long long*)nodes;
  const auto dflt = (unsigned long long)default_value;
  EuProfScope ps(c, "emb_fwd", M);
  with_dtype(table_dtype, [&](auto e) {
    using E = typename decltype(e)::type;
    auto k = vec ? k_emb_fwd<true, E> : k_emb_fwd<false, E>;
    k<<<blocks, 256, 0, c->stream>>>(c->g->d, nd, M, fid, dflt, static_cast<const E*>(table), dim, G, combiner, out);
  });
  EU_LAUNCHED();
  return EU_OK;
}

// eu_shallow_encode(_dtype)
static int shallow_encode(eu_ctx* c, const eu_shallow_problem* p, int32_t table_dtype, float* out, float* dense_out, const char* who) {
  ShallowDev d;
  EmbTables T;
  int rc = dtype_check(table_dtype, who, "table");
  if (rc || (rc = shallow_resolve(c, p, &d, &T, who))) return rc;
  if (p->M > 0 && ((d.W > 0 && !out) || (d.add && d.dense_w > 0 && !dense_out))) {
    set_error("%s: bad argument (out%s is required)", who, d.add ? " and dense_out" : "");
    return EU_ERR_INVALID;
  }
  EU_CUDA(cudaSetDevice(c->g->device));
  if (p->M == 0 || (d.W == 0 && d.dense_w == 0)) return EU_OK;
  if ((rc = shallow_id_check(c, p, who))) return rc;
  d.out = out;
  d.dense_out = dense_out;
  const int G = shallow_lanes(&d, out, table_dtype);
  EuProfScope ps(c, "shallow_fwd", p->M);
  const unsigned blocks = (unsigned)ceil_div(p->M * G, 256);
  with_feat(c->g->d, [&](auto t, auto p) {
    with_dtype(table_dtype, [&](auto e) {
      k_shallow_fwd<typename decltype(t)::type, typename decltype(e)::type, decltype(p)::value><<<blocks, 256, 0, c->stream>>>(c->g->d, d, G);
    });
  });
  EU_LAUNCHED();
  return EU_OK;
}

// eu_shallow_encode_pool(_dtype)
static int shallow_pool(eu_ctx* c, const eu_shallow_problem* p, int32_t table_dtype, int32_t count, int32_t pool, float* out,
                        const char* who) {
  ShallowDev d;
  EmbTables T;
  GradRows gr;
  int rc = dtype_check(table_dtype, who, "table");
  if (rc || (rc = shallow_resolve(c, p, &d, &T, who)) || (rc = pool_check(p, count, pool, &gr, who))) return rc;
  if (p->M > 0 && d.W > 0 && !out) {
    set_error("%s: bad argument (out is required)", who);
    return EU_ERR_INVALID;
  }
  EU_CUDA(cudaSetDevice(c->g->device));
  if (p->M == 0 || d.W == 0) return EU_OK;
  if ((rc = shallow_id_check(c, p, who))) return rc;
  d.out = out;
  // the group's graph rows live in shared memory: wider groups until a block's fit in the default 48 KB
  int G = shallow_lanes(&d, out, table_dtype);
  while ((256 / G) * (size_t)count * sizeof(int64_t) > 48 * 1024) G *= 2;
  const int64_t R = p->M / count;
  EuProfScope ps(c, "shallow_pool", p->M);
  const unsigned blocks = (unsigned)ceil_div(R * G, 256);
  const size_t smem = (256 / G) * (size_t)count * sizeof(int64_t);
  with_feat(c->g->d, [&](auto t, auto p) {
    with_dtype(table_dtype, [&](auto e) {
      k_shallow_pool<typename decltype(t)::type, typename decltype(e)::type, decltype(p)::value><<<blocks, 256, smem, c->stream>>>(
          c->g->d, d, count, gr.pool_den, G);
    });
  });
  EU_LAUNCHED();
  return EU_OK;
}

}  // namespace eu

using namespace eu;

extern "C" {

int eu_sparse_embedding_lookup(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int64_t default_value, const float* table,
                               int64_t n_rows, int32_t dim, int32_t combiner, float* out) {
  return emb_lookup(c, nodes, M, fid, default_value, table, n_rows, dim, combiner, EU_FEAT_F32, out, "eu_sparse_embedding_lookup");
}

int eu_sparse_embedding_lookup_dtype(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int64_t default_value, const void* table,
                                     int64_t n_rows, int32_t dim, int32_t combiner, int32_t table_dtype, float* out) {
  return emb_lookup(c, nodes, M, fid, default_value, table, n_rows, dim, combiner, table_dtype, out, "eu_sparse_embedding_lookup_dtype");
}

int eu_sparse_embedding_lookup_backward(eu_ctx* c, const float* grad_out, const int64_t* nodes, int64_t M, int32_t fid,
                                        int64_t default_value, int64_t n_rows, int32_t dim, int32_t combiner, float* grad_table) {
  const char* who = "eu_sparse_embedding_lookup_backward";
  int rc = emb_check(c, nodes, M, fid, default_value, grad_table != nullptr, n_rows, dim, combiner, grad_out, who);
  if (rc) return rc;
  return single_backward(c, grad_out, nodes, M, fid, default_value, n_rows, dim, combiner, grad_table, nullptr, nullptr, who);
}

int eu_sparse_embedding_lookup_backward_sparse(eu_ctx* c, const float* grad_out, const int64_t* nodes, int64_t M, int32_t fid,
                                               int64_t default_value, int64_t n_rows, int32_t dim, int32_t combiner, int64_t* rows,
                                               float* values, int64_t* n) {
  const char* who = "eu_sparse_embedding_lookup_backward_sparse";
  int rc = emb_check(c, nodes, M, fid, default_value, n && (M == 0 || (rows && values)), n_rows, dim, combiner, grad_out, who);
  if (rc) return rc;
  return single_backward(c, grad_out, nodes, M, fid, default_value, n_rows, dim, combiner, values, rows, n, who);
}

int eu_shallow_encode(eu_ctx* c, const eu_shallow_problem* p, float* out, float* dense_out) {
  return shallow_encode(c, p, EU_FEAT_F32, out, dense_out, "eu_shallow_encode");
}

int eu_shallow_encode_dtype(eu_ctx* c, const eu_shallow_problem* p, int32_t table_dtype, float* out, float* dense_out) {
  return shallow_encode(c, p, table_dtype, out, dense_out, "eu_shallow_encode_dtype");
}

int eu_shallow_encode_backward(eu_ctx* c, const eu_shallow_problem* p, const float* grad_out, float* const* grads) {
  const char* who = "eu_shallow_encode_backward";
  ShallowDev d;
  EmbTables T;
  int rc = shallow_resolve(c, p, &d, &T, who);
  if (rc) return rc;
  return shallow_backward(c, p, d, T, GradRows(), grad_out, grads, who);
}

int eu_shallow_encode_backward_sparse(eu_ctx* c, const eu_shallow_problem* p, const float* grad_out, int64_t* const* rows,
                                      float* const* values, int64_t* counts) {
  const char* who = "eu_shallow_encode_backward_sparse";
  ShallowDev d;
  EmbTables T;
  int rc = shallow_resolve(c, p, &d, &T, who);
  if (rc) return rc;
  return shallow_backward_sparse(c, p, d, T, GradRows(), grad_out, rows, values, counts, who);
}

int eu_shallow_encode_pool(eu_ctx* c, const eu_shallow_problem* p, int32_t count, int32_t pool, float* out) {
  return shallow_pool(c, p, EU_FEAT_F32, count, pool, out, "eu_shallow_encode_pool");
}

int eu_shallow_encode_pool_dtype(eu_ctx* c, const eu_shallow_problem* p, int32_t table_dtype, int32_t count, int32_t pool, float* out) {
  return shallow_pool(c, p, table_dtype, count, pool, out, "eu_shallow_encode_pool_dtype");
}

int eu_shallow_encode_pool_backward(eu_ctx* c, const eu_shallow_problem* p, int32_t count, int32_t pool, const float* grad_out,
                                    float* const* grads) {
  const char* who = "eu_shallow_encode_pool_backward";
  ShallowDev d;
  EmbTables T;
  GradRows gr;
  int rc = shallow_resolve(c, p, &d, &T, who);
  if (rc || (rc = pool_check(p, count, pool, &gr, who))) return rc;
  return shallow_backward(c, p, d, T, gr, grad_out, grads, who);
}

int eu_shallow_encode_pool_backward_sparse(eu_ctx* c, const eu_shallow_problem* p, int32_t count, int32_t pool, const float* grad_out,
                                           int64_t* const* rows, float* const* values, int64_t* counts) {
  const char* who = "eu_shallow_encode_pool_backward_sparse";
  ShallowDev d;
  EmbTables T;
  GradRows gr;
  int rc = shallow_resolve(c, p, &d, &T, who);
  if (rc || (rc = pool_check(p, count, pool, &gr, who))) return rc;
  return shallow_backward_sparse(c, p, d, T, gr, grad_out, rows, values, counts, who);
}

}  // extern "C"
