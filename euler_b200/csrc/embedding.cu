// SparseEmbedding's lookup from node ids, forward and backward: the uint64 ("sparse") slot of each node, turned into one
// f32 row by an embedding table, with no host round trip and no intermediate COO.
//
// Reference semantics (file:line in the upstream alibaba/euler tree):
//   SparseEmbedding.call      tf_euler/python/utils/layers.py:152-169  tf.nn.embedding_lookup_sparse(table, sp_ids, None,
//                                                                       combiner), default combiner 'sum'
//   its input                 tf_euler/kernels/get_sparse_feature_op.cc:52-130  the node's values of the slot in stored
//                             order; a node without values (absent id, empty or unknown slot) gets one entry, the default
//   callers                   tf_euler/python/utils/encoders.py:151-160 (ShallowEncoder), :590-612 (SageEncoderNew)
//
// Forward, for node i with bag v_0 .. v_{n-1} (n >= 1):
//   acc = table[v_0]; acc = __fadd_rn(acc, table[v_k]) for k = 1 .. n-1   (from the first row, not from +0)
//   out_i = acc (sum), __fdiv_rn(acc, fl(n)) (mean), __fdiv_rn(acc, __fsqrt_rn(fl(n))) (sqrtn)
// A group of G lanes per node: the bag's values are loaded G at a time, one per lane, and broadcast by shuffle; kEmbUnroll
// table rows are loaded ahead of the ordered adds.  float4 loads when dim % 4 == 0 and table / out are 16-byte aligned,
// scalar otherwise: the same adds in the same order, so the bits do not depend on the alignment.  No scratch, no
// synchronisation: the forward is capturable in a CUDA graph.
//
// Backward, grad_table[v] = sum over the entries (i, k) with v_k = v of s_i(g_i), where s_i is the identity (sum),
// __fdiv_rn(., fl(n_i)) (mean) or __fdiv_rn(., __fsqrt_rn(fl(n_i))) (sqrtn), elementwise.  The entries are listed again from
// the graph, ordered stably by value (order_by) and summed per distinct value in fixed chunks of kSegChunk entries
// (plan_distinct, segment.cuh): deterministic, no atomics, and a hot value (the default fills every empty slot) is spread
// over many CTAs.  Rows no entry touches are zero.
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
  static __device__ __forceinline__ T load(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
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
  static __device__ __forceinline__ T load(const float* p) { return __ldg(p); }
  static __device__ __forceinline__ void store(float* p, T v) { *p = v; }
  static __device__ __forceinline__ T add(T a, T b) { return __fadd_rn(a, b); }
  static __device__ __forceinline__ T div(T a, float den) { return __fdiv_rn(a, den); }
};

// G lanes per node r, W columns per lane and step; blocks of G * W columns with a group-uniform trip count, so every lane of
// the group takes part in the shuffles.  The sum starts from the bag's first row (its bits, -0.0 and NaN payloads included).
template <bool VEC>
__global__ void __launch_bounds__(256, 1) k_emb_fwd(DevGraph g, const unsigned long long* __restrict__ nodes, int64_t M, int32_t fid,
                                                 unsigned long long dflt, const float* __restrict__ table, int dim, int G, int comb,
                                                 float* __restrict__ out) {
  using V = EmbVec<VEC>;
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t r = tid >> (31 - __clz(G));
  const int sub = (int)(tid & (G - 1));
  if (r >= M) return;   // group-uniform
  const unsigned gm = group_mask(G);
  int64_t b, e;
  ragged_slice(g.u64_ptr, g.n_u64_slots, lookup_row(g, __ldg(nodes + r)), fid, &b, &e);
  const bool empty = e == b;
  const int64_t n = empty ? 1 : e - b;
  const float den = emb_den(n, comb);
  for (int d0 = 0; d0 < dim; d0 += G * V::W) {
    const int d = d0 + sub * V::W;
    const bool act = d < dim;
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
    if (act) V::store(out + r * (int64_t)dim + d, acc);
  }
  if (comb == EU_COMBINE_SUM) return;
  // mean / sqrtn: one division per column, in a pass of its own over the row this group just wrote (L1-resident), so that
  // nothing of the bag loop is live across the division's slow-path subroutine
  __syncwarp(gm);
  float* o = out + r * (int64_t)dim;
  for (int d = sub; d < dim; d += G) o[d] = __fdiv_rn(o[d], den);
}

// One warp per node i: the value (as the sort key) and the node of each of its entries, at [ptr[i], ptr[i + 1])
__global__ void __launch_bounds__(256) k_emb_entries(DevGraph g, const unsigned long long* __restrict__ nodes, int64_t M, int32_t fid,
                                                     int32_t dflt, const int64_t* __restrict__ ptr, int32_t* __restrict__ key,
                                                     int32_t* __restrict__ node) {
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; i < M; i += nwarps) {
    int64_t b, e;
    ragged_slice(g.u64_ptr, g.n_u64_slots, lookup_row(g, __ldg(nodes + i)), fid, &b, &e);
    const int64_t o = __ldg(ptr + i);
    if (e == b) {
      if (lane == 0) { key[o] = dflt; node[o] = (int32_t)i; }
      continue;
    }
    for (int64_t k = lane; k < e - b; k += 32) {
      key[o + k] = (int32_t)__ldg(g.u64_val + b + k);
      node[o + k] = (int32_t)i;
    }
  }
}

// gs[i, d] = g[i, d] / den(n_i) (one __fdiv_rn), n_i = ptr[i + 1] - ptr[i]: the scaled gradient of the mean and sqrtn
// combiners, once per node and column rather than once per entry
__global__ void k_emb_scale_grad(const float* __restrict__ g, const int64_t* __restrict__ ptr, int64_t M, int dim, int comb,
                                 float* __restrict__ gs) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < M * dim; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / dim;
    gs[t] = __fdiv_rn(__ldg(g + t), emb_den(__ldg(ptr + i + 1) - __ldg(ptr + i), comb));
  }
}

// G lanes per chunk c of the distinct-value segments (grid-stride over the chunks, whose number is on the device).  Chunk
// c - chunk_off[p] of segment p covers the sorted positions [start[p] + (c - chunk_off[p]) * kSegChunk, ...), up to kSegChunk
// of them: the sum, left to right from +0, of the (scaled) gradient rows gs of their nodes.  A segment of one chunk writes
// its table row; the chunks of a longer one write their partial rows for k_emb_bwd_combine.
template <bool VEC>
__global__ void __launch_bounds__(256, 1) k_emb_bwd_chunks(const float* __restrict__ gs, const int32_t* __restrict__ node,
                                                        const int32_t* __restrict__ perm, DistinctPlan P, int dim, int G,
                                                        float* __restrict__ grad_table) {
  using V = EmbVec<VEC>;
  const int lg = 31 - __clz(G);
  const int sub = (int)(threadIdx.x & (G - 1));
  const int64_t nch_all = __ldg(P.chunk_off + P.E);
  const int64_t step = ((int64_t)gridDim.x * blockDim.x) >> lg;
  for (int64_t c = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> lg; c < nch_all; c += step) {
    const int64_t p = key_upper_bound(P.chunk_off, P.E + 1, c) - 1;
    const int64_t c0 = __ldg(P.chunk_off + p), nch = __ldg(P.chunk_off + p + 1) - c0;
    const int64_t b = __ldg(P.start + p) + (c - c0) * kSegChunk;
    const int64_t e = min(b + kSegChunk, (int64_t)__ldg(P.start + p + 1));
    float* o = nch == 1 ? grad_table + (int64_t)__ldg(P.key + p) * dim : P.partial + (int64_t)(__ldg(P.part_off + p) + (c - c0)) * dim;
    for (int d = sub * V::W; d < dim; d += G * V::W) {
      typename V::T acc = V::zero(0.f);
      for (int64_t k0 = b; k0 < e; k0 += kEmbUnroll) {
        typename V::T x[kEmbUnroll];
#pragma unroll
        for (int q = 0; q < kEmbUnroll; ++q)
          if (k0 + q < e) x[q] = V::load(gs + (int64_t)__ldg(node + __ldg(perm + k0 + q)) * dim + d);
#pragma unroll
        for (int q = 0; q < kEmbUnroll; ++q)
          if (k0 + q < e) acc = V::add(acc, x[q]);
      }
      V::store(o + d, acc);
    }
  }
}

// grad_table[key[p], f] = the partial rows of segment p added in chunk order from +0, for the segments of several chunks
__global__ void k_emb_bwd_combine(DistinctPlan P, int dim, float* __restrict__ grad_table) {
  const int64_t n = (int64_t)__ldg(P.nd) * dim;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = t / dim, f = t - p * dim;
    const int64_t nch = __ldg(P.chunk_off + p + 1) - __ldg(P.chunk_off + p);
    if (nch == 1) continue;
    const float* part = P.partial + (int64_t)__ldg(P.part_off + p) * dim + f;
    float acc = 0.f;
    for (int64_t j = 0; j < nch; ++j) acc = __fadd_rn(acc, __ldg(part + j * dim));
    grad_table[(int64_t)__ldg(P.key + p) * dim + f] = acc;
  }
}

// The checks both passes share.  Every value of slot fid and the default must index the table: the slot's largest value is
// kept on the graph, so this costs no device work.
static int emb_check(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int64_t default_value, const float* table, int64_t n_rows,
                     int32_t dim, int32_t combiner, const void* out, const char* who) {
  if (!c || M < 0 || n_rows < 1 || dim < 1 || combiner < EU_COMBINE_SUM || combiner > EU_COMBINE_SQRTN || (M > 0 && (!nodes || !out)) ||
      !table) {
    set_error("%s: bad argument", who);
    return EU_ERR_INVALID;
  }
  if (M >= ((int64_t)1 << 31) || n_rows >= ((int64_t)1 << 31)) {
    set_error("%s: 2^31 or more nodes or table rows are not supported", who);
    return EU_ERR_UNSUPPORTED;
  }
  const eu_graph* g = c->g;
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

}  // namespace eu

using namespace eu;

extern "C" {

int eu_sparse_embedding_lookup(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int64_t default_value, const float* table,
                               int64_t n_rows, int32_t dim, int32_t combiner, float* out) {
  const char* who = "eu_sparse_embedding_lookup";
  int rc = emb_check(c, nodes, M, fid, default_value, table, n_rows, dim, combiner, out, who);
  if (rc) return rc;
  EU_CUDA(cudaSetDevice(c->g->device));
  if (M == 0) return EU_OK;
  const bool vec = dim % 4 == 0 && aligned16(table) && aligned16(out);
  const int G = group_lanes(ceil_div(dim, vec ? 4 : 1));
  const unsigned blocks = (unsigned)ceil_div(M * G, 256);
  EuProfScope ps(c, "emb_fwd", M);
  if (vec) k_emb_fwd<true><<<blocks, 256, 0, c->stream>>>(c->g->d, (const unsigned long long*)nodes, M, fid, (unsigned long long)default_value,
                                                          table, dim, G, combiner, out);
  else k_emb_fwd<false><<<blocks, 256, 0, c->stream>>>(c->g->d, (const unsigned long long*)nodes, M, fid, (unsigned long long)default_value,
                                                       table, dim, G, combiner, out);
  EU_LAUNCHED();
  return EU_OK;
}

int eu_sparse_embedding_lookup_backward(eu_ctx* c, const float* grad_out, const int64_t* nodes, int64_t M, int32_t fid,
                                        int64_t default_value, int64_t n_rows, int32_t dim, int32_t combiner, float* grad_table) {
  const char* who = "eu_sparse_embedding_lookup_backward";
  int rc = emb_check(c, nodes, M, fid, default_value, grad_table, n_rows, dim, combiner, grad_out, who);
  if (rc) return rc;
  EU_CUDA(cudaSetDevice(c->g->device));
  cudaStream_t s = c->stream;
  EU_CUDA(cudaMemsetAsync(grad_table, 0, 4 * (size_t)n_rows * dim, s));
  if (M == 0) return EU_OK;
  // ptr [M + 1] | scan temp | then, once the entry count E is known: key [E] | node [E] | the order by value | the plan
  const size_t o_tmp = a256(8 * (size_t)(M + 1)), tmp = ragged_scan_bytes(M), o_key = o_tmp + a256(tmp);
  if ((rc = ctx_misc(c, (int64_t)o_key))) return rc;
  if ((rc = sparse_entry_ptr(c, nodes, M, fid, (char*)c->d_misc + o_tmp, tmp, (int64_t*)c->d_misc))) return rc;
  int64_t E = 0;
  EU_CUDA(cudaMemcpyAsync(&E, (int64_t*)c->d_misc + M, sizeof(E), cudaMemcpyDeviceToHost, s));
  EU_CUDA(cudaStreamSynchronize(s));
  if (E + E / kSegChunk + 1 >= ((int64_t)1 << 31)) {
    set_error("%s: 2^31 or more entries are not supported", who);
    return EU_ERR_UNSUPPORTED;
  }
  const size_t o_node = o_key + a256(4 * (size_t)E), o_ord = o_node + a256(4 * (size_t)E), o_plan = o_ord + order_bytes(E, n_rows);
  const size_t o_gs = o_plan + distinct_plan_bytes(E, dim);
  const size_t total = o_gs + (combiner == EU_COMBINE_SUM ? 0 : a256(4 * (size_t)M * dim));
  if ((int64_t)total > c->misc_bytes) {   // the growth reallocates: the offsets again (no read-back needed)
    if ((rc = ctx_misc(c, (int64_t)total))) return rc;
    if ((rc = sparse_entry_ptr(c, nodes, M, fid, (char*)c->d_misc + o_tmp, tmp, (int64_t*)c->d_misc))) return rc;
  }
  char* m = (char*)c->d_misc;
  const int64_t* ptr = (const int64_t*)m;
  int32_t* key = (int32_t*)(m + o_key);
  int32_t* node = (int32_t*)(m + o_node);
  EdgeOrder ord;
  DistinctPlan P;
  {
    EuProfScope ps(c, "emb_bwd_order", E);
    k_emb_entries<<<stride_grid(M * 32), 256, 0, s>>>(c->g->d, (const unsigned long long*)nodes, M, fid, (int32_t)default_value, ptr, key,
                                                      node);
    EU_LAUNCHED();
    if ((rc = order_by(c, key, E, n_rows, m + o_ord, &ord))) return rc;
    if ((rc = plan_distinct(c, ord, E, m + o_plan, &P))) return rc;
  }
  EuProfScope ps(c, "emb_bwd_sums", E);
  const float* gs = grad_out;
  if (combiner != EU_COMBINE_SUM) {
    float* scaled = (float*)(m + o_gs);
    k_emb_scale_grad<<<stride_grid(M * dim), 256, 0, s>>>(grad_out, ptr, M, dim, combiner, scaled);
    EU_LAUNCHED();
    gs = scaled;
  }
  const bool vec = dim % 4 == 0 && aligned16(gs) && aligned16(grad_table);
  const int G = group_lanes(ceil_div(dim, vec ? 4 : 1));
  const unsigned blocks = stride_grid((E + E / kSegChunk + 1) * G);   // >= one group per chunk, up to the grid cap
  if (vec) k_emb_bwd_chunks<true><<<blocks, 256, 0, s>>>(gs, node, ord.perm, P, dim, G, grad_table);
  else k_emb_bwd_chunks<false><<<blocks, 256, 0, s>>>(gs, node, ord.perm, P, dim, G, grad_table);
  EU_LAUNCHED();
  k_emb_bwd_combine<<<stride_grid(E * dim), 256, 0, s>>>(P, dim, grad_table);
  EU_LAUNCHED();
  return EU_OK;
}

}  // extern "C"
