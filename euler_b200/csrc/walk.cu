// random_walk: uniform (p=q=1) and node2vec-biased walks, walkers resident on the device for all L steps.
//
// Reference (file:line relative to /root/reference):
//   RandomWalk::ComputeAsync          tf_euler/kernels/random_walk_op.cc:249-289
//   TraditionalRandomWalk (p=q=1)     :207-247  = L chained sampleNB(count=1) hops, id 0 -> default_node
//   RWCallback::operator() (node2vec) :83-138   per step: full neighbor list of the current node
//                                               (Node::__GetFullNeighbor, euler/core/graph/node.cc:176-198),
//   BuildWeights                      :140-168  two-pointer merge against the parent's list,
//   CompactWeightedCollection::Init/Sample      euler/common/compact_weighted_collection.h:82-128
//                                               sequential f32 prefix + one RandomSelect draw.
// The reference makes one host round trip (a GQL query) per step; here a step is two small kernels
// and the frontier never leaves HBM.  Exact-RNG order: one uniform per LIVE walker, in walker order.
#include <stdlib.h>

#include "internal.h"

namespace eu {

struct ETypes2 {
  int32_t K;
  int32_t v[EU_MAX_ETYPES];
};

// Sequential view of Node::GetFullNeighbor(edge_types): listed types in listed order (invalid ones
// skipped, duplicates repeated), stored order within a group; weight = cum[j] - cum[j-1] (0 at row start).
struct NbIter {
  const DevGraph* g;
  const int64_t* gp;  // grp_ptr + row*T
  int64_t base;
  const ETypes2* et;
  int32_t k;          // position in et
  int64_t j, jend;
  __device__ void init(const DevGraph* g_, int64_t row, const ETypes2* et_) {
    g = g_; et = et_; k = -1; j = 0; jend = 0;
    if (row < 0) { gp = nullptr; k = et_->K; return; }
    gp = g->grp_ptr + row * g->T;
    base = gp[0];
    advance_group();
  }
  __device__ void advance_group() {
    while (j >= jend) {
      ++k;
      if (k >= et->K) return;
      int32_t t = et->v[k];
      if (t < 0 || t >= g->T) continue;
      j = gp[t];
      jend = gp[t + 1];
    }
  }
  __device__ bool done() const { return k >= et->K; }
  __device__ long long id() const { return (long long)__ldg(g->nbr + j); }
  __device__ float w() const {
    float hi = __ldg(g->cum_w + j);
    float lo = j == base ? 0.f : __ldg(g->cum_w + j - 1);
    return __fsub_rn(hi, lo);
  }
  __device__ void next() { ++j; if (j >= jend) advance_group(); }
};

__device__ __forceinline__ int64_t list_len(const DevGraph& g, int64_t row, const ETypes2& et) {
  if (row < 0) return 0;
  int64_t n = 0;
  for (int32_t k = 0; k < et.K; ++k) {
    int32_t t = et.v[k];
    if (t >= 0 && t < g.T) n += g.grp_ptr[row * g.T + t + 1] - g.grp_ptr[row * g.T + t];
  }
  return n;
}

struct WalkState {
  long long* cur;       // [B] current node id
  long long* parent;    // [B] parent id
  int64_t* cur_row;     // [B] row of cur (-1 absent)
  int64_t* parent_row;  // [B] row whose list is the parent list (-1 = empty list)
};

__global__ void k_walk_init(const long long* __restrict__ nodes, int64_t B, int32_t L, WalkState s,
                            long long* __restrict__ out) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= B) return;
  long long id = nodes[i];
  out[i * (L + 1)] = id;
  s.cur[i] = id;
  s.parent[i] = id;       // step 0: parent = the start node itself, empty parent list (:272-287)
  s.parent_row[i] = -1;
}

// liveness: the walker draws this step iff its current node has a non-empty neighbor list
__global__ void k_walk_live(DevGraph g, int64_t B, ETypes2 et, WalkState s, uint8_t* live) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= B) return;
  int64_t row = lookup_row(g, (unsigned long long)s.cur[i]);
  s.cur_row[i] = row;
  live[i] = list_len(g, row, et) > 0 ? 1 : 0;
}

// One thread walks the merge (BuildWeights :140-168) and the running f32 prefix
// (CompactWeightedCollection::Init :82-97).  Returns the total; if pick >= 0.0 also returns in *sel
// the first position whose prefix exceeds `pick` (RandomSelect closed form), else the last position.
__device__ float biased_prefix(const DevGraph& g, int64_t crow, const ETypes2& cet, int64_t prow,
                               const ETypes2& pet, long long parent_id, float p, float q, bool select,
                               double pick, long long* sel_id) {
  NbIter c, pn;
  c.init(&g, crow, &cet);
  pn.init(&g, prow, &pet);
  float sum = 0.f;
  long long last_id = 0;
  bool found = false;
  long long pk = pn.done() ? 0 : pn.id();
  while (!c.done()) {
    const long long cid = c.id();
    float w = c.w();
    // advance the parent pointer past smaller ids ("else ++k")
    while (!pn.done() && cid > pk) { pn.next(); if (!pn.done()) pk = pn.id(); }
    if (!pn.done() && cid == pk) {
      pn.next(); if (!pn.done()) pk = pn.id();          // shared neighbor: d_tx = 1, weight unchanged
    } else {
      w = cid != parent_id ? __fdiv_rn(w, q) : __fdiv_rn(w, p);  // d_tx = 2 / d_tx = 0
    }
    sum = __fadd_rn(sum, w);
    last_id = cid;
    if (select && !found && (double)sum > pick) { *sel_id = cid; found = true; if (select) break; }
    c.next();
  }
  if (select && !found) *sel_id = last_id;
  return sum;
}

// Note on the merge above: the reference loop is
//   while (j < nc && k < np) { if (c[j] < p[k]) {bias; ++j} else if (c[j] == p[k]) {++k; ++j} else ++k }
//   while (j < nc) {bias; ++j}
// For a fixed j the inner "else ++k" steps are exactly the `while (cid > pk)` loop, then one of the
// first two branches fires (or k ran out and the tail loop biases) -- same visit order, same state.

__global__ void __launch_bounds__(128) k_walk_step(DevGraph g, int64_t B, int32_t L, int32_t step, ETypes2 cet,
                                                   ETypes2 pet, float p, float q, long long default_node,
                                                   WalkState s, const uint8_t* __restrict__ live,
                                                   const uint32_t* __restrict__ state, bool philox,
                                                   unsigned long long key, long long* __restrict__ out) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= B) return;
  const long long cur = s.cur[i];
  const int64_t crow = s.cur_row[i];
  long long next = default_node;
  if (live[i]) {
    const int64_t prow = s.parent_row[i];
    const long long parent_id = s.parent[i];
    const float total = biased_prefix(g, crow, cet, prow, pet, parent_id, p, q, false, 0.0, nullptr);
    double u, u2;
    if (philox) {
      philox_uniform2((unsigned long long)i, (uint32_t)step, 0x77616C6Bu, key, u, u2);
    } else {
      uint32_t x = state[i];
      u = minstd_uniform(x);
    }
    const double r = pick_r(u, 0.f, total);
    biased_prefix(g, crow, cet, prow, pet, parent_id, p, q, true, r, &next);
  }
  out[i * (L + 1) + step + 1] = next;
  // parent_neighbors_ = this step's lists, parent_ids_ = this step's nodes (:128-131)
  s.parent[i] = cur;
  s.parent_row[i] = crow;
  s.cur[i] = next;
}

// ---------------------------------------------------------------------------------------------
// Warp-cooperative exact step for the common case: ONE edge type per step and adjacency groups sorted by
// neighbor id (DevGraph::adj_sorted; the reference's merge assumes sorted lists as well).  For sorted
// multisets C (children) and P (parent's list) the two-pointer merge of BuildWeights (:140-168) marks the
// m-th copy (m = 0,1,..) of value v in C as "shared" iff P holds more than m copies of v; everything else is
// biased (/p if it is the parent id, /q otherwise).  That is a per-element predicate, so 32 lanes classify 32
// children at once by streaming P in 32-wide chunks next to C; only the f32 prefix sum (CompactWeightedCollection
// ::Init, compact_weighted_collection.h:82-97) stays serial -- it is evaluated left to right through shuffles,
// ~5 cycles per neighbor.  Pass 1 = total, pass 2 = select.  Used for rows of up to kWalkBig edges (k_walk_prefix); longer
// rows go through k_walk_weights + block_exact_prefix, which evaluates the same sequential sum 1024 elements at a time.
struct WarpWalk {
  const DevGraph* g;
  int64_t cb, ce, cbase;   // child group [cb, ce), first edge of the child's row
  int64_t pb, pe;          // parent group [pb, pe) (empty at step 0 / for dead parents)
  long long parent_id;
  float p, q;
  int lane;

  __device__ float pass(bool select, double pick, long long* sel) const {
    const unsigned FULL = 0xffffffffu;
    const long long BIG = 0x7fffffffffffffffLL;
    float run = 0.f;                // running prefix, replicated in every lane
    int64_t pk = pb;                // first parent chunk that can still hold values >= the current child minimum
    long long prev_val = 0;
    int prev_run = 0;               // copies of prev_val seen so far at the end of the previous child chunk
    long long last_id = 0;
    for (int64_t cj = cb; cj < ce; cj += 32) {
      const int nvalid = (int)min((int64_t)32, ce - cj);
      const int64_t j = cj + lane;
      const bool valid = lane < nvalid;
      const long long cv = valid ? (long long)__ldg(g->nbr + j) : BIG;
      float w = 0.f;
      if (valid) {
        const float hi = __ldg(g->cum_w + j);
        const float lo = j == cbase ? 0.f : __ldg(g->cum_w + j - 1);
        w = __fsub_rn(hi, lo);
      }
      // m = copies of cv that precede this one in C
      const unsigned peers = __match_any_sync(FULL, cv);
      int m = __popc(peers & ((1u << lane) - 1u));
      if (prev_run && cv == prev_val) m += prev_run;
      // cnt = copies of cv in P: walk the parent chunks whose value range meets [vmin, vmax]
      const long long vmin = __shfl_sync(FULL, cv, 0), vmax = __shfl_sync(FULL, cv, nvalid - 1);
      int cnt = 0;
      for (int64_t tk = pk; tk < pe; tk += 32) {
        const int np = (int)min((int64_t)32, pe - tk);  // parent lanes holding a list entry; the others are padding
        const long long pv = lane < np ? (long long)__ldg(g->nbr + tk + lane) : BIG;
        const long long pmin = __shfl_sync(FULL, pv, 0);
        const long long pmax = __shfl_sync(FULL, pv, np - 1);
        if (pmax < vmin) { pk = tk + 32; continue; }   // below every remaining child value: never needed again
        if (pmin > vmax) break;                         // above this child chunk: the next chunk restarts at pk
        // count valid lanes only: a child id equal to the padding value (2^63-1) must not match the padding
#pragma unroll 8
        for (int k = 0; k < 32; ++k) cnt += (__shfl_sync(FULL, pv, k) == cv && k < np) ? 1 : 0;
        if (pmax > vmax) break;
      }
      const bool shared = m < cnt;
      if (valid && !shared) w = cv != parent_id ? __fdiv_rn(w, q) : __fdiv_rn(w, p);   // d_tx = 2 / d_tx = 0
      // serial f32 prefix over the chunk, left to right
      float mine = 0.f;
      for (int k = 0; k < nvalid; ++k) {
        run = __fadd_rn(run, __shfl_sync(FULL, w, k));
        if (lane == k) mine = run;
      }
      if (select) {
        const unsigned hit = __ballot_sync(FULL, valid && (double)mine > pick);
        if (hit) { *sel = __shfl_sync(FULL, cv, __ffs(hit) - 1); return run; }
      }
      last_id = __shfl_sync(FULL, cv, nvalid - 1);
      prev_val = last_id;
      prev_run = __shfl_sync(FULL, m, nvalid - 1) + 1;
    }
    if (select) *sel = last_id;   // RandomSelect's fall-through: the last entry
    return run;
  }
};

// ---------------------------------------------------------------------------------------------
// Exact node2vec step for BIG rows (deg > kWalkBig), split so that nothing latency-heavy sits inside the sequential part:
//   k_walk_plan     one block: RNG engine states of the live walkers (the reference draws one uniform per live walker, in
//                   walker order), the work lists, offsets of every live walker's row in the weight scratch V
//   k_walk_weights  fully parallel over (walker, neighbor): BuildWeights' bias (:140-168) per element -- membership of the
//                   child in the parent's sorted list by binary search, multiset rule as in WarpWalk -- written to V.  No
//                   walker streams its parent's list (a small row behind a 137K-edge parent cost 4300 dependent loads)
//   k_walk_prefix   CTA per big walker (deg > kWalkBig): the SEQUENTIAL f32 prefix of CompactWeightedCollection::Init
//                   (:82-97) evaluated 1024 elements per iteration without changing a single rounding (block_exact_prefix
//                   below), total -> one uniform -> RandomSelect; warp per small walker: the same chain through shuffles
//
// block_exact_prefix: S_k = fl(S_{k-1} + v_k) for v_k >= 0.  While S stays in one binade (ulp u = 2^(e-23), S = M u with
// 2^23 <= M < 2^24) and v_k's exponent does not exceed e, fl(S + v) = (M + a + c) u with a = floor(v / u) and c = 1 iff the
// discarded part of v exceeds u / 2 -- an INTEGER increment that does not depend on M, except (i) exact ties (discarded
// part == u / 2: round-half-even needs M's parity), (ii) M reaching 2^24 (the binade changes) and (iii) v above S's binade.
// So the block computes the increments of 1024 elements in parallel, prefix-sums them as integers, accepts everything
// before the first exception, lets one thread redo the next kPrefSer elements with real FADDs, and continues.  Exceptions are
// common only while S is within a few binades of the addends (the first dozens of elements of a row); a 137K-edge hub row
// of the R-MAT graph takes 143 iterations instead of 137K dependent FADDs.  tests/test_walk_prefix_gpu.py compares it bit for
// bit with the oracle's sequential sum on tie-heavy, zero-laden, wide-exponent, subnormal and randomly rounding rows at
// every length where the step switches kernels (tests/walk_rows.py builds them and counts the events each one causes).
static constexpr int kWalkBig = 512;        // rows longer than this get a 256-thread CTA (shorter ones a warp)
static constexpr int kWalkHuge = 16384;     // rows longer than this get a 1024-thread CTA
static constexpr int kWalkChunk = 256;      // elements per k_walk_weights chunk
static constexpr int kPrefT = 256;          // threads of a k_walk_prefix CTA
static constexpr int kPrefE = 4;            // elements per thread and iteration
static constexpr int kPrefCH = kPrefT * kPrefE;
static constexpr int kPrefSer = 96;         // elements redone serially after an exception (4 cycles each: far cheaper than an iteration)
static constexpr int kPrefHead = 768;       // elements of a row summed serially before the first parallel iteration
static constexpr int kPrefCk = 256;         // checkpoints kept per row

struct WalkPlan {
  int32_t* deg;         // [B] length of the walker's child list (single type), 0 if dead
  int32_t* live_list;   // [B] live walkers whose row fits in V, walker order (k_walk_weights maps chunks to them)
  int32_t* coff;        // [B+1] first k_walk_weights chunk of live_list[k]
  long long* voff;      // [B] V offset of walker i's row (by walker id)
  int32_t* huge_list;   // [B] walkers with deg > kWalkHuge: one 1024-thread CTA each
  int32_t* big_list;    // [B] walkers with kWalkBig < deg <= kWalkHuge: one 256-thread CTA each
  int32_t* small_list;  // [B] the other walkers with a V row: one warp each
  int32_t* ovf_list;    // [B] live walkers whose row does not fit in V: the self-contained warp path (WarpWalk)
  unsigned int* ctr;    // [16]: 0 n_big, 1 n_small, 2 n_chunks, 3 big ticket, 4 small ticket, 5 n_ovf, 6 ovf ticket, 7 n_fit,
                        //       8 n_huge, 9 huge ticket
  float* V;
  long long capV;
};

__global__ void k_walk_deg(DevGraph g, int64_t B, int32_t ctype, WalkState s, uint8_t* live, int32_t* deg) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= B) return;
  const int64_t row = lookup_row(g, (unsigned long long)s.cur[i]);
  s.cur_row[i] = row;
  int64_t d = 0;
  if (row >= 0) d = g.grp_ptr[row * g.T + ctype + 1] - g.grp_ptr[row * g.T + ctype];
  live[i] = d > 0 ? 1 : 0;
  deg[i] = (int32_t)min(d, (int64_t)0x7fffffff);
}

// one block of 1024 threads; thread t owns a contiguous stretch of walkers
__global__ void __launch_bounds__(1024) k_walk_plan(int64_t B, const uint8_t* __restrict__ live, bool minstd, uint32_t F,
                                                    uint32_t* __restrict__ state, EuRngState* rng, WalkPlan wp) {
  __shared__ uint32_t s_prod[1024];
  __shared__ uint32_t s_cnt[1024];
  __shared__ uint32_t s_big[1024];
  __shared__ uint32_t s_huge[1024];
  __shared__ uint32_t s_chunks[1024];
  __shared__ unsigned long long s_el[1024];
  __shared__ unsigned int s_fit, s_fitbig, s_fithuge, s_fitchunks;
  const int t = threadIdx.x;
  if (t == 0) { wp.ctr[5] = 0; s_fit = 0; s_fitbig = 0; s_fithuge = 0; s_fitchunks = 0; }
  const int64_t per = (B + 1023) / 1024;
  const int64_t b = min((int64_t)t * per, B), e = min(b + per, B);
  uint32_t prod = 1, cnt = 0, nbig = 0, nhuge = 0, chunks = 0;
  unsigned long long el = 0;
  for (int64_t i = b; i < e; ++i) {
    if (!live[i]) continue;
    prod = modmul(prod, F); ++cnt;
    const int32_t d = wp.deg[i];
    el += (unsigned long long)d;
    chunks += (uint32_t)((d + kWalkChunk - 1) / kWalkChunk);
    if (d > kWalkHuge) ++nhuge; else if (d > kWalkBig) ++nbig;
  }
  s_prod[t] = prod; s_cnt[t] = cnt; s_big[t] = nbig; s_huge[t] = nhuge; s_chunks[t] = chunks; s_el[t] = el;
  __syncthreads();
  for (int off = 1; off < 1024; off <<= 1) {   // inclusive Hillis-Steele scans (modmul is associative and commutative)
    uint32_t v = 1, c = 0, g1 = 0, g2 = 0, g3 = 0; unsigned long long g4 = 0;
    if (t >= off) { v = s_prod[t - off]; c = s_cnt[t - off]; g1 = s_big[t - off]; g2 = s_huge[t - off]; g3 = s_chunks[t - off]; g4 = s_el[t - off]; }
    __syncthreads();
    if (t >= off) { s_prod[t] = modmul(s_prod[t], v); s_cnt[t] += c; s_big[t] += g1; s_huge[t] += g2; s_chunks[t] += g3; s_el[t] += g4; }
    __syncthreads();
  }
  const uint32_t x0 = minstd ? rng->x : 0u;
  uint32_t run = minstd ? modmul(x0, t > 0 ? s_prod[t - 1] : 1u) : 0u;
  uint32_t kl = t > 0 ? s_cnt[t - 1] : 0u, kb = t > 0 ? s_big[t - 1] : 0u, kh = t > 0 ? s_huge[t - 1] : 0u, kc = t > 0 ? s_chunks[t - 1] : 0u;
  unsigned long long ke = t > 0 ? s_el[t - 1] : 0ull;
  unsigned int fit = 0, fitbig = 0, fithuge = 0, fitchunks = 0;
  for (int64_t i = b; i < e; ++i) {
    if (minstd) state[i] = run;
    if (!live[i]) continue;
    if (minstd) run = modmul(run, F);
    const int32_t d = wp.deg[i];
    const uint32_t nch = (uint32_t)((d + kWalkChunk - 1) / kWalkChunk);
    if (ke + (unsigned long long)d <= (unsigned long long)wp.capV) {
      // V offsets are monotone in walker order, so the walkers that fit are a prefix of the live ones: their positions in
      // the live / big / small lists are the scanned counts
      wp.live_list[kl] = (int32_t)i; wp.coff[kl] = (int32_t)kc; wp.voff[i] = (long long)ke;
      if (d > kWalkHuge) { wp.huge_list[kh] = (int32_t)i; ++fithuge; }
      else if (d > kWalkBig) { wp.big_list[kb] = (int32_t)i; ++fitbig; }
      else wp.small_list[kl - kb - kh] = (int32_t)i;
      ++fit; fitchunks += nch;
    } else {
      wp.ovf_list[atomicAdd(&wp.ctr[5], 1u)] = (int32_t)i;   // V is full: the self-contained warp path serves it
    }
    ++kl; ke += (unsigned long long)d; kc += nch;
    if (d > kWalkHuge) ++kh; else if (d > kWalkBig) ++kb;
  }
  if (fit) { atomicAdd(&s_fit, fit); atomicAdd(&s_fitbig, fitbig); atomicAdd(&s_fithuge, fithuge); atomicAdd(&s_fitchunks, fitchunks); }
  __syncthreads();
  if (t == 1023 && minstd) { rng->x = modmul(x0, s_prod[1023]); rng->draws += (unsigned long long)s_cnt[1023]; }
  if (t == 0) {
    wp.ctr[0] = s_fitbig;
    wp.ctr[1] = s_fit - s_fitbig - s_fithuge;
    wp.ctr[2] = s_fitchunks;
    wp.ctr[3] = 0; wp.ctr[4] = 0; wp.ctr[6] = 0;
    wp.ctr[7] = s_fit;
    wp.ctr[8] = s_fithuge; wp.ctr[9] = 0;
    wp.coff[s_fit] = (int32_t)s_fitchunks;
  }
}

// first j in [lo, hi) with (signed) a[j] >= key
__device__ __forceinline__ int64_t lower_bound_ll(const unsigned long long* __restrict__ a, int64_t lo, int64_t hi, long long key) {
  while (lo < hi) {
    const int64_t mid = lo + ((hi - lo) >> 1);
    if ((long long)__ldg(a + mid) < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(kWalkChunk) k_walk_weights(DevGraph g, int32_t ctype, int32_t ptype, float p, float q, WalkState s,
                                                             WalkPlan wp) {
  __shared__ int s_k;
  const unsigned int n_chunks = wp.ctr[2], n_fit = wp.ctr[7];
  for (unsigned int c = blockIdx.x; c < n_chunks; c += gridDim.x) {
    if (threadIdx.x == 0) {   // walker of chunk c: last k with coff[k] <= c
      int lo = 0, hi = (int)n_fit;
      while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if ((unsigned int)wp.coff[mid] <= c) lo = mid; else hi = mid; }
      s_k = lo;
    }
    __syncthreads();
    const int k = s_k;
    const int64_t i = wp.live_list[k];
    const int64_t crow = s.cur_row[i];
    const int64_t cbase = g.grp_ptr[crow * g.T];
    const int64_t cb = g.grp_ptr[crow * g.T + ctype];
    const int64_t off = (int64_t)(c - (unsigned int)wp.coff[k]) * kWalkChunk + threadIdx.x;
    const int32_t d = wp.deg[i];
    if (off < d) {
      const int64_t j = cb + off;
      const long long cv = (long long)__ldg(g.nbr + j);
      const float hi_w = __ldg(g.cum_w + j);
      const float lo_w = j == cbase ? 0.f : __ldg(g.cum_w + j - 1);
      float w = __fsub_rn(hi_w, lo_w);
      // m = copies of cv that precede this one in the child list (sorted: they are adjacent)
      int64_t m = 0;
      while (j - 1 - m >= cb && (long long)__ldg(g.nbr + j - 1 - m) == cv) ++m;
      bool shared = false;
      const int64_t prow = s.parent_row[i];
      if (prow >= 0 && ptype >= 0 && ptype < g.T) {
        const int64_t pb = g.grp_ptr[prow * g.T + ptype], pe = g.grp_ptr[prow * g.T + ptype + 1];
        const int64_t lb = lower_bound_ll(g.nbr, pb, pe, cv);
        shared = lb + m < pe && (long long)__ldg(g.nbr + lb + m) == cv;   // the parent holds more than m copies
      }
      if (!shared) w = cv != s.parent[i] ? __fdiv_rn(w, q) : __fdiv_rn(w, p);   // d_tx = 2 / d_tx = 0
      wp.V[wp.voff[i] + off] = w;
    }
    __syncthreads();
  }
}

template <int T>
struct PrefShared {
  float v[T * kPrefE];
  unsigned int warp_tot[T / 32];
  float ck_S[kPrefCk];
  int32_t ck_pos[kPrefCk];
  int n_ck;
  float S;
  int32_t pos;
  int first, hit;
  unsigned int m_prev;
  double r;
  int32_t answer;
};

// Runs the exact prefix over V[0, n) from (sh.pos, sh.S).  select: stop at the first k with (double)S_k > r and leave k in
// sh.answer (-1 if none).  record: store a checkpoint every ck_stride iterations.  Returns with sh.S = S_{n-1} when !select.
template <int T>
__device__ void block_exact_prefix(PrefShared<T>& sh, const float* __restrict__ V, int32_t n, bool select, bool record, int ck_stride) {
  constexpr int CH = T * kPrefE;   // elements per iteration
  // software pipeline: the values of the NEXT iteration (assuming this one ends without an exception, i.e. at pos + CH) are
  // requested before this iteration's scan, so their latency hides behind it; an exception moves pos elsewhere and they are dropped
  float vn[kPrefE];
  int32_t pre_pos = -1;
  const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
  int it = 0;
  while (true) {
    __syncthreads();
    const int32_t pos = sh.pos;
    if (pos >= n || (select && sh.answer >= 0)) break;
    const float S = sh.S;
    if (record && t == 0 && (it % ck_stride) == 0 && sh.n_ck < kPrefCk) { sh.ck_pos[sh.n_ck] = pos; sh.ck_S[sh.n_ck] = S; ++sh.n_ck; }
    ++it;
    if (it > n + 16) __trap();   // every iteration consumes at least one element: anything else is a bug, not a wait
    const int32_t n_it = min((int32_t)CH, n - pos);
    if (pos == 0) {
      // Head of the row: while S is within a few binades of the addends nearly every element is an exception (ties, binade
      // steps), so the first kPrefHead elements are summed the plain way by one thread out of shared memory -- 4 cycles per
      // element, ~1.5 us in all, instead of a dozen exception iterations.
      const int32_t nh = min(n_it, (int32_t)kPrefHead);
      for (int32_t k = t; k < nh; k += T) sh.v[k] = V[k];
      __syncthreads();
      if (t == 0) {
        float Sc = S;
        int32_t k = 0, ans = -1;
        for (; k < nh; ++k) {
          Sc = __fadd_rn(Sc, sh.v[k]);
          if (select && (double)Sc > sh.r) { ans = k; ++k; break; }
        }
        sh.S = Sc;
        sh.pos = k;
        if (ans >= 0) sh.answer = ans;
      }
      continue;
    }
    const uint32_t sb = __float_as_uint(S);
    const uint32_t eS = (sb >> 23) & 0xffu;
    const uint32_t M_in = eS ? ((sb & 0x7fffffu) | 0x800000u) : 0u;
    // select threshold in units of this binade's ulp: S_k > r  <=>  M_k > floor(r / ulp)
    uint32_t Mthr = 0x1000000u;
    if (select && eS) {
      const double x = ldexp(sh.r, 150 - (int)eS);   // r / 2^(eS-127-23)
      if (x < 16777216.0) Mthr = (uint32_t)floor(x);
    }
    uint32_t inc[kPrefE];
    bool flg[kPrefE];
    uint32_t l = 0;
    int myfirst = CH;
    float vcur[kPrefE];
    const bool have = pre_pos == pos;
#pragma unroll
    for (int e = 0; e < kPrefE; ++e) {
      const int32_t k = t * kPrefE + e;
      vcur[e] = have ? vn[e] : (k < n_it ? V[pos + k] : 0.f);
    }
    pre_pos = pos + CH;
#pragma unroll
    for (int e = 0; e < kPrefE; ++e) {
      const int32_t k2 = pre_pos + t * kPrefE + e;
      vn[e] = k2 < n ? V[k2] : 0.f;
    }
#pragma unroll
    for (int e = 0; e < kPrefE; ++e) {
      const int32_t k = t * kPrefE + e;
      const float v = vcur[e];
      sh.v[k] = v;
      const uint32_t vb = __float_as_uint(v);
      uint32_t in = 0; bool f = false;
      if (vb != 0u) {
        if (vb >> 31) f = true;                       // a negative weight: never speculated
        else {
          uint32_t ev = vb >> 23;
          const uint32_t mant = ev ? ((vb & 0x7fffffu) | 0x800000u) : (vb & 0x7fffffu);
          if (ev == 0u) ev = 1u;
          if (eS == 0u || ev > eS) f = true;
          else {
            const uint32_t sft = eS - ev;
            if (sft == 0u) in = mant;
            else if (sft <= 24u) {
              const uint32_t rem = mant & ((1u << sft) - 1u), half = 1u << (sft - 1u);
              in = (mant >> sft) + (rem > half ? 1u : 0u);
              f = rem == half;
            }
          }
        }
      }
      inc[e] = in; flg[e] = f;
      l += in;
    }
    // warp inclusive scan of the thread sums (l <= 4 * 2^24)
    uint32_t ws = l;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, ws, o); if (lane >= o) ws += y; }
    if (lane == 31) sh.warp_tot[wid] = min(ws, 0x2000000u);   // anything >= 2^24 means "crossed": clamp so that sums stay in 32 bits
    if (t == 0) { sh.first = CH; sh.hit = CH; }
    __syncthreads();
    uint32_t base = M_in + (ws - l);
    for (int w2 = 0; w2 < wid; ++w2) base += sh.warp_tot[w2];
    uint32_t Mk = base, Mbefore = base;
    int myhit = CH;
#pragma unroll
    for (int e = 0; e < kPrefE; ++e) {
      const int32_t k = t * kPrefE + e;
      const uint32_t prev = Mk;
      Mk += inc[e];
      if (k < n_it) {
        if ((flg[e] || Mk >= 0x1000000u) && myfirst == CH) { myfirst = k; Mbefore = prev; }
        if (select && Mk > Mthr && myhit == CH) myhit = k;
      }
    }
    if (myfirst < CH) atomicMin(&sh.first, myfirst);
    if (myhit < CH) atomicMin(&sh.hit, myhit);
    __syncthreads();
    const int f = sh.first, h = sh.hit;
    if (select && h < f) {   // every element before the first exception is final: the hit is real
      if (t == 0) sh.answer = pos + h;
      continue;
    }
    if (f >= n_it) {         // no exception: the whole stretch is accepted
      if (t * kPrefE < n_it && (t + 1) * kPrefE >= n_it) {   // owner of the last element: Mk of element n_it-1
        uint32_t Ml = base;
#pragma unroll
        for (int e = 0; e < kPrefE; ++e) if (t * kPrefE + e < n_it) Ml += inc[e];
        if (eS) sh.S = __uint_as_float((eS << 23) | (Ml & 0x7fffffu));
        sh.pos = pos + n_it;
      }
      continue;
    }
    if (myfirst == f) sh.m_prev = Mbefore;   // M before element f
    __syncthreads();
    if (t == 0) {
      float Sc = eS ? __uint_as_float((eS << 23) | (sh.m_prev & 0x7fffffu)) : S;
      int32_t k = f;
      const int32_t kend = min(f + kPrefSer, n_it);
      int32_t ans = -1;
      for (; k < kend; ++k) {
        Sc = __fadd_rn(Sc, sh.v[k]);
        if (select && (double)Sc > sh.r) { ans = pos + k; ++k; break; }
      }
      sh.S = Sc;
      sh.pos = pos + k;
      if (ans >= 0) sh.answer = ans;
    }
  }
}

// CTA per walker of `list` (T threads, T * kPrefE elements per iteration): huge rows get 1024-thread CTAs, big rows 256
template <int T>
__global__ void __launch_bounds__(T) k_walk_prefix_cta(DevGraph g, int32_t L, int32_t step, int32_t ctype, WalkState s,
                                                       const uint32_t* __restrict__ state, bool philox, unsigned long long key, WalkPlan wp,
                                                       const int32_t* __restrict__ list, int n_idx, int ticket_idx,
                                                       long long* __restrict__ out) {
  __shared__ PrefShared<T> sh;
  __shared__ unsigned int s_tk;
  const int t = threadIdx.x;
  const unsigned int n_list = wp.ctr[n_idx];
  while (true) {
    if (t == 0) s_tk = atomicAdd(&wp.ctr[ticket_idx], 1u);
    __syncthreads();
    const unsigned int k = s_tk;
    __syncthreads();
    if (k >= n_list) break;
    const int64_t i = list[k];
    const int32_t n = wp.deg[i];
    const float* V = wp.V + wp.voff[i];
    if (t == 0) { sh.pos = 0; sh.S = 0.f; sh.n_ck = 0; sh.answer = -1; }
    const int ck_stride = 1 + (n / (T * kPrefE)) / (kPrefCk / 2);
    block_exact_prefix(sh, V, n, false, true, ck_stride);
    if (t == 0) {
      const float total = sh.S;
      double u, u2;
      if (philox) philox_uniform2((unsigned long long)i, (uint32_t)step, 0x77616C6Bu, key, u, u2);
      else { uint32_t x = state[i]; u = minstd_uniform(x); }
      const double r = pick_r(u, 0.f, total);
      sh.r = r;
      // resume from the last checkpoint whose prefix does not exceed r (prefixes are non-decreasing; checkpoint 0 is 0)
      int c = 0;
      for (int j = 1; j < sh.n_ck; ++j) if (!((double)sh.ck_S[j] > r)) c = j; else break;
      sh.pos = sh.ck_pos[c]; sh.S = sh.ck_S[c]; sh.answer = -1;
    }
    block_exact_prefix(sh, V, n, true, false, 1);
    if (t == 0) {
      const int64_t crow = s.cur_row[i];
      const int64_t cb = g.grp_ptr[crow * g.T + ctype];
      const int32_t a = sh.answer >= 0 ? sh.answer : n - 1;    // RandomSelect's fall-through: the last entry
      const long long next = (long long)__ldg(g.nbr + cb + a);
      out[i * (L + 1) + step + 1] = next;
      s.parent[i] = s.cur[i];
      s.parent_row[i] = crow;
      s.cur[i] = next;
    }
    __syncthreads();
  }
}

// warp per walker: rows of up to kWalkBig edges over V, then the walkers whose row did not fit in V (self-contained WarpWalk)
__global__ void __launch_bounds__(256) k_walk_prefix_warp(DevGraph g, int32_t L, int32_t step, int32_t ctype, int32_t ptype, float p, float q,
                                                          long long default_node, WalkState s, const uint32_t* __restrict__ state, bool philox,
                                                          unsigned long long key, WalkPlan wp, long long* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const unsigned int n_small = wp.ctr[1];
  // ---- small walkers (deg <= kWalkBig): one warp each over the row's biased weights in V.  The prefix is the plain
  // left-to-right f32 chain evaluated through shuffles (<= 16 chunks of 32); pass 1 = total, pass 2 = select.
  while (true) {
    unsigned int k = 0;
    if (lane == 0) k = atomicAdd(&wp.ctr[4], 1u);
    k = __shfl_sync(0xffffffffu, k, 0);
    if (k >= n_small) break;
    const int64_t i = wp.small_list[k];
    const int32_t n = wp.deg[i];
    const float* V = wp.V + wp.voff[i];
    float run = 0.f;
    for (int32_t c0 = 0; c0 < n; c0 += 32) {
      const float w = c0 + lane < n ? V[c0 + lane] : 0.f;
      const int nv = min(32, n - c0);
      for (int j = 0; j < nv; ++j) run = __fadd_rn(run, __shfl_sync(0xffffffffu, w, j));
    }
    double u, u2;
    if (philox) philox_uniform2((unsigned long long)i, (uint32_t)step, 0x77616C6Bu, key, u, u2);
    else { uint32_t x = state[i]; u = minstd_uniform(x); }
    const double r = pick_r(u, 0.f, run);
    int32_t ans = n - 1;                 // RandomSelect's fall-through: the last entry
    run = 0.f;
    for (int32_t c0 = 0; c0 < n; c0 += 32) {
      const float w = c0 + lane < n ? V[c0 + lane] : 0.f;
      const int nv = min(32, n - c0);
      float mine = 0.f;
      for (int j = 0; j < nv; ++j) { run = __fadd_rn(run, __shfl_sync(0xffffffffu, w, j)); if (lane == j) mine = run; }
      const unsigned hit = __ballot_sync(0xffffffffu, lane < nv && (double)mine > r);
      if (hit) { ans = c0 + __ffs(hit) - 1; break; }
    }
    if (lane == 0) {
      const int64_t crow = s.cur_row[i];
      const long long next = (long long)__ldg(g.nbr + g.grp_ptr[crow * g.T + ctype] + ans);
      out[i * (L + 1) + step + 1] = next;
      s.parent[i] = s.cur[i];
      s.parent_row[i] = crow;
      s.cur[i] = next;
    }
  }
  // ---- walkers whose row did not fit in V: the self-contained warp path
  const unsigned int n_ovf = wp.ctr[5];
  while (true) {
    unsigned int k = 0;
    if (lane == 0) k = atomicAdd(&wp.ctr[6], 1u);
    k = __shfl_sync(0xffffffffu, k, 0);
    if (k >= n_ovf) break;
    const int64_t i = wp.ovf_list[k];
    const long long cur = s.cur[i];
    const int64_t crow = s.cur_row[i];
    const int64_t prow = s.parent_row[i];
    WarpWalk ww;
    ww.g = &g; ww.lane = lane; ww.p = p; ww.q = q; ww.parent_id = s.parent[i];
    ww.cbase = g.grp_ptr[crow * g.T];
    ww.cb = g.grp_ptr[crow * g.T + ctype];
    ww.ce = g.grp_ptr[crow * g.T + ctype + 1];
    ww.pb = ww.pe = 0;
    if (prow >= 0 && ptype >= 0 && ptype < g.T) { ww.pb = g.grp_ptr[prow * g.T + ptype]; ww.pe = g.grp_ptr[prow * g.T + ptype + 1]; }
    const float total = ww.pass(false, 0.0, nullptr);
    double u, u2;
    if (philox) philox_uniform2((unsigned long long)i, (uint32_t)step, 0x77616C6Bu, key, u, u2);
    else { uint32_t x = state[i]; u = minstd_uniform(x); }
    long long next = default_node;
    ww.pass(true, pick_r(u, 0.f, total), &next);
    if (lane == 0) {
      out[i * (L + 1) + step + 1] = next;
      s.parent[i] = cur;
      s.parent_row[i] = crow;
      s.cur[i] = next;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------- fast mode
// EU_RNG_PHILOX ("throughput mode": same algorithm and distribution, counter-based stream): a node2vec step by REJECTION
// instead of the O(deg) biased prefix.  The target is P(j) ~ w_j * b_j with b_j in {1/p, 1, 1/q} (BuildWeights,
// random_walk_op.cc:140-168); propose j ~ w_j by one inverse-CDF search in the row's stored cumulative weights, accept with
// probability b_j / max(b): O(log deg(cur) + log deg(prev)) per try, expected tries <= max(b) / min(b) (4 at p=0.5, q=2).
// A walker no longer depends on any other walker, so one thread carries it through every step of the launch; after kFastTries
// rejections (extreme p/q) the thread evaluates the biased row exactly.  Multi-edges follow the reference's multiset rule: the
// m-th copy of id v in the child list is "shared" iff the parent's list holds more than m copies of v.
static constexpr int kFastSteps = 96;
static constexpr int kFastTries = 96;
struct FastTypes {
  int32_t prev;                 // edge type of the step before the first one of this launch (-1 = empty parent list)
  int32_t v[kFastSteps];
};

__device__ __forceinline__ double fast_bias(const DevGraph& g, int64_t cb, int64_t j, long long cv, int64_t pb, int64_t pe, long long parent,
                                            double bp, double bq) {
  int64_t m = 0;
  while (j - 1 - m >= cb && (long long)__ldg(g.nbr + j - 1 - m) == cv) ++m;
  if (pe > pb) {
    const int64_t lb = lower_bound_ll(g.nbr, pb, pe, cv);
    if (lb + m < pe && (long long)__ldg(g.nbr + lb + m) == cv) return 1.0;
  }
  return cv != parent ? bq : bp;
}

__global__ void k_walk_fast_done(EuRngState* rng) { rng->calls += 1; }

__global__ void __launch_bounds__(128) k_walk_fast(DevGraph g, int64_t B, int32_t L, int32_t l0, int32_t nl, FastTypes ft, float p, float q,
                                                   long long default_node, WalkState s, unsigned long long key, const EuRngState* __restrict__ rng,
                                                   long long* __restrict__ out) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= B) return;
  key ^= rng->calls * 0x9E3779B97F4A7C15ull;       // a new stream per call (device-side counter: CUDA-graph replays advance too)
  long long cur = s.cur[i], parent = s.parent[i];
  int64_t prow = s.parent_row[i];
  const double bp = 1.0 / (double)p, bq = 1.0 / (double)q;
  const double bmax = fmax(1.0, fmax(bp, bq));
  int32_t ptype = ft.prev;
  for (int32_t k = 0; k < nl; ++k) {
    const int32_t step = l0 + k, ctype = ft.v[k];
    const int64_t crow = lookup_row(g, (unsigned long long)cur);
    int64_t cb = 0, ce = 0, cbase = 0;
    if (crow >= 0 && ctype >= 0 && ctype < g.T) {
      cbase = g.grp_ptr[crow * g.T];
      cb = g.grp_ptr[crow * g.T + ctype];
      ce = g.grp_ptr[crow * g.T + ctype + 1];
    }
    long long next = default_node;
    if (ce > cb) {
      int64_t pb = 0, pe = 0;
      if (prow >= 0 && ptype >= 0 && ptype < g.T) { pb = g.grp_ptr[prow * g.T + ptype]; pe = g.grp_ptr[prow * g.T + ptype + 1]; }
      const double lo = cb == cbase ? 0.0 : (double)__ldg(g.cum_w + cb - 1);
      const double hi = (double)__ldg(g.cum_w + ce - 1);
      int64_t pick = ce - 1;                       // RandomSelect's fall-through (a row of zero weights): the last entry
      if (hi > lo) {
        bool done = false;
        for (int a = 0; a < kFastTries && !done; ++a) {
          double u, u2;
          philox_uniform2((unsigned long long)i, (uint32_t)step, 0x66617374u + (uint32_t)a, key, u, u2);
          const double r = lo + u * (hi - lo);
          int64_t x = cb, y = ce - 1;              // first j with cum_w[j] > r, clamped to the last entry
          while (x < y) { const int64_t mid = x + ((y - x) >> 1); if ((double)__ldg(g.cum_w + mid) > r) y = mid; else x = mid + 1; }
          const long long cv = (long long)__ldg(g.nbr + x);
          if (u2 * bmax < fast_bias(g, cb, x, cv, pb, pe, parent, bp, bq)) { pick = x; done = true; }
        }
        if (!done) {
          // exact evaluation of the biased row (two passes, f64 accumulation)
          double tot = 0.0;
          for (int64_t j = cb; j < ce; ++j) {
            const double w = (double)__ldg(g.cum_w + j) - (j == cbase ? 0.0 : (double)__ldg(g.cum_w + j - 1));
            tot += w * fast_bias(g, cb, j, (long long)__ldg(g.nbr + j), pb, pe, parent, bp, bq);
          }
          double u, u2;
          philox_uniform2((unsigned long long)i, (uint32_t)step, 0x66617374u + (uint32_t)kFastTries, key, u, u2);
          const double r = u * tot;
          double run = 0.0;
          for (int64_t j = cb; j < ce; ++j) {
            const double w = (double)__ldg(g.cum_w + j) - (j == cbase ? 0.0 : (double)__ldg(g.cum_w + j - 1));
            run += w * fast_bias(g, cb, j, (long long)__ldg(g.nbr + j), pb, pe, parent, bp, bq);
            if (run > r) { pick = j; break; }
          }
        }
      }
      next = (long long)__ldg(g.nbr + pick);
    }
    out[i * (L + 1) + step + 1] = next;
    parent = cur;
    prow = crow;                                   // dead walkers keep the bookkeeping of the live ones (k_walk_dead)
    cur = next;
    ptype = ctype;
  }
  s.cur[i] = cur; s.parent[i] = parent; s.parent_row[i] = prow;
}

// dead walkers: default_node forever (:232-241); parent bookkeeping as for the live ones
__global__ void k_walk_dead(int64_t B, int32_t L, int32_t step, long long default_node, WalkState s, const uint8_t* __restrict__ live,
                            long long* __restrict__ out) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= B || live[i]) return;
  out[i * (L + 1) + step + 1] = default_node;
  s.parent[i] = s.cur[i];
  s.parent_row[i] = s.cur_row[i];
  s.cur[i] = default_node;
}

__global__ void k_walk_col(const unsigned long long* __restrict__ eng, int64_t B, int32_t L, int32_t col,
                           long long default_node, long long* __restrict__ out) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= B) return;
  unsigned long long v = eng[i];
  out[i * (L + 1) + col] = v == 0ull ? default_node : (long long)v;
}

// tf_euler gen_pair (tf_euler/kernels/gen_pair_op.cc:41-100): skip-gram pairs of every path.  For position j the pairs
// (path[j], path[j-1]), ..., (path[j], path[j-lw]) then (path[j], path[j+1]), ..., (path[j], path[j+rw]), clipped to the
// path; positions in ascending j.  pairs_before(j) is a closed form, so every (path, j) writes independently.
__device__ __forceinline__ long long pairs_before(long long j, long long len, long long lw, long long rw) {
  // sum_{x<j} min(x, lw) + sum_{x<j} min(len-1-x, rw)
  const long long a = j <= lw ? j * (j - 1) / 2 : lw * (lw - 1) / 2 + (j - lw) * lw;
  // right: y = len-1-x runs over len-1 .. len-j ; min(y, rw)
  const long long hi = len - 1, lo = len - j;              // y in [lo, hi], j terms
  long long b = 0;
  if (j > 0) {
    if (lo >= rw) b = j * rw;
    else {
      const long long full = hi >= rw ? hi - rw + 1 : 0;   // y in [rw, hi] -> rw each
      const long long top = hi >= rw ? rw - 1 : hi;        // y in [lo, top] -> y each
      b = full * rw + (top >= lo ? (lo + top) * (top - lo + 1) / 2 : 0);
    }
  }
  return a + b;
}

__global__ void k_gen_pair(const long long* __restrict__ paths, int64_t B, int32_t len, int32_t lw, int32_t rw, long long pair_count,
                           long long* __restrict__ out) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= B * (int64_t)len) return;
  const int64_t r = i / len;
  const int32_t j = (int32_t)(i - r * len);
  const long long* path = paths + r * len;
  long long* o = out + (r * pair_count + pairs_before(j, len, lw, rw)) * 2;
  const long long me = path[j];
  for (int32_t k = 0; j - k - 1 >= 0 && k < lw; ++k) { *o++ = me; *o++ = path[j - k - 1]; }
  for (int32_t k = 0; j + k + 1 < len && k < rw; ++k) { *o++ = me; *o++ = path[j + k + 1]; }
}

}  // namespace eu

using namespace eu;

// pairs per path, exactly as the kernel counts them (gen_pair_op.cc:47-53)
extern "C" int64_t eu_gen_pair_count(int32_t path_len, int32_t left_win_size, int32_t right_win_size) {
  long long pc = (long long)path_len * ((long long)left_win_size + right_win_size);
  for (int i = left_win_size, j = 0; i > 0 && j < path_len; --i, ++j) pc -= i;
  for (int i = right_win_size, j = 0; i > 0 && j < path_len; --i, ++j) pc -= i;
  return pc;
}

// tf_euler.gen_pair: paths i64[B, path_len] -> out i64[B, eu_gen_pair_count(...), 2]   (device pointers)
extern "C" int eu_gen_pair(eu_ctx* c, const int64_t* paths, int64_t B, int32_t path_len, int32_t left_win_size, int32_t right_win_size,
                           int64_t* out) {
  if (!c || B < 0 || path_len < 0 || left_win_size < 0 || right_win_size < 0) { set_error("eu_gen_pair: bad argument"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  const long long pc = eu_gen_pair_count(path_len, left_win_size, right_win_size);
  if (B == 0 || path_len == 0 || pc == 0) return EU_OK;     // nothing to write (a path of one node has no pairs)
  if (!paths || !out) { set_error("eu_gen_pair: null buffer"); return EU_ERR_INVALID; }
  k_gen_pair<<<(unsigned)ceil_div(B * (int64_t)path_len, 256), 256, 0, c->stream>>>((const long long*)paths, B, path_len, left_win_size,
                                                                                    right_win_size, pc, (long long*)out);
  EU_LAUNCHED();
  return EU_OK;
}

extern "C" int eu_random_walk(eu_ctx* c, const int64_t* nodes, int64_t B, const int32_t* etypes, int32_t K,
                              int32_t L, float p, float q, int64_t default_node, int64_t* out) {
  if (!c || B < 0 || L < 0 || K < 0 || K > EU_MAX_ETYPES || (L > 0 && K > 0 && !etypes) || (B > 0 && (!nodes || !out))) {
    set_error("eu_random_walk: bad argument");
    return EU_ERR_INVALID;
  }
  EU_CUDA(cudaSetDevice(c->g->device));
  if (B == 0) return EU_OK;
  const DevGraph& d = c->g->d;
  cudaStream_t s = c->stream;
  const int tb = 256;
  int rc = ctx_reserve(c, hop_scratch_rows(1, B), hop_table_slots(1, B));
  if (rc) return rc;
  const float kEps = 1.0e-6f;
  if (fabs((double)p - 1.0) <= kEps && fabs((double)q - 1.0) <= kEps) {
    // TraditionalRandomWalk: chained sampleNB(count=1); the frontier is the ENGINE id (0 placeholder)
    EU_CUDA(cudaMemcpy2DAsync(out, sizeof(int64_t) * (L + 1), nodes, sizeof(int64_t), sizeof(int64_t), (size_t)B,
                              cudaMemcpyDeviceToDevice, s));
    const unsigned long long* seeds = (const unsigned long long*)nodes;
    for (int l = 0; l < L; ++l) {
      unsigned long long* eng = c->d_front[l & 1];
      rc = hop(c, seeds, B, etypes + (int64_t)l * K, K, 1, default_node, eng, nullptr, nullptr, nullptr,
               l, l > 0 && c->rng == EU_RNG_MINSTD, l + 1 < L, 1);
      if (rc) return rc;
      k_walk_col<<<(unsigned)ceil_div(B, tb), tb, 0, s>>>(eng, B, L, l + 1, default_node, (long long*)out);
      EU_LAUNCHED();
      seeds = eng;
    }
    return EU_OK;
  }
  // node2vec
  const int64_t plan_bytes = B * (4 + 4 + 4 + 4 + 4 + 4) + (B + 1) * (8 + 4) + 128 + 256;
  rc = ctx_misc(c, 256 + B * (8 + 8 + 8 + 8) + plan_bytes);
  if (rc) return rc;
  char* m = (char*)c->d_misc + 256;
  WalkState ws;
  ws.cur = (long long*)m; m += 8 * B;
  ws.parent = (long long*)m; m += 8 * B;
  ws.cur_row = (int64_t*)m; m += 8 * B;
  ws.parent_row = (int64_t*)m; m += 8 * B;
  WalkPlan wp{};
  wp.voff = (long long*)m; m += 8 * (B + 1);
  wp.deg = (int32_t*)m; m += 4 * B;
  wp.live_list = (int32_t*)m; m += 4 * B;
  wp.huge_list = (int32_t*)m; m += 4 * B;
  wp.big_list = (int32_t*)m; m += 4 * B;
  wp.small_list = (int32_t*)m; m += 4 * B;
  wp.ovf_list = (int32_t*)m; m += 4 * B;
  wp.coff = (int32_t*)m; m += 4 * (B + 1);
  m = (char*)(((uintptr_t)m + 63) & ~(uintptr_t)63);
  wp.ctr = (unsigned int*)m;
  k_walk_init<<<(unsigned)ceil_div(B, tb), tb, 0, s>>>((const long long*)nodes, B, L, ws, (long long*)out);
  EU_LAUNCHED();
  ETypes2 pet{};
  pet.K = 0;
  const bool philox = c->rng == EU_RNG_PHILOX;
  const unsigned long long wkey = c->seed ^ 0x6E32766563ull;
  if (philox && K == 1 && d.adj_sorted && !getenv("EU_WALK_FAST_OFF")) {
    // throughput mode: rejection steps, every walker independent, kFastSteps steps per launch
    for (int l0 = 0; l0 < L; l0 += kFastSteps) {
      FastTypes ft{};
      ft.prev = l0 == 0 ? -1 : etypes[l0 - 1];
      const int nl = std::min(kFastSteps, L - l0);
      for (int k = 0; k < nl; ++k) ft.v[k] = etypes[l0 + k];
      EuProfScope ps(c, "k_walk_fast", B);
      k_walk_fast<<<(unsigned)ceil_div(B, 128), 128, 0, s>>>(d, B, L, l0, nl, ft, p, q, default_node, ws, wkey, c->d_rng, (long long*)out);
      EU_LAUNCHED();
    }
    k_walk_fast_done<<<1, 1, 0, s>>>(c->d_rng);
    EU_LAUNCHED();
    return EU_OK;
  }
  for (int l = 0; l < L; ++l) {
    ETypes2 cet{};
    cet.K = K;
    for (int k = 0; k < K; ++k) cet.v[k] = etypes[(int64_t)l * K + k];
    const bool one_sorted_type = d.adj_sorted && cet.K == 1 && pet.K <= 1 && cet.v[0] >= 0 && cet.v[0] < d.T && B < ((int64_t)1 << 31);
    if (one_sorted_type) {
      // V: biased weights of the big rows of this step (k_walk_weights -> k_walk_prefix); walkers that do not fit take the
      // warp path, so the capacity bounds memory, not correctness
      if (!c->d_walkv) {
        const char* e = getenv("EU_WALK_V_ELEMS");
        const long long want = e && atoll(e) > 0 ? atoll(e) : (32ll << 20);
        if ((rc = refuse_growth_in_capture(c, "the node2vec weight scratch"))) return rc;
        EU_CUDA(cudaMalloc(&c->d_walkv, sizeof(float) * (size_t)want));
        c->walkv_cap = want;
      }
      wp.V = c->d_walkv; wp.capV = c->walkv_cap;
      if (!c->aux[0]) {
        if ((rc = refuse_growth_in_capture(c, "the node2vec auxiliary streams"))) return rc;
        for (int i = 0; i < 2; ++i) {
          EU_CUDA(cudaStreamCreateWithFlags(&c->aux[i], cudaStreamNonBlocking));
          EU_CUDA(cudaEventCreateWithFlags(&c->ev_join[i], cudaEventDisableTiming));
        }
        EU_CUDA(cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming));
      }
      const int32_t ctype = cet.v[0], ptype = pet.K == 1 ? pet.v[0] : -1;
      { EuProfScope ps(c, "k_walk_deg", B);
        k_walk_deg<<<(unsigned)ceil_div(B, tb), tb, 0, s>>>(d, B, ctype, ws, c->d_elig, wp.deg); }
      EU_LAUNCHED();
      { EuProfScope ps(c, "k_walk_plan", B);
        k_walk_plan<<<1, 1024, 0, s>>>(B, c->d_elig, !philox, modpow_a(2ull), c->d_state, c->d_rng, wp); }
      EU_LAUNCHED();
      { EuProfScope ps(c, "k_walk_weights", B);
        k_walk_weights<<<kSMs * 8, kWalkChunk, 0, s>>>(d, ctype, ptype, p, q, ws, wp); }
      EU_LAUNCHED();
      if (c->prof) {   // per-kernel timing: one after the other on the ctx stream
        { EuProfScope ps(c, "k_walk_prefix_cta<1024>", B);
          k_walk_prefix_cta<1024><<<kSMs, 1024, 0, s>>>(d, L, l, ctype, ws, c->d_state, philox, wkey, wp, wp.huge_list, 8, 9, (long long*)out); }
        EU_LAUNCHED();
        { EuProfScope ps(c, "k_walk_prefix_cta<256>", B);
          k_walk_prefix_cta<256><<<kSMs * 4, 256, 0, s>>>(d, L, l, ctype, ws, c->d_state, philox, wkey, wp, wp.big_list, 0, 3, (long long*)out); }
        EU_LAUNCHED();
        { EuProfScope ps(c, "k_walk_prefix_warp", B);
          k_walk_prefix_warp<<<kSMs * 4, 256, 0, s>>>(d, L, l, ctype, ptype, p, q, default_node, ws, c->d_state, philox, wkey, wp, (long long*)out); }
        EU_LAUNCHED();
      } else {
        // the three are independent (disjoint walkers): fork onto two auxiliary streams, join back -- a step then costs its
        // longest list, not the sum
        EU_CUDA(cudaEventRecord(c->ev_fork, s));
        EU_CUDA(cudaStreamWaitEvent(c->aux[0], c->ev_fork, 0));
        EU_CUDA(cudaStreamWaitEvent(c->aux[1], c->ev_fork, 0));
        k_walk_prefix_cta<1024><<<kSMs, 1024, 0, c->aux[0]>>>(d, L, l, ctype, ws, c->d_state, philox, wkey, wp, wp.huge_list, 8, 9, (long long*)out);
        EU_LAUNCHED();
        k_walk_prefix_cta<256><<<kSMs * 4, 256, 0, c->aux[1]>>>(d, L, l, ctype, ws, c->d_state, philox, wkey, wp, wp.big_list, 0, 3, (long long*)out);
        EU_LAUNCHED();
        k_walk_prefix_warp<<<kSMs * 4, 256, 0, s>>>(d, L, l, ctype, ptype, p, q, default_node, ws, c->d_state, philox, wkey, wp, (long long*)out);
        EU_LAUNCHED();
        EU_CUDA(cudaEventRecord(c->ev_join[0], c->aux[0]));
        EU_CUDA(cudaEventRecord(c->ev_join[1], c->aux[1]));
        EU_CUDA(cudaStreamWaitEvent(s, c->ev_join[0], 0));
        EU_CUDA(cudaStreamWaitEvent(s, c->ev_join[1], 0));
      }
      k_walk_dead<<<(unsigned)ceil_div(B, tb), tb, 0, s>>>(B, L, l, default_node, ws, c->d_elig, (long long*)out);
      EU_LAUNCHED();
    } else {
      k_walk_live<<<(unsigned)ceil_div(B, tb), tb, 0, s>>>(d, B, cet, ws, c->d_elig);
      EU_LAUNCHED();
      if (!philox) {
        rc = launch_state_scan(c, B, 1);
        if (rc) return rc;
      }
      EuProfScope ps(c, "k_walk_step(sequential)", B);
      k_walk_step<<<(unsigned)ceil_div(B, 128), 128, 0, s>>>(d, B, L, l, cet, pet, p, q, default_node, ws, c->d_elig,
                                                             c->d_state, philox, wkey, (long long*)out);
      EU_LAUNCHED();
    }
    pet = cet;
  }
  return EU_OK;
}

