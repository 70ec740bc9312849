// euler_b200 device-side building blocks (sm_90a).
//   * DevGraph: the HBM-resident CSR a kernel sees
//   * exact RNG: minstd_rand0 + libstdc++ generate_canonical<double,53>, with multiplicative
//     jump-ahead so each warp/lane starts at its own position of the ONE serial stream the
//     reference consumes (euler/common/random.cc:22-28; SURVEY.md section 8c, Appendix A-15)
//   * Philox4x32-10 keyed on (node id, draw) for the throughput mode
//   * inverse-CDF pick equivalent to RandomSelect (euler/common/compact_weighted_collection.h:30-52)
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#define EU_WARP 32
#define EU_MAX_ETYPES 32
#define EU_MAX_FEAT_SLOTS 16

namespace eu {

struct HashSlot {  // 16 B, one 128-bit load
  unsigned long long key;
  unsigned long long row;  // EU_EMPTY_ROW if free
};
static constexpr unsigned long long kEmptyRow = 0xFFFFFFFFFFFFFFFFull;
// SMs of an H100 SXM: the grid caps of the grid-stride and persistent kernels are multiples of it
static constexpr int kSMs = 132;

struct DevGraph {
  int64_t n;        // rows
  int64_t E;        // edges
  int32_t T;        // edge-type groups per row
  int32_t n_node_types;
  const unsigned long long* ids;  // [n]
  const int32_t* node_type;       // [n]
  const float* node_w;            // [n]
  const int64_t* grp_ptr;         // [n*T+1]
  const unsigned long long* nbr;  // [E]
  const float* cum_w;             // [E]
  const float* grp_cum;           // [n*T] (T>1) or nullptr
  // id -> row
  int32_t adj_sorted;             // every adjacency group is non-decreasing in (signed) neighbor id
  int32_t dense_ids;              // ids[r] == id_base + r * id_stride for all r
  unsigned long long id_base;
  unsigned long long id_stride;   // 1, or the shard count for a shard's rows (ids congruent mod shards)
  const HashSlot* htab;
  unsigned long long hmask;       // capacity-1 (capacity is a power of two)
  // dense features: row-major [n, feat_dim] of feat_dtype (EU_FEAT_F32: float, EU_FEAT_BF16: __nv_bfloat16), read only
  // through feat_cols / feat_ld / feat_ld4; slot s occupies columns [slot_off[s], +slot_dim[s])
  int32_t feat_dim;
  int32_t feat_dtype;             // fills the padding after feat_dim: every other member keeps its offset
  const void* feat;
  int32_t n_slots;
  int32_t slot_off[EU_MAX_FEAT_SLOTS];
  int32_t slot_dim[EU_MAX_FEAT_SLOTS];
  // ragged features (Node::uint64_features_ / binary_features_ with their *_idx_ ends, node.h): slot s of row r is
  // [ptr[r*S+s], ptr[r*S+s+1]) of the value array; S = 0 when the graph has none
  int32_t n_u64_slots;
  const int64_t* u64_ptr;
  const unsigned long long* u64_val;
  int32_t n_bin_slots;
  const int64_t* bin_ptr;
  const unsigned char* bin_val;
  // where the dense table lives (eu_feat_place: kFeatDevice / kFeatHost; appended so every member above keeps its offset).
  // Host: feat is the device pointer of a mapped pinned host table holding every row, feat_cache [feat_cache_rows, feat_dim]
  // of feat_dtype in HBM copies the rows of highest in-degree, and feat_slot[n] (HBM) maps a row to its cache row or -1.
  // Read rows only through feat_row.
  int32_t feat_place;
  const void* feat_cache;
  const int32_t* feat_slot;
  int64_t feat_cache_rows;
};

// edge store (edges.cu): SoA edge arrays + (src, dst, type) -> row table + features with the node layout
struct EdgeSlot {   // 32 B
  unsigned long long src, dst;
  int32_t type, pad;
  long long row;    // -1 = free
};
struct DevEdges {
  int64_t n;
  const unsigned long long* src;
  const unsigned long long* dst;
  const int32_t* type;
  const float* w;
  const EdgeSlot* htab;
  unsigned long long hmask;
  int32_t feat_dim;
  const float* feat;
  int32_t n_slots;
  int32_t slot_off[EU_MAX_FEAT_SLOTS];
  int32_t slot_dim[EU_MAX_FEAT_SLOTS];
  int32_t n_u64_slots;
  const int64_t* u64_ptr;
  const unsigned long long* u64_val;
  int32_t n_bin_slots;
  const int64_t* bin_ptr;
  const unsigned char* bin_val;
};

__host__ __device__ __forceinline__ unsigned long long mix64(unsigned long long k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdULL; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ULL; k ^= k >> 33;
  return k;
}

// Graph::GetNodeByID (euler/core/graph/graph.h:87-93): row or -1.
__device__ __forceinline__ int64_t lookup_row(const DevGraph& g, unsigned long long id) {
  if (g.dense_ids) {
    unsigned long long r = id - g.id_base;
    if (g.id_stride != 1) {
      if (id < g.id_base || r % g.id_stride) return -1;
      r /= g.id_stride;
    }
    return r < (unsigned long long)g.n ? (int64_t)r : -1;
  }
  unsigned long long h = mix64(id) & g.hmask;
  while (true) {
    const ulonglong2 s = __ldg(reinterpret_cast<const ulonglong2*>(g.htab + h));
    if (s.y == kEmptyRow) return -1;
    if (s.x == id) return (int64_t)s.y;
    h = (h + 1) & g.hmask;
  }
}

// the row i of listed entry e: the last i in [lo, hi] with ptr[i] <= e (rows before it may be empty)
__device__ __forceinline__ int64_t hop_row_of(const long long* __restrict__ ptr, int64_t lo, int64_t hi, int64_t e) {
  while (lo < hi) {
    const int64_t mid = (lo + hi + 1) >> 1;
    if (ptr[mid] <= e) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// Dense slot `fid`'s columns of a feature row: [*off, *off + *width).  An unknown slot has none, so every fetch of it reads
// zeros (Node::GetFloat32Feature skips it, node.cc:353-364; api.cc:71-73).
__host__ __device__ __forceinline__ void dense_slot(const DevGraph& g, int32_t fid, int32_t* off, int32_t* width) {
  const bool have = fid >= 0 && fid < g.n_slots;
  *off = have ? g.slot_off[fid] : 0;
  *width = have ? g.slot_dim[fid] : 0;
}

// ---------------------------------------------------------------------------------- dense feature storage
// The one place that knows how a dense feature table is stored.  A kernel that reads rows is instantiated for its storage
// type T (float or __nv_bfloat16), takes the table as feat_cols<T>(g) and loads columns with feat_ld (one) or feat_ld4 (four
// consecutive), which widen to f32 (f32 / bf16 elements, below).  A bf16 table is written only through feat_st, the device's
// round to nearest even.
template <typename T>
__host__ __device__ __forceinline__ const T* feat_cols(const DevGraph& g) { return static_cast<const T*>(g.feat); }

// eu_feat_place (include/euler_b200.h)
enum : int { kFeatDevice = 0, kFeatHost = 1 };

// Where a kernel finds row `row` (>= 0) of the table, for the table's placement P (kFeatDevice or kFeatHost, a template
// argument like T, picked by the launcher from g.feat_place).  Device: the HBM table.  Host: the HBM cache row when the slot
// map gives one, else the row of the mapped host table.  Both tiers hold the same bits, so what a kernel reads never depends
// on the placement or the cache size.  feat_row(g, row, W, col) is column col of the row, with W the row width where the
// kernel knows it at compile time (it must equal g.feat_dim).  The device forms are the expressions the kernels used before
// placement existed, term for term, so the device instantiations compile to the same instructions.
template <typename T, int P>
__device__ __forceinline__ const T* feat_row(const DevGraph& g, int64_t row, int32_t W, int32_t col) {
  if (P == kFeatHost) {
    const int32_t s = __ldg(g.feat_slot + row);
    if (s >= 0) return static_cast<const T*>(g.feat_cache) + col + (int64_t)s * W;
  }
  return feat_cols<T>(g) + col + row * (int64_t)W;
}
template <typename T, int P>
__device__ __forceinline__ const T* feat_row(const DevGraph& g, int64_t row) {
  if (P == kFeatHost) {
    const int32_t s = __ldg(g.feat_slot + row);
    if (s >= 0) return static_cast<const T*>(g.feat_cache) + (int64_t)s * g.feat_dim;
  }
  return feat_cols<T>(g) + row * (int64_t)g.feat_dim;
}
// column col of row `row` when ok, else the table's first element (which the caller must not read): a row that may be absent
template <typename T, int P>
__device__ __forceinline__ const T* feat_row_if(const DevGraph& g, bool ok, int64_t row, int32_t col) {
  if (P == kFeatHost) return ok ? feat_row<T, P>(g, row) + col : feat_cols<T>(g);
  return feat_cols<T>(g) + (ok ? row * (int64_t)g.feat_dim + col : 0);
}

// Row `row`'s slice of ragged slot `fid` (ptr of S slots per row): [b, e) in the value array, b == e when the node / slot does
// not exist
__device__ __forceinline__ void ragged_slice(const int64_t* __restrict__ ptr, int32_t S, int64_t row, int32_t fid, int64_t* b, int64_t* e) {
  *b = *e = 0;
  if (row < 0 || fid < 0 || fid >= S || !ptr) return;
  *b = ptr[row * S + fid];
  *e = ptr[row * S + fid + 1];
}

// ---------------------------------------------------------------------------------- minstd_rand0
static constexpr uint32_t kM = 2147483647u;  // 2^31-1
static constexpr uint32_t kA = 16807u;

__host__ __device__ __forceinline__ uint32_t modmul(uint32_t a, uint32_t b) {
  unsigned long long p = (unsigned long long)a * b;     // < 2^62
  unsigned long long r = (p & kM) + (p >> 31);          // < 2^32
  r = (r & kM) + (r >> 31);
  return (uint32_t)(r >= kM ? r - kM : r);
}

__host__ __device__ __forceinline__ uint32_t modpow_a(unsigned long long e) {  // A^e mod M
  uint32_t base = kA, acc = 1;
  while (e) {
    if (e & 1) acc = modmul(acc, base);
    base = modmul(base, base);
    e >>= 1;
  }
  return acc;
}

// A^(e) for small e (< 256) with compile-time squarings: used for per-lane offsets.
__device__ __forceinline__ uint32_t modpow_a_small(uint32_t e) {
  // A^(2^k) mod M, k = 0..7
  constexpr uint32_t P0 = 16807u;
  uint32_t acc = 1, base = P0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    if (e & (1u << k)) acc = modmul(acc, base);
    base = modmul(base, base);
  }
  return acc;
}

// One uniform_real_distribution<double>(0,1) draw from engine state `x` (state BEFORE the draw);
// advances x by two engine steps.  Arithmetic order of libstdc++ 13 generate_canonical<double,53>:
//   sum = double(x1-1); sum += double(x2-1) * R; ret = sum / (R*R); ret >= 1 -> nextafter(1,0)
// with R = 2147483646.0.  Explicit _rn intrinsics: no FMA contraction allowed (Appendix A-13/15).
__device__ __forceinline__ double minstd_uniform(uint32_t& x) {
  const double R = 2147483646.0;
  const double RR = 4611686009837453316.0;  // fl(R*R)
  x = modmul(x, kA);
  double sum = (double)(x - 1u);
  x = modmul(x, kA);
  sum = __dadd_rn(sum, __dmul_rn((double)(x - 1u), R));
  double ret = __ddiv_rn(sum, RR);
  if (ret >= 1.0) ret = 0x1.fffffffffffffp-1;  // nextafter(1.0, 0.0)
  return ret;
}

// ---------------------------------------------------------------------------------- per-call seed dedup table
// tab[h] = {id+1, min index}.  key 0 = free.
__device__ __forceinline__ void dedup_insert_one(HashSlot* tab, unsigned long long mask, unsigned long long id,
                                                 int64_t i) {
  const unsigned long long tag = id + 1;
  if (tag == 0ull) {  // id == 2^64-1 (e.g. default_node -1 fed back as a seed): dedicated slot [mask+1]
    atomicMin(&tab[mask + 1].row, (unsigned long long)i);
    return;
  }
  unsigned long long h = mix64(id) & mask;
  while (true) {
    unsigned long long prev = atomicCAS(&tab[h].key, 0ull, tag);
    if (prev == 0ull || prev == tag) {
      atomicMin(&tab[h].row, (unsigned long long)i);
      return;
    }
    h = (h + 1) & mask;
  }
}


// Slots a batch's dedup region really uses: the power of two >= 2 * live rows (>= 64), at most the region's capacity.  A
// sharded owner sizes its regions for the worst case (every request of every rank) and learns the live count on the device:
// inserting, probing and wiping with this mask keeps the table -- and its wipe -- proportional to the rows that exist.
__device__ __forceinline__ int64_t dedup_cap_eff(int64_t cap_b, const int32_t* __restrict__ rows_act, int b) {
  if (!rows_act) return cap_b;
  const long long r2 = 2ll * (long long)rows_act[b];
  int64_t cap = 64;
  if (r2 > 64) cap = (int64_t)1 << (64 - __clzll(r2 - 1));
  return cap < cap_b ? cap : cap_b;
}

// ---------------------------------------------------------------------------------- philox4x32-10
__device__ __forceinline__ void philox_round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
  uint32_t hi0 = __umulhi(M0, c[0]), lo0 = M0 * c[0];
  uint32_t hi1 = __umulhi(M1, c[2]), lo1 = M1 * c[2];
  uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
  c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
}

// 2 uniforms in [0,1) with 53 bits from counter (id, draw) and key (seed, call)
__device__ __forceinline__ void philox_uniform2(unsigned long long id, uint32_t draw, uint32_t salt,
                                                unsigned long long key, double& u0, double& u1) {
  uint32_t c[4] = {(uint32_t)id, (uint32_t)(id >> 32), draw, salt};
  uint32_t k0 = (uint32_t)key, k1 = (uint32_t)(key >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    philox_round(c, k0, k1);
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  unsigned long long a = ((unsigned long long)c[0] << 32) | c[1];
  unsigned long long b = ((unsigned long long)c[2] << 32) | c[3];
  u0 = (double)(a >> 11) * (1.0 / 9007199254740992.0);
  u1 = (double)(b >> 11) * (1.0 / 9007199254740992.0);
}

// the 128 bits of one Philox4x32-10 block: counter (element lo, element hi, step, tensor), key seed
__device__ __forceinline__ uint4 philox_bits(unsigned long long seed, uint32_t step, uint32_t tensor, unsigned long long element) {
  uint32_t c[4] = {(uint32_t)element, (uint32_t)(element >> 32), step, tensor};
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    philox_round(c, k0, k1);
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return make_uint4(c[0], c[1], c[2], c[3]);
}

// ---------------------------------------------------------------------------------- f32 / bf16 elements
// The one place that knows how an element of an f32 or bf16 table (T = float or __nv_bfloat16) is read and written.  Reads
// return f32: widening bf16 is exact (its bits are the upper half of the f32's).  The 4-wide forms move four consecutive
// elements as one 16-byte f32 / 8-byte bf16 access, so the address must be aligned to four elements.  An f32 value is stored
// as it is; a bf16 one is rounded.
//   feat_ld, feat_ld4   loads through the read-only data cache (__ldg), for tables the kernel does not write
//   rw_ld, rw_ld4       plain loads, for kernels that write the table they read (the stores, the optimizers)
//   feat_st, rn_st4     round to nearest even: NaN becomes the canonical NaN, +-Inf stays, a finite value becomes +-Inf only
//                       where the rounding says so, and subnormals round like any other value
//   sr_st, sr_st4       stochastic rounding from given random words (SrKey), for trained tables
__device__ __forceinline__ float bf16_bits_f32(uint32_t h) { return __uint_as_float(h << 16); }
// four bf16 elements as the two words of one 8-byte access: columns 0..3 are the low and high halves of x, then of y
__device__ __forceinline__ float4 bf16x4_f32(uint2 u) {
  return make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xFFFF0000u), __uint_as_float(u.y << 16),
                     __uint_as_float(u.y & 0xFFFF0000u));
}
__device__ __forceinline__ uint2 bf16x4_bits(__nv_bfloat16 a, __nv_bfloat16 b, __nv_bfloat16 c, __nv_bfloat16 d) {
  return make_uint2(__bfloat16_as_ushort(a) | (uint32_t)__bfloat16_as_ushort(b) << 16,
                    __bfloat16_as_ushort(c) | (uint32_t)__bfloat16_as_ushort(d) << 16);
}

template <typename T> __device__ __forceinline__ float feat_ld(const T* p);
template <> __device__ __forceinline__ float feat_ld<float>(const float* p) { return __ldg(p); }
template <> __device__ __forceinline__ float feat_ld<__nv_bfloat16>(const __nv_bfloat16* p) {
  return bf16_bits_f32(__ldg(reinterpret_cast<const unsigned short*>(p)));
}
template <typename T> __device__ __forceinline__ float4 feat_ld4(const T* p);
template <> __device__ __forceinline__ float4 feat_ld4<float>(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
template <> __device__ __forceinline__ float4 feat_ld4<__nv_bfloat16>(const __nv_bfloat16* p) {
  return bf16x4_f32(__ldg(reinterpret_cast<const uint2*>(p)));
}

__device__ __forceinline__ float rw_ld(const float* p) { return *p; }
__device__ __forceinline__ float rw_ld(const __nv_bfloat16* p) { return bf16_bits_f32(*reinterpret_cast<const unsigned short*>(p)); }
__device__ __forceinline__ float4 rw_ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 rw_ld4(const __nv_bfloat16* p) { return bf16x4_f32(*reinterpret_cast<const uint2*>(p)); }

template <typename T> __device__ __forceinline__ T feat_st(float v);
template <> __device__ __forceinline__ float feat_st<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 feat_st<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
__device__ __forceinline__ void rn_st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ void rn_st4(__nv_bfloat16* p, float4 v) {
  *reinterpret_cast<uint2*>(p) = bf16x4_bits(feat_st<__nv_bfloat16>(v.x), feat_st<__nv_bfloat16>(v.y), feat_st<__nv_bfloat16>(v.z),
                                             feat_st<__nv_bfloat16>(v.w));
}

// Stochastic rounding with a 16-bit random integer r (the low half of a random word), added to the low half of the f32 bits
// before they are truncated, so v rounds up with probability (its distance from the value below) / ulp and the rounding is
// unbiased.  r = 0 truncates toward zero; r = 0x8000 rounds to nearest with ties away from zero.  +-Inf stays; a NaN keeps
// its sign and upper payload and is made quiet; a finite value can carry into +-Inf only from above the largest finite bf16.
// Round to nearest would lose every update smaller than half an ulp.
__device__ __forceinline__ __nv_bfloat16 sr_st(float v, uint32_t r) {
  const uint32_t u = __float_as_uint(v);
  const uint32_t h = (u & 0x7F800000u) == 0x7F800000u ? (u >> 16) | ((u & 0x007FFFFFu) ? 0x0040u : 0u)
                                                      : (u + (r & 0xFFFFu)) >> 16;
  return __ushort_as_bfloat16((unsigned short)h);
}
__device__ __forceinline__ void sr_st(float* p, float v, uint32_t) { *p = v; }
__device__ __forceinline__ void sr_st(__nv_bfloat16* p, float v, uint32_t r) {
  *reinterpret_cast<unsigned short*>(p) = __bfloat16_as_ushort(sr_st(v, r));
}
__device__ __forceinline__ void sr_st4(float* p, float4 v, const uint32_t (&)[4]) { rn_st4(p, v); }
__device__ __forceinline__ void sr_st4(__nv_bfloat16* p, float4 v, const uint32_t (&r)[4]) {
  *reinterpret_cast<uint2*>(p) = bf16x4_bits(sr_st(v.x, r[0]), sr_st(v.y, r[1]), sr_st(v.z, r[2]), sr_st(v.w, r[3]));
}

// The key of the random words that round a trained bf16 table: element e's words at a step are the four of philox_bits(seed,
// step, tensor, e), with step the low 32 bits of the device counter *step, read on the device (a captured CUDA graph replays
// with the live count) and once per thread.  An f32 table never reads it.
struct SrKey {
  unsigned long long seed;
  const int64_t* step;   // device step counter
  uint32_t tensor;
};
__device__ __forceinline__ uint4 sr_bits(const SrKey& k, uint32_t step, unsigned long long e) {
  return philox_bits(k.seed, step, k.tensor, e);
}
// the words of the elements [e, e + VW) of a table updated with up to three tensors: r[w][i] rounds tensor w of element e + i
template <int VW>
__device__ __forceinline__ void sr_words(const SrKey& k, int64_t e, uint32_t (&r)[3][VW]) {
  const uint32_t step = (uint32_t)__ldg(k.step);
#pragma unroll
  for (int i = 0; i < VW; ++i) {
    const uint4 q = sr_bits(k, step, (unsigned long long)(e + i));
    r[0][i] = q.x; r[1][i] = q.y; r[2][i] = q.z;
  }
}

// the host's widening of n bf16 bit patterns h to f32
inline void bf16_bits_f32_host(const uint16_t* h, int64_t n, float* out) {
  for (int64_t i = 0; i < n; ++i) {
    const uint32_t u = (uint32_t)h[i] << 16;
    memcpy(out + i, &u, sizeof(u));
  }
}

// ---------------------------------------------------------------------------------- TMA bulk copy (sm_90+)
// 1-D bulk copy global -> shared through the TMA unit, completion signalled on an mbarrier (SASS: UBLKCP + SYNCS).  One
// elected lane issues it and moves on; the consumers wait on the barrier's phase parity.  src, dst and bytes must be
// multiples of 16.
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// generic-proxy accesses to shared memory ordered before subsequent async-proxy (TMA) accesses of the same thread
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned long long* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
               : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}

// ---------------------------------------------------------------------------------- CDF pick
// r for a pick in [begin,end] of a cumulative array (compact_weighted_collection.h:33-36):
//   limit_begin = begin==first ? 0 : cum[begin-1]; r = u * (double)(limit_end - limit_begin) + limit_begin
// (f32 subtraction, then f64 multiply and f64 add, unfused).
__device__ __forceinline__ double pick_r(double u, float limit_begin, float limit_end) {
  float diff = __fsub_rn(limit_end, limit_begin);
  return __dadd_rn(__dmul_rn(u, (double)diff), (double)limit_begin);
}

// Smallest f32 whose value exceeds r (r >= 0: cumulative weights are non-negative).  For an f32 c,
// (double)c > r  <=>  c >= gt_threshold(r), which turns every probe of the search into one FSETP instead of
// F2F.F64 + DSETP.
__device__ __forceinline__ float gt_threshold(double r) {
  float f = __double2float_ru(r);                       // (double)f >= r
  if ((double)f == r) f = __int_as_float(__float_as_int(f) + 1);  // next f32 up (valid for f >= +0)
  return f;
}

// RandomSelect == min(end, first j in [begin,end] with (double)cum[j] > r) for non-decreasing cum
// (proof sketch in DESIGN.md; checked against the literal search in tests/test_oracle_golden.py).
// Search over a row slice in global memory; `base` points at the slice, offsets are 32-bit (a row has
// < 2^31 edges), thr = gt_threshold(r).  Returns the offset in [lo, hi].
// Invariant: the answer lies in [lo, hi]; hi is the clamp or an offset with base[hi] >= thr.
// 8-ary descent: 7 independent probes per round trip, for a search whose round trips are its cost.  Where the loads
// themselves are (the fanout sampler's deep hop), sample.cu bisects instead: same answer, a seventh of the probes per round.
__device__ __forceinline__ int32_t upper_bound_clamped(const float* __restrict__ base, int32_t lo, int32_t hi,
                                                       float thr) {
  while (hi - lo >= 8) {
    // probes p_i = lo + (i+1)*s + min(i+1, r), s = n/8, r = n%8: lo < p_0 < .. < p_6 < hi (any increasing probe set
    // gives the same answer; this one needs no 64-bit multiply)
    const int32_t n = hi - lo, s = n >> 3, r = n & 7;
    float v[7];
#pragma unroll
    for (int i = 0; i < 7; ++i) v[i] = __ldg(base + lo + (i + 1) * s + min(i + 1, r));
    int c = 0;
#pragma unroll
    for (int i = 0; i < 7; ++i) c += (v[i] >= thr) ? 0 : 1;                                          // monotone: a prefix is below thr
    const int32_t nlo = c > 0 ? lo + c * s + min(c, r) + 1 : lo;
    const int32_t nhi = c < 7 ? lo + (c + 1) * s + min(c + 1, r) : hi;
    lo = nlo; hi = nhi;
  }
  if (lo < hi) {  // fewer than 8 candidates below hi: one round of independent probes
    const int32_t n = hi - lo;
    int c = 0;
#pragma unroll
    for (int i = 0; i < 7; ++i) {
      const float v = i < n ? __ldg(base + lo + i) : __int_as_float(0x7f800000);
      c += (v >= thr) ? 0 : 1;
    }
    lo += c;
  }
  return lo;
}

}  // namespace eu
