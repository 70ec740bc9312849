// Host-side internals shared by the translation units of libeuler_b200.so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string.h>

#include <atomic>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/euler_b200.h"
#include "common.cuh"

namespace eu {

void set_error(const char* fmt, ...);
extern std::atomic<uint64_t> g_launches;

#define EU_CUDA(call)                                                                    \
  do {                                                                                   \
    cudaError_t _e = (call);                                                             \
    if (_e != cudaSuccess) {                                                             \
      ::eu::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e)); \
      return EU_ERR_CUDA;                                                                \
    }                                                                                    \
  } while (0)

#define EU_LAUNCHED()                                                              \
  do {                                                                             \
    ::eu::g_launches.fetch_add(1, std::memory_order_relaxed);                      \
    cudaError_t _e = cudaPeekAtLastError();                                        \
    if (_e != cudaSuccess) {                                                       \
      ::eu::set_error("%s:%d launch -> %s", __FILE__, __LINE__, cudaGetErrorString(_e)); \
      return EU_ERR_CUDA;                                                          \
    }                                                                              \
  } while (0)

static_assert((int)kFeatDevice == (int)EU_FEAT_DEVICE && (int)kFeatHost == (int)EU_FEAT_HOST, "eu_feat_place");

inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
// a table of eu_feat_dtype dtype takes 4-wide loads (16 bytes of f32, 8 of bf16) where p is aligned to four of its elements
inline bool aligned4_elems(const void* p, int dtype) { return ((uintptr_t)p & (dtype == EU_FEAT_BF16 ? 7 : 15)) == 0; }

// ---- the storage type of a table or feature row (eu_feat_dtype)
inline bool dtype_ok(int32_t dtype) { return dtype == EU_FEAT_F32 || dtype == EU_FEAT_BF16; }
// EU_OK for an eu_feat_dtype code, else EU_ERR_INVALID with "<who>: unknown <noun> dtype <dtype>"; a table's or a store's
// text also names the codes, a graph's feature text does not
inline int dtype_check(int32_t dtype, const char* who, const char* noun) {
  if (dtype_ok(dtype)) return EU_OK;
  set_error("%s: unknown %s dtype %d%s", who, noun, (int)dtype, strcmp(noun, "feature") ? " (EU_FEAT_F32 or EU_FEAT_BF16)" : "");
  return EU_ERR_INVALID;
}

template <typename T>
struct TypeTag { using type = T; };
// f(TypeTag<T>{}) with T the element type of a checked eu_feat_dtype code: float or __nv_bfloat16
template <typename F>
auto with_dtype(int32_t dtype, F&& f) {
  if (dtype == EU_FEAT_BF16) return f(TypeTag<__nv_bfloat16>{});
  return f(TypeTag<float>{});
}
// f(TypeTag<T>{}, std::integral_constant<int, P>{}) for the graph's dense feature table: T its element type, P its placement
// (kFeatDevice or kFeatHost)
template <typename F>
auto with_feat(const DevGraph& g, F&& f) {
  return with_dtype(g.feat_dtype, [&](auto t) {
    if (g.feat_place == EU_FEAT_HOST) return f(t, std::integral_constant<int, kFeatHost>{});
    return f(t, std::integral_constant<int, kFeatDevice>{});
  });
}

struct ETList {           // an edge-type list passed by value to the full-neighbor kernels
  int32_t K;
  int32_t v[EU_MAX_ETYPES];
};

struct TypeSampler {      // FastWeightedCollection of one node type (fast_weighted_collection.h:27-100)
  int64_t n = 0;
  unsigned long long* ids = nullptr;  // device, sampler order
  float* prob = nullptr;              // device
  int32_t* alias = nullptr;           // device
  float fwc_sum = 0.f;                // FWC::sum_weight_
};

}  // namespace eu

struct eu_graph {
  int device = 0;
  eu::DevGraph d{};
  std::vector<void*> allocs;
  int64_t hbm_bytes = 0;
  // mapped pinned host memory (a host-placed feature table: d.feat is its device pointer, feat_host the host one)
  std::vector<void*> host_allocs;
  int64_t host_bytes = 0;
  const void* feat_host = nullptr;
  // global node sampler (Graph::BuildGlobalSampler, graph.cc:333-370); built lazily
  bool sampler_built = false;
  std::vector<eu::TypeSampler> samplers;
  std::vector<float> type_sums;        // node_weight_sums_
  std::vector<float> type_prob;        // node_type_collection_ alias tables (host; tiny)
  std::vector<int32_t> type_alias;
  float type_fwc_sum = 0.f;
  float* d_type_prob = nullptr;
  int32_t* d_type_alias = nullptr;
  std::vector<int64_t> sampler_order;  // optional explicit order (rows)
  std::vector<std::string> edge_type_names, node_type_names;
  std::vector<std::string> dense_feature_names;  // per slot, without the "dense_" prefix
  std::vector<std::string> sparse_feature_names, binary_feature_names;   // per slot, without the "sparse_" / "binary_" prefix
  std::vector<uint64_t> u64_slot_max;  // per uint64 slot: its largest value (0 when it has none); bounds embedding lookups
  // edges (eu_graph_set_edges): device store, per-type alias samplers in edge_map_ order, feature names
  eu::DevEdges e{};
  bool edges_set = false;
  struct EdgeSampler { int64_t n = 0; const int64_t* order = nullptr; const float* prob = nullptr; const int32_t* alias = nullptr; float fwc_sum = 0.f; };
  std::vector<EdgeSampler> edge_samplers;
  std::vector<std::string> edge_dense_names, edge_sparse_names, edge_binary_names;
  // graph-label table (graph_label.cu), built lazily by the first graph-label call: the label list in Graph::GetGraphLabel's
  // order, and the rows of label l as the node ids [label_ptr[l], label_ptr[l + 1]) of label_ids, ascending
  bool labels_built = false;
  std::vector<std::string> labels;
  int32_t* d_label_ptr = nullptr;                 // [L + 1]
  unsigned long long* d_label_ids = nullptr;      // [label_ptr[L]]

  template <typename T>
  int alloc(T** p, int64_t count) {
    size_t bytes = (size_t)(count > 0 ? count : 1) * sizeof(T);
    bytes = (bytes + 255) & ~(size_t)255;
    void* q = nullptr;
    cudaError_t e = cudaMalloc(&q, bytes);
    if (e != cudaSuccess) {
      eu::set_error("cudaMalloc(%zu) -> %s", bytes, cudaGetErrorString(e));
      return EU_ERR_CUDA;
    }
    allocs.push_back(q);
    hbm_bytes += (int64_t)bytes;
    *p = (T*)q;
    return EU_OK;
  }
  // count elements of mapped pinned host memory: *host for the host, *dev for kernels
  template <typename T>
  int host_alloc(T** host, T** dev, int64_t count) {
    const size_t bytes = (size_t)(count > 0 ? count : 1) * sizeof(T);
    void* q = nullptr;
    cudaError_t e = cudaHostAlloc(&q, bytes, cudaHostAllocMapped);
    if (e != cudaSuccess) {
      cudaGetLastError();
      eu::set_error("cudaHostAlloc(%zu, mapped) -> %s", bytes, cudaGetErrorString(e));
      return EU_ERR_CUDA;
    }
    host_allocs.push_back(q);
    host_bytes += (int64_t)bytes;
    void* qd = nullptr;
    e = cudaHostGetDevicePointer(&qd, q, 0);
    if (e != cudaSuccess) { eu::set_error("cudaHostGetDevicePointer -> %s", cudaGetErrorString(e)); return EU_ERR_CUDA; }
    *host = (T*)q;
    *dev = (T*)qd;
    return EU_OK;
  }
};

// Device-resident engine state of one ctx.
struct EuRngState {
  uint32_t x;                 // minstd engine state
  uint32_t x_prev;             // engine state before the hop in flight (rows derive theirs from it)
  unsigned long long draws;   // uniforms produced since seed
  unsigned long long calls;   // philox: hop counter (salt)
  unsigned int blocks_done;   // last-block-done ticket
  unsigned int pad2;
  unsigned long long key;     // philox: per-engine key
};

struct eu_ctx {
  eu_graph* g = nullptr;
  eu_rng_kind rng = EU_RNG_MINSTD;
  uint64_t seed = 0;
  cudaStream_t stream = nullptr;
  EuRngState* d_rng = nullptr;       // [n_eng] engines; batch b of a batched call uses engine b, plain ops engine 0
  int n_eng = 1;
  // scratch (device), sized for `cap_rows` (padded) rows of the widest hop
  int64_t cap_rows = 0;
  eu::HashSlot* d_dedup = nullptr;   // two table sets of tab_set_slots slots each
  int64_t tab_set_slots = 0;
  int32_t* d_first = nullptr;        // [rows] first occurrence index of each seed
  int64_t* d_rowof = nullptr;        // [rows] graph row (valid where first==i), -1 if absent
  uint8_t* d_elig = nullptr;         // [rows]
  uint32_t* d_state = nullptr;       // [rows] engine state before the row's first draw (walks)
  uint32_t* d_emask = nullptr;       // [rows/32] eligible-first-occurrence ballots
  uint32_t* d_woff = nullptr;        // [rows/32] F^(count in earlier warps of the block)
  uint32_t* d_blkpre = nullptr;      // [rows/256] count in earlier blocks
  uint32_t* d_blkmul = nullptr;      // [rows/256] F^that count
  int32_t* d_live = nullptr;         // [rows] rows that draw (eligible first occurrences), compacted by k_prepare
  int32_t* d_dup = nullptr;          // [rows] eligible duplicates, compacted by k_prepare
  unsigned int* d_nlive = nullptr;   // [0]: rows in d_live, [1]: rows in d_dup
  unsigned long long* d_front[2] = {nullptr, nullptr};  // engine-id frontier ping-pong [rows]
  // segment dedup of the fused SAGE aggregation (mp_ops.cu), sized for agg_rows rows and agg_slots table slots
  int64_t agg_rows = 0, agg_slots = 0;
  unsigned long long* d_agg_tab = nullptr;  // [agg_slots] {hash bits, representative + 1}; all-free (0) between calls
  int32_t* d_agg_src = nullptr;      // [agg_rows] per row: itself (representative), its representative, or -1 (no neighbor)
  int32_t* d_agg_rep = nullptr;      // [agg_rows] representatives, compacted
  uint32_t* d_agg_slot = nullptr;    // [agg_rows] the table slot each representative claimed
  unsigned int* d_agg_nrep = nullptr;  // their number
  // extra scratch for walks / scatter
  void* d_misc = nullptr;
  int64_t misc_bytes = 0;
  float* d_walkv = nullptr;          // node2vec: biased weights of the big rows of one step (walk.cu)
  long long walkv_cap = 0;
  // node2vec: the three prefix kernels of a step (huge / big / small rows) are independent -> forked onto two auxiliary
  // streams and joined back (event fork/join: capturable in a CUDA graph)
  cudaStream_t aux[2] = {nullptr, nullptr};
  cudaEvent_t ev_fork = nullptr, ev_join[2] = {nullptr, nullptr};
  // pinned staging for *_host calls
  void* h_pin = nullptr;
  int64_t pin_bytes = 0;
  void* d_stage = nullptr;
  int64_t stage_bytes = 0;
  // optional per-kernel timing (eu_ctx_profile): CUDA events on the ctx stream around each kernel
  bool prof = false;
  struct ProfRec { const char* name; int64_t rows; cudaEvent_t e0, e1; };
  std::vector<ProfRec> prof_recs;
};

// RAII-free helper: EU_PROF(c, "name", rows) { launch; }  records events around the launch when profiling
struct EuProfScope {
  eu_ctx* c; size_t idx;
  EuProfScope(eu_ctx* c_, const char* name, int64_t rows) : c(c_), idx((size_t)-1) {
    if (!c->prof) return;
    eu_ctx::ProfRec r{name, rows, nullptr, nullptr};
    cudaEventCreate(&r.e0); cudaEventCreate(&r.e1);
    cudaEventRecord(r.e0, c->stream);
    c->prof_recs.push_back(r);
    idx = c->prof_recs.size() - 1;
  }
  ~EuProfScope() { if (idx != (size_t)-1) cudaEventRecord(c->prof_recs[idx].e1, c->stream); }
};

namespace eu {
// Rows from which a launch looks for repeated work (sampler: duplicate seeds copy their first occurrence's draws; fused SAGE
// aggregation: each distinct segment is reduced once).  The extra passes have a fixed cost -- a launch and a latency-bound
// classification -- that only a large hop repays: a fanout's repeats sit in its deeper hops, where a seed's draws with
// replacement come back as seeds (headline step on an H100: 69 % of the live hop-2 rows repeat; its 32K-row first hop and
// the 64K-row hops of the heterogeneous config are slower with the extra passes).
static constexpr int64_t kRepeatMinRows = (int64_t)1 << 17;
int ctx_reserve(eu_ctx* c, int64_t rows, int64_t table_slots);
int64_t hop_scratch_rows(int nb, int64_t rows_b);
int64_t hop_table_slots(int nb, int64_t rows_b);
int64_t hop_table_cap(int64_t rows_b);   // dedup slots per batch (region stride = cap + 1)
int ctx_misc(eu_ctx* c, int64_t bytes);
inline size_t a256(size_t b) { return (b + 255) & ~(size_t)255; }   // scratch offsets: 256-byte aligned
struct EdgeOrder;   // segment.cuh
// gat.cu (shared with relation.cu): out[r, :] = sum of w[e] * rows[row_e, :] over the edges of segment r of the order o, in
// edge order (k_gat_bwd_src, H = 1); a segment without edges gets a zero row
int segmented_row_sum(eu_ctx* c, const float* rows, const float* w, const EdgeOrder& o, const int32_t* row, int64_t E, int64_t n,
                      int dim, float* out);
// features.cu: ptr i64[M + 1] = the entry offsets of get_sparse_feature's CSR over slot fid (a node without values counts one
// default entry), with tmp (>= ragged_scan_bytes(M) bytes) as the scan scratch; no host synchronisation
size_t ragged_scan_bytes(int64_t M);
int sparse_entry_ptr(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, void* tmp, size_t tmp_bytes, int64_t* ptr);
int agg_reserve(eu_ctx* c, int64_t rows, int64_t table_slots);   // the fused SAGE aggregation's dedup scratch
int refuse_growth_in_capture(eu_ctx* c, const char* what);   // EU_ERR_STATE if the ctx stream is being captured
int graph_build_sampler(eu_graph* g);
// graph.cu: *st = the storage descriptor `in` (null: f32 in HBM) once it is valid for a table of n rows; else EU_ERR_INVALID /
// EU_ERR_UNSUPPORTED naming `who`, before anything is allocated
int feat_storage_check(const eu_feat_storage* in, int64_t n, const char* who, eu_feat_storage* st);
int graph_build_labels(eu_graph* g);   // graph_label.cu: the label table (EU_ERR_STATE without a graph_label slot)
// graph_label.cu: Graph::GetGraphLabel's list (graph.cc:439-457) from the binary slot `fid` (S slots per row) of the rows
// visited in node_map_ order (`order`, empty = row order); row_label (may be null) gets each row's label index, or L for a
// row without a value (the empty label lists no nodes)
void graph_label_list(const std::vector<int64_t>& order, int64_t n, const int64_t* bin_ptr, const uint8_t* bin_val, int32_t S,
                      int32_t fid, std::vector<std::string>* labels, std::vector<int32_t>* row_label);
// sample.cu: the engine after `uniforms` draws of a plain op (both modes: the Philox salt advances too)
__global__ void k_advance_engine(EuRngState* rng, unsigned long long uniforms);
// sample.cu: stats[0] = ptr[rows], stats[1] = the longest row of the CSR ptr; stats zeroed by the caller
__global__ void k_ragged_stats(const long long* __restrict__ ptr, int64_t rows, long long* __restrict__ stats);
// gat.cu: dot[e] = <a[ia_e], b[ib_e]> in k_agnn_dot's fixed order over E > 0 pairs (ia null = the identity), scaled[e] =
// beta * dot[e]; either output may be null
int agnn_dot(eu_ctx* c, const float* a, const float* b, const int32_t* ia, const int32_t* ib, int64_t E, int dim,
             const float* beta, float* dot, float* scaled);
int get_node_weight(eu_ctx* c, const int64_t* nodes, int64_t B, float* out);   // neighbor.cu, for eu_get_node_weight_host
int launch_state_scan(eu_ctx* c, int64_t rows, unsigned long long uniforms_per_row);
// one sampleNB hop (sample.cu): seeds u64[rows] -> engine ids u64[rows*count] (0 placeholders, may be
// null) and TF-packed outputs (may be null)
int hop(eu_ctx* c, const unsigned long long* seeds, int64_t rows, const int32_t* etypes, int32_t K,
        int32_t count, int64_t default_node, unsigned long long* eng_ids, int64_t* out_ids,
        float* out_w, int32_t* out_t, int hop_index, bool pre_inserted, bool insert_next, int nb,
        const int32_t* rows_act = nullptr, bool raw = false);
}  // namespace eu
