/* euler_b200 -- C ABI of the H100-native minibatch-construction path of alibaba/euler.
 *
 * This is the drop-in boundary (SURVEY.md section 8b, seam B2).  The reference exports exactly one
 * C symbol, `bool InitQueryProxy(const char*)` (tf_euler/utils/init_query_proxy.cc:19-36); every
 * other entry point of the hot path is a TensorFlow op registered in C++.  Since TF's registry is
 * not part of this build, each TF op of the path is exported here as a flat function with the
 * op's own argument meaning; the reference-side binding a maintainer would add is shown in
 * INTEGRATION.md.  Plain pointers and sizes only -- no torch / TF types.
 *
 * Conventions
 *   - every function returns 0 (EU_OK) or a nonzero eu_status; nothing throws across the ABI;
 *   - `eu_ctx` = one execution lane: a CUDA stream + one RNG engine + scratch.  It plays the role of
 *     one thread of the reference's client pool (euler/client/query_proxy.cc:205-210: 8 threads,
 *     each with its own thread_local engine, euler/common/random.cc:22).  Calls on one ctx are
 *     stream-ordered; different ctxs may run concurrently; the graph is immutable after creation;
 *   - functions without a `_host` suffix take DEVICE pointers and only enqueue work on the ctx
 *     stream (no host synchronisation, capturable in a CUDA graph);
 *   - `_host` variants take HOST pointers and return after the results have landed (this is what a
 *     CPU-tensor framework binds): pageable buffers are staged through pinned memory owned by the ctx,
 *     buffers that are already page-locked (cudaHostAlloc / cudaHostRegister) are DMA'd in place;
 *   - edge-type / count lists are HOST arrays (they are op attributes / tiny tensors upstream).
 */
#ifndef EULER_B200_H_
#define EULER_B200_H_

#include <stdbool.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  EU_OK = 0,
  EU_ERR_INVALID = 1,      /* bad argument */
  EU_ERR_CUDA = 2,         /* a CUDA call failed; see eu_last_error() */
  EU_ERR_NO_GPU = 3,       /* no CUDA device: this library has no CPU fallback */
  EU_ERR_UNSUPPORTED = 4,  /* valid in the reference but outside this path (e.g. `condition`) */
  EU_ERR_IO = 5,
  EU_ERR_STATE = 6         /* e.g. op called before a graph was initialised */
} eu_status;

/* RNG engines.  EU_RNG_MINSTD reproduces the reference's engine and draw order bit-exactly
 * (std::default_random_engine + uniform_real_distribution<double>, euler/common/random.cc:22-28);
 * EU_RNG_PHILOX is a counter-based engine keyed on (node id, draw) for throughput runs: same
 * algorithm, same distribution, different stream. */
typedef enum { EU_RNG_MINSTD = 0, EU_RNG_PHILOX = 1 } eu_rng_kind;

typedef struct eu_graph eu_graph;
typedef struct eu_ctx eu_ctx;

const char* eu_last_error(void);
const char* eu_version(void);
/* number of kernels this library has launched in this process (bench.py's gpu_launches) */
uint64_t eu_launch_count(void);

/* ------------------------------------------------------------------ graph -------------------- */
/* CSR description, HOST arrays.  Mirrors what a reference Node holds (euler/core/graph/node.h:49-57,
 * node.cc:37-96): for row r and edge type t the adjacency group is
 *   [grp_ptr[r*T+t], grp_ptr[r*T+t+1])  -- neighbor_groups_idx, made global;
 * cum_w is the NODE-GLOBAL cumulative f32 weight exactly as stored (node.cc:59-65); grp_cum[r*T+t] is
 * edge_group_collection.sum_weights_[t].  If cum_w == NULL, `w` (raw weights) must be given and the
 * prefix sums are accumulated the way Node::Init does (sequential f32, eu_graph builds them). */
typedef struct {
  int64_t n_nodes;
  int32_t n_edge_types;    /* T */
  int32_t n_node_types;
  const uint64_t* ids;     /* [n] node id of each row; id 0 is unusable (DEFAULT_UINT64) */
  const int32_t* node_type;/* [n] or NULL (all 0) */
  const float* node_w;     /* [n] or NULL (all 1.0) */
  const int64_t* grp_ptr;  /* [n*T+1] */
  const uint64_t* nbr;     /* [E] */
  const float* cum_w;      /* [E] or NULL */
  const float* grp_cum;    /* [n*T] or NULL (required iff cum_w given and T > 1) */
  const float* w;          /* [E] raw weights, used iff cum_w == NULL */
  int32_t feat_dim;        /* dense f32 feature slot 0: row length, 0 = none */
  const float* feat;       /* [n*feat_dim] or NULL */
  const int64_t* sampler_order; /* [n] rows in the order the global node sampler enumerates them
                                   (graph.cc:349-354 uses unordered_map order); NULL = row order */
  /* optional: several dense f32 feature slots (Node::float_features_idx_, node.h); when
   * n_feat_slots > 0, feat is [n, sum(feat_slot_dims)] and feat_dim must equal that sum */
  int32_t n_feat_slots;
  const int32_t* feat_slot_dims;
  /* optional ragged features (Node::uint64_features_ / binary_features_, euler/core/graph/node.h): slot s of row r is
   * [ptr[r*S+s], ptr[r*S+s+1]) of the value array; S = 0 / NULL = none */
  int32_t n_u64_slots;
  const int64_t* u64_ptr;   /* [n*S+1] */
  const uint64_t* u64_val;
  int32_t n_bin_slots;
  const int64_t* bin_ptr;   /* [n*S+1] */
  const uint8_t* bin_val;
} eu_graph_desc;

int eu_graph_create(const eu_graph_desc* desc, int device, eu_graph** out);
/* Storage type of the dense node feature table.  Every graph constructor stores f32; its *_dtype sibling takes one of
 * these.  EU_FEAT_BF16 halves the table: each value is rounded to bfloat16 on the device (round to nearest even; NaN
 * becomes a canonical NaN, +-Inf stays, a finite value becomes +-Inf only where the rounding says so), and every op that
 * reads dense node features widens it exactly to f32, so its output is bit for bit the f32 op's on the rounded table.
 * Host f32 arrays go up in bounded chunks and are rounded on the device: the peak is the bf16 table plus one chunk.  Edge
 * features and ragged features are not affected.  An unknown dtype: EU_ERR_INVALID before any allocation.  The sharded
 * feature paths (eu_sym_get_dense_feature, eu_sym_sage_mean) refuse a bf16 graph with EU_ERR_UNSUPPORTED. */
typedef enum { EU_FEAT_F32 = 0, EU_FEAT_BF16 = 1 } eu_feat_dtype;
int eu_graph_create_dtype(const eu_graph_desc* desc, int device, int32_t feat_dtype, eu_graph** out);
/* Synthetic R-MAT graph generated, sorted and prefix-summed on the device (SURVEY.md section 8d "G-RMAT"):
 * ids 1..n, one node/edge type, n_edges directed edges with (a,b,c,d), adjacency sorted by dst,
 * weight = 1 + (hash(src,dst) % 100) / 10, feat ~ U(-1,1).  feat_dim may be 0. */
int eu_graph_create_rmat(int64_t n_nodes, int64_t n_edges, double a, double b, double c,
                         uint64_t seed, int32_t feat_dim, uint64_t feat_seed, int device,
                         eu_graph** out);
/* The rows of that same graph that shard `shard_index` of `shard_number` owns: owner(id) = id % shard_number
 * (the reference's routing (id % partitions) % shards with partitions a multiple of shards,
 * euler/core/kernels/id_split_op.cc:46-49).  The union of the shards is exactly eu_graph_create_rmat's graph. */
int eu_graph_create_rmat_shard(int64_t n_nodes, int64_t n_edges, double a, double b, double c,
                               uint64_t seed, int32_t feat_dim, uint64_t feat_seed, int device,
                               int shard_index, int shard_number, eu_graph** out);
/* Heterogeneous variant (BASELINE configs[4]): edge type = hash(edge) % n_edge_types (adjacency grouped by
 * (row, type), one node-global cumulative weight array as node.cc:59-65), node type = id % n_node_types. */
int eu_graph_create_rmat_hetero(int64_t n_nodes, int64_t n_edges, int32_t n_edge_types, int32_t n_node_types, double a,
                                double b, double c, uint64_t seed, int32_t feat_dim, uint64_t feat_seed, int device,
                                int shard_index, int shard_number, eu_graph** out);
/* The three R-MAT constructors with the feature table's storage type (eu_feat_dtype); a bf16 table holds the f32 values
 * above, rounded on the device. */
int eu_graph_create_rmat_dtype(int64_t n_nodes, int64_t n_edges, double a, double b, double c, uint64_t seed, int32_t feat_dim,
                               uint64_t feat_seed, int device, int32_t feat_dtype, eu_graph** out);
int eu_graph_create_rmat_shard_dtype(int64_t n_nodes, int64_t n_edges, double a, double b, double c, uint64_t seed,
                                     int32_t feat_dim, uint64_t feat_seed, int device, int shard_index, int shard_number,
                                     int32_t feat_dtype, eu_graph** out);
int eu_graph_create_rmat_hetero_dtype(int64_t n_nodes, int64_t n_edges, int32_t n_edge_types, int32_t n_node_types, double a,
                                      double b, double c, uint64_t seed, int32_t feat_dim, uint64_t feat_seed, int device,
                                      int shard_index, int shard_number, int32_t feat_dtype, eu_graph** out);
/* Where the dense node feature table lives.  EU_FEAT_DEVICE (every constructor above): in HBM.  EU_FEAT_HOST: the whole table
 * [n, feat_dim] sits in mapped pinned host memory (cudaHostAllocMapped) and kernels read it in place over the host link;
 * cache_rows = C (0 <= C <= n) rows are also copied once, at build time, into an HBM cache [C, feat_dim], and an int32 slot map
 * [n] in HBM sends each row to its cache row or to -1.  The cached rows are the C first by (in-degree descending, row
 * ascending), where a row's in-degree counts the adjacency entries, over all rows and edge types, whose neighbour id is that
 * row's (ids without a row count for nothing).  Row r is read from the cache when its slot is >= 0 and from the host table
 * otherwise; both hold the same bits (the table is never written after the build), so every op's output is bit for bit the
 * one it gives on the same graph held in HBM, whatever C is.  The storage type rules above hold for both places: a bf16 host
 * table is rounded on the device.
 * Refusals, before any allocation: an unknown dtype or place, C < 0, C > n, or C > 0 with EU_FEAT_DEVICE: EU_ERR_INVALID; a
 * host table of 2^31 rows or more: EU_ERR_UNSUPPORTED.  A failed pinned allocation returns EU_ERR_CUDA and frees what was
 * allocated.  The sharded feature paths (eu_sym_get_dense_feature, eu_sym_sage_mean) refuse a host-placed graph with
 * EU_ERR_UNSUPPORTED, as they refuse bf16.  A NULL storage descriptor is {EU_FEAT_F32, EU_FEAT_DEVICE, 0}. */
typedef enum { EU_FEAT_DEVICE = 0, EU_FEAT_HOST = 1 } eu_feat_place;
typedef struct {
  int32_t dtype;        /* eu_feat_dtype */
  int32_t place;        /* eu_feat_place */
  int64_t cache_rows;   /* rows cached in HBM; 0 unless place is EU_FEAT_HOST */
} eu_feat_storage;
int eu_graph_create_storage(const eu_graph_desc* desc, int device, const eu_feat_storage* storage, eu_graph** out);
int eu_graph_create_rmat_storage(int64_t n_nodes, int64_t n_edges, double a, double b, double c, uint64_t seed,
                                 int32_t feat_dim, uint64_t feat_seed, int device, const eu_feat_storage* storage,
                                 eu_graph** out);
int eu_graph_create_rmat_hetero_storage(int64_t n_nodes, int64_t n_edges, int32_t n_edge_types, int32_t n_node_types,
                                        double a, double b, double c, uint64_t seed, int32_t feat_dim, uint64_t feat_seed,
                                        int device, int shard_index, int shard_number, const eu_feat_storage* storage,
                                        eu_graph** out);
/* Euler 2.0 on-disk format (euler.meta + the Node and Edge partition files; SURVEY.md Appendix B), shard `shard_index` of
 * `shard_number` with the reference's file filter (graph.cc:90-98).  = Graph::Init, graph.h:53-56. */
int eu_graph_load(const char* data_path, int shard_index, int shard_number, int device,
                  eu_graph** out);
/* load_edges = 0: node data only (Graph::Init's load_data_type "node"); eu_graph_load = load_edges 1 ("all"): the Edge
 * files, when the directory has them, feed eu_sample_edge and the edge feature ops. */
int eu_graph_load_ex(const char* data_path, int shard_index, int shard_number, int device, int load_edges,
                     eu_graph** out);
/* eu_graph_load_ex with the node feature table's storage type (eu_feat_dtype) */
int eu_graph_load_dtype(const char* data_path, int shard_index, int shard_number, int device, int load_edges,
                        int32_t feat_dtype, eu_graph** out);
/* eu_graph_load_ex with the node feature table's storage descriptor (eu_feat_storage) */
int eu_graph_load_storage(const char* data_path, int shard_index, int shard_number, int device, int load_edges,
                          const eu_feat_storage* storage, eu_graph** out);
/* Edge records (Edge files of the Euler format; euler/core/graph/edge.h): needed only by sample_edge and the edge feature ops.
 * HOST arrays; features use the node layout (dense slots concatenated per edge, ragged uint64 / binary slots).
 * sampler_order: edge rows in the order the reference's edge_map_ iterates (graph.cc:372-399); NULL = row order. */
typedef struct {
  int64_t n_edges;
  const uint64_t* src;      /* [nE] */
  const uint64_t* dst;      /* [nE] */
  const int32_t* type;      /* [nE] */
  const float* w;           /* [nE] or NULL (all 1.0) */
  int32_t feat_dim;         /* total dense width, 0 = none */
  const float* feat;        /* [nE * feat_dim] */
  int32_t n_feat_slots;     /* 0 = one slot of feat_dim */
  const int32_t* feat_slot_dims;
  int32_t n_u64_slots; const int64_t* u64_ptr; const uint64_t* u64_val;
  int32_t n_bin_slots; const int64_t* bin_ptr; const uint8_t* bin_val;
  const int64_t* sampler_order;
} eu_edge_desc;
int eu_graph_set_edges(eu_graph* g, const eu_edge_desc* desc);
int64_t eu_graph_num_edge_records(const eu_graph* g);
int32_t eu_graph_edge_dense_feature_id(const eu_graph* g, const char* name);
/* Rename dense edge slot fid (eu_graph_set_edges names them feat0, feat1, ...), e.g. to 'id' for the knowledge-graph models'
 * relation ids.  EU_ERR_INVALID for an unknown slot. */
int eu_graph_set_edge_dense_feature_name(eu_graph* g, int32_t fid, const char* name);
int32_t eu_graph_edge_sparse_feature_id(const eu_graph* g, const char* name);
int32_t eu_graph_edge_binary_feature_id(const eu_graph* g, const char* name);
int eu_graph_destroy(eu_graph* g);
int64_t eu_graph_num_nodes(const eu_graph* g);
int64_t eu_graph_num_edges(const eu_graph* g);
int32_t eu_graph_num_edge_types(const eu_graph* g);
/* Host-only (no GPU needed): parse an Euler 2.0 data directory exactly as eu_graph_load does -- same file filter, same record
 * decoding, same replay of the reference's node_map_ iteration order (euler/core/graph/graph.cc:349-354) -- and report what would
 * be uploaded: counts and, for the first `cap` entries, node ids and types in GLOBAL SAMPLER ORDER.  Any out pointer may be NULL. */
int eu_graph_load_inspect(const char* data_path, int shard_index, int shard_number, int64_t* n_nodes, int64_t* n_edges,
                          int32_t* n_edge_types, int32_t* n_node_types, int64_t cap, int64_t* order_ids, int32_t* order_types);
/* Host-only helper (no GPU needed): the sampler tables eu_graph_create / eu_graph_load build for the global node and edge samplers --
 * FastWeightedCollection::Init + AliasMethod::Init (euler/common/fast_weighted_collection.h:54-74, alias_method.cc:23-63):
 * weights f32[n] -> prob f32[n], alias i32[n], *sum = the f32 weight sum.  Exposed so the tables can be checked bit for bit
 * against the reference's without a device. */
int eu_build_alias_table(const float* weights, int64_t n, float* prob, int32_t* alias, float* sum);
int32_t eu_graph_num_node_types(const eu_graph* g);
int32_t eu_graph_feat_dim(const eu_graph* g);
/* the eu_feat_dtype of the dense node feature table; -1 for a NULL graph */
int32_t eu_graph_feat_dtype(const eu_graph* g);
/* the eu_feat_place of the dense node feature table, and the rows its HBM cache holds; -1 for a NULL graph */
int32_t eu_graph_feat_place(const eu_graph* g);
int64_t eu_graph_feat_cache_rows(const eu_graph* g);
/* device bytes the graph holds (a bf16 feature table counts 2 bytes per element; a host-placed table counts only its cache
 * and slot map) */
int64_t eu_graph_hbm_bytes(const eu_graph* g);
/* pinned host bytes the graph holds: the host-placed feature table, 0 otherwise; -1 for a NULL graph */
int64_t eu_graph_host_bytes(const eu_graph* g);
/* Copy the feature rows' cache slots to the HOST array slots[n]: a row's HBM cache row, or -1.  A device-placed table has no
 * cache: every slot is -1. */
int eu_graph_export_feat_slots(const eu_graph* g, int32_t* slots);
/* Copy the device CSR back to caller-allocated HOST arrays (any pointer may be NULL).  feat is f32 whatever the table's
 * storage type: a bf16 table comes back widened, exactly. */
int eu_graph_export(const eu_graph* g, uint64_t* ids, int32_t* node_type, float* node_w,
                    int64_t* grp_ptr, uint64_t* nbr, float* cum_w, float* grp_cum, float* feat);
/* type-name lookup from euler.meta (tf_euler/python/euler_ops/type_ops.py:31-64); -1 if unknown */
int32_t eu_graph_edge_type_id(const eu_graph* g, const char* name);
int32_t eu_graph_node_type_id(const eu_graph* g, const char* name);
/* dense feature slot of feature `name` (looked up as "dense_"+name like get_dense_feature_op.cc:83);
 * -1 if unknown.  eu_graph_dense_feature_dim: stored width of a slot. */
int32_t eu_graph_dense_feature_id(const eu_graph* g, const char* name);
int32_t eu_graph_dense_feature_dim(const eu_graph* g, int32_t fid);
/* slots of the uint64 ("sparse_"+name, get_sparse_feature_op.cc:75) and binary ("binary_"+name) features; -1 if unknown */
int32_t eu_graph_sparse_feature_id(const eu_graph* g, const char* name);
int32_t eu_graph_binary_feature_id(const eu_graph* g, const char* name);

/* ------------------------------------------------------------------ contexts ----------------- */
/* stream: a cudaStream_t (NULL = legacy default stream). */
int eu_ctx_create(eu_graph* g, eu_rng_kind rng, uint64_t seed, void* stream, eu_ctx** out);
int eu_ctx_destroy(eu_ctx* c);
int eu_ctx_set_stream(eu_ctx* c, void* stream);
int eu_ctx_seed(eu_ctx* c, uint64_t seed);           /* engine e <- seed + e; stream-ordered */
/* A ctx may carry several engines: batch b of a *_batched call runs on engine b (its own draw stream and
 * its own dedup scope), i.e. each batch is exactly one reference op call on one client thread; batching only
 * shares kernel launches.  seeds == NULL: engine e <- seed + e.  Plain ops use engine 0. */
int eu_ctx_set_engines(eu_ctx* c, int32_t n, const uint64_t* seeds);
int eu_ctx_reserve(eu_ctx* c, int64_t max_rows);      /* pre-size scratch (required before graph capture) */
int eu_ctx_sync(eu_ctx* c);
/* number of uniforms the MINSTD engine has produced since the last seed (synchronises) */
int eu_ctx_draws(eu_ctx* c, uint64_t* draws);
/* Per-kernel timing: while enabled, every kernel this ctx launches is bracketed by CUDA events on the
 * ctx stream.  eu_ctx_profile_read synchronises and returns "name,rows,launches,total_ms" lines. */
int eu_ctx_profile(eu_ctx* c, int enable);
int eu_ctx_profile_read(eu_ctx* c, char* buf, int64_t cap);

/* ------------------------------------------------------------------ sampling ops ------------- */
/* tf_euler.sample_neighbor -- TF op SampleNeighbor (tf_euler/ops/neighbor_ops.cc:138-163, kernel
 * tf_euler/kernels/sample_neighbor_op.cc:54-129).  nodes i64[B]; etypes i32[K] (host);
 * outputs [B,count]: ids i64 (default_node fill), w f32 (0 fill), t i32 (-1 fill). */
int eu_sample_neighbor(eu_ctx* c, const int64_t* nodes, int64_t B, const int32_t* etypes, int32_t K,
                       int32_t count, int64_t default_node, int64_t* out_ids, float* out_w,
                       int32_t* out_t);
int eu_sample_neighbor_host(eu_ctx* c, const int64_t* nodes, int64_t B, const int32_t* etypes,
                            int32_t K, int32_t count, int64_t default_node, int64_t* out_ids,
                            float* out_w, int32_t* out_t);
/* euler::SampleNeighbor of the C++ api (euler/core/api/api.cc:223-236): one Node::SampleNeighbor per element of `nodes`,
 * in order, WITHOUT the engine's unique/gather rule -- a repeated id draws again.  Engine-form outputs [B,count]: rows
 * without a result (absent node / no edge of the requested types) are (0, 0.0, -1).  Exact-RNG contexts only. */
int eu_sample_neighbor_raw(eu_ctx* c, const int64_t* nodes, int64_t B, const int32_t* etypes, int32_t K,
                           int32_t count, int64_t* out_ids, float* out_w, int32_t* out_t);
int eu_sample_neighbor_raw_host(eu_ctx* c, const int64_t* nodes, int64_t B, const int32_t* etypes, int32_t K,
                                int32_t count, int64_t* out_ids, float* out_w, int32_t* out_t);
/* tf_euler.sample_fanout -- TF op SampleFanout (tf_euler/ops/neighbor_ops.cc:228-280, kernel
 * tf_euler/kernels/sample_fanout_op.cc:60-145).  etypes i32[L,K] (host), counts i32[L] (host);
 * out_*[l] point to B*prod(counts[0..l]) elements.  The frontier never leaves the device. */
int eu_sample_fanout(eu_ctx* c, const int64_t* nodes, int64_t B, const int32_t* etypes, int32_t K,
                     const int32_t* counts, int32_t L, int64_t default_node, int64_t* const* out_ids,
                     float* const* out_w, int32_t* const* out_t);
/* nb independent batches of B seeds in one set of launches (nodes / outputs batch-major). */
int eu_sample_fanout_batched(eu_ctx* c, const int64_t* nodes, int32_t nb, int64_t B, const int32_t* etypes, int32_t K,
                             const int32_t* counts, int32_t L, int64_t default_node, int64_t* const* out_ids,
                             float* const* out_w, int32_t* const* out_t);
int eu_sample_fanout_host(eu_ctx* c, const int64_t* nodes, int64_t B, const int32_t* etypes,
                          int32_t K, const int32_t* counts, int32_t L, int64_t default_node,
                          int64_t* const* out_ids, float* const* out_w, int32_t* const* out_t);
int eu_sample_fanout_batched_host(eu_ctx* c, const int64_t* nodes, int32_t nb, int64_t B, const int32_t* etypes,
                                  int32_t K, const int32_t* counts, int32_t L, int64_t default_node,
                                  int64_t* const* out_ids, float* const* out_w, int32_t* const* out_t);
/* tf_euler.sample_fanout_with_feature -- TF op SampleFanoutWithFeature (tf_euler/kernels/sample_fanout_with_feature_op.cc:95-275,
 * wrapper neighbor_ops.py:49-69): eu_sample_fanout's hops -- the same draws, outputs and draw count on the same ctx state --
 * followed by the features of every hop.  counts i32[L] >= 1 (host).  out_ids / out_w / out_t[l] as eu_sample_fanout
 * (B*prod(counts[0..l]) elements, TF-packed); eng_ids[l] i64[same] receives hop l's ENGINE ids (0 = DEFAULT_UINT64 where a row
 * was filled), from which the features are taken as the reference's v_select(nb_l) does: a row whose first draw is node 0 is
 * packed as default_node but has the features of its real draws.  Hop 0's features are those of `nodes`.  Hop-major, hop l
 * and feature j at index l * n + j of the (L+1) * n outputs:
 *   out_dense   f32[rows_l, dense_dims[j]]   eu_get_dense_feature of slot dense_fids[j]
 *   sparse_ptr  i64[rows_l + 1]              eu_get_sparse_feature's offsets of slot sparse_fids[j] (one default entry per node
 *                                            without values); sparse_total / sparse_max_len (HOST) its entry count and longest row
 * The values are then written by eu_get_sparse_feature(c, ids_l, rows_l, fid, default, sparse_total[k], sparse_ptr[k], values)
 * with ids_l = nodes or eng_ids[l - 1] (no synchronisation).  Device pointers except the lists and the host arrays; the call
 * synchronises the stream once when n_sparse > 0 (every total and longest row together), never otherwise. */
int eu_sample_fanout_with_feature(eu_ctx* c, const int64_t* nodes, int64_t B, const int32_t* etypes, int32_t K, const int32_t* counts,
                                  int32_t L, int64_t default_node, int64_t* const* out_ids, float* const* out_w, int32_t* const* out_t,
                                  int64_t* const* eng_ids, int32_t n_dense, const int32_t* dense_fids, const int32_t* dense_dims,
                                  float* const* out_dense, int32_t n_sparse, const int32_t* sparse_fids, int64_t* const* sparse_ptr,
                                  int64_t* sparse_total, int64_t* sparse_max_len);
/* eu_sample_fanout_with_feature with every out_dense[k] of dense_dtype (an eu_feat_dtype code; the rule of
 * eu_get_dense_feature_out_dtype).  The hops, weights, types, engine ids, sparse outputs and the draws the engine consumes are
 * exactly the f32 call's.  An unknown dense_dtype: EU_ERR_INVALID before any draw or write. */
int eu_sample_fanout_with_feature_out_dtype(eu_ctx* c, const int64_t* nodes, int64_t B, const int32_t* etypes, int32_t K,
                                            const int32_t* counts, int32_t L, int64_t default_node, int64_t* const* out_ids,
                                            float* const* out_w, int32_t* const* out_t, int64_t* const* eng_ids, int32_t n_dense,
                                            const int32_t* dense_fids, const int32_t* dense_dims, int32_t dense_dtype,
                                            void* const* out_dense, int32_t n_sparse, const int32_t* sparse_fids,
                                            int64_t* const* sparse_ptr, int64_t* sparse_total, int64_t* sparse_max_len);
/* tf_euler.sample_node -- TF op SampleNode (tf_euler/ops/sample_ops.cc:22-37, kernel
 * tf_euler/kernels/sample_node_op.cc:39-96; euler::SampleNode api.cc:32-37).  types i32[n_types]
 * (host); a single -1 means all types.  out i64[count]. */
int eu_sample_node(eu_ctx* c, int32_t count, const int32_t* types, int32_t n_types, int64_t* out);
int eu_sample_node_host(eu_ctx* c, int32_t count, const int32_t* types, int32_t n_types,
                        int64_t* out);
/* tf_euler.sample_n_with_types -- TF op SampleNWithTypes (tf_euler/kernels/sample_n_with_types_op.cc, engine op
 * euler/core/kernels/sample_n_with_types_op.cc): row i of out i64[n, count] is SampleNode({types[i]}, count), the rows drawn
 * in order from the ctx's one engine (Graph::SampleNode(int, count), graph.cc:221-245: 2 uniforms per draw).  Under
 * EU_RNG_MINSTD row i's draw j starts at uniform 2 (i count + j) of the call, and the engine then advances by 2 n count
 * uniforms, so a following sampling op continues the reference's stream; EU_RNG_PHILOX keys draw (i, j) on the call counter.
 * types i32[n] and out are device pointers.  Refused, with out and the engine untouched: a row whose type is INT32_MIN (its
 * source is not a node, as eu_get_node_type reports it) or outside [0, n_node_types) -> EU_ERR_INVALID (upstream indexes
 * node_samplers_ with it); a type whose total node weight is 0 -> EU_ERR_STATE (upstream aborts on the short result).  The
 * check is read back in the call's one stream synchronisation.  n = 0 or count = 0 returns at once. */
int eu_sample_n_with_types(eu_ctx* c, const int32_t* types, int64_t n, int32_t count, int64_t* out);
/* tf_euler.random_walk -- TF op RandomWalk (tf_euler/ops/walk_ops.cc:77-107, kernel
 * tf_euler/kernels/random_walk_op.cc:83-289).  etypes i32[L,K] (host); out i64[B,L+1].
 * EU_RNG_MINSTD: the reference's walks bit for bit (serial engine stream, sequential f32 prefix of the biased weights).
 * EU_RNG_PHILOX with one edge type per step on sorted adjacency: node2vec steps by rejection sampling (propose from the
 * stored CDF, accept with bias / max bias) -- the same transition distribution at O(log deg) per step. */
int eu_random_walk(eu_ctx* c, const int64_t* nodes, int64_t B, const int32_t* etypes, int32_t K,
                   int32_t L, float p, float q, int64_t default_node, int64_t* out);
int eu_random_walk_host(eu_ctx* c, const int64_t* nodes, int64_t B, const int32_t* etypes,
                        int32_t K, int32_t L, float p, float q, int64_t default_node, int64_t* out);
/* tf_euler.get_dense_feature, one feature -- TF op GetDenseFeature (tf_euler/ops/feature_ops.cc:94-140,
 * kernel tf_euler/kernels/get_dense_feature_op.cc:63-121).  out f32[M,dim], zero fill. */
int eu_get_dense_feature(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int32_t dim,
                         float* out);
int eu_get_dense_feature_host(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int32_t dim,
                              float* out);
/* Output dtype of the graph-feature ops.  Each *_out_dtype twin below takes an eu_feat_dtype code `out_dtype` and an output
 * `void* out` of that element type (f32 or bf16, same shape as the f32 call), and is otherwise its f32 sibling: same
 * arguments, statuses and synchronisation (the device twins never synchronise the host and are capturable).
 * Exactness: with out_dtype = EU_FEAT_BF16 the output is, bit for bit, the f32 call's output converted on the device
 * (torch's .to(torch.bfloat16) of it): every value is computed in f32 exactly as the f32 call computes it (sums and
 * divisions included) and rounded once, at the store, to nearest even -- NaN becomes the canonical NaN, +-Inf stays, a
 * finite value becomes +-Inf only where the rounding says so, and subnormals round like any other value.  This holds for
 * either table dtype, either placement and any cache size.  On a bf16 table, eu_get_dense_feature_out_dtype and the rows of
 * eu_neighbor_top_k_feature_out_dtype return the stored bits unchanged.  Every output offset is 64-bit: a bf16 output may
 * pass 2^31 elements.  An unknown out_dtype: EU_ERR_INVALID ("<entry point>: unknown output dtype <code> (EU_FEAT_F32 or
 * EU_FEAT_BF16)") before anything is enqueued or written.  The _host twins stage out_dtype-sized elements; their buffers may
 * be pageable or page-locked as for every _host call.  The sharded entry points have no twin. */
int eu_get_dense_feature_out_dtype(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int32_t dim, int32_t out_dtype, void* out);
int eu_get_dense_feature_host_out_dtype(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int32_t dim, int32_t out_dtype,
                                        void* out);
/* LGCEncoder's input block (tf_euler/python/utils/encoders.py:895-922, "Large-Scale Learnable Graph Convolutional
 * Networks"), fused from the ids: nodes i64[B], neighbors i64[B, count] (sample_neighbor's rows), out f32[B, k + 1, dim]:
 *   out[b, 0, :]      = eu_get_dense_feature(nodes[b], fid, dim) exactly (zeros past the slot's stored width, clipped before
 *                       it, a zero row for an absent id or an unknown slot)
 *   out[b, 1 + j, d]  = for j < k, the j-th largest of the count values feature(neighbors[b, i])[d], each read under the same
 *                       rule (an absent neighbour, such as sample_neighbor's -1, gives 0.0), in descending order.
 * Ties: equal values keep the lower neighbour index first, tf.nn.top_k's rule (TF's TopKV2), so +0.0 / -0.0 ties are
 * determined to the bit; NaN ranks above every number (torch.sort's order), NaNs among themselves by index.  The result is
 * bit-exact against a stable descending sort of the fetched rows.  No [B, count, dim] intermediate; no host
 * synchronisation and no scratch: capturable in a CUDA graph.  No backward pass (the input is graph data).
 * k < 1 or k > count (tf.nn.top_k refuses k above the row length): EU_ERR_INVALID; k above EU_NEIGHBOR_TOP_K_MAX (each
 * column's k candidates are held in registers): EU_ERR_UNSUPPORTED.  Negative B or dim, or a NULL pointer that is needed:
 * EU_ERR_INVALID.  out is not written on any refusal; B = 0 or dim = 0 does nothing.  Device pointers. */
#define EU_NEIGHBOR_TOP_K_MAX 16
int eu_neighbor_top_k_feature(eu_ctx* c, const int64_t* nodes, int64_t B, const int64_t* neighbors, int32_t count, int32_t fid,
                              int32_t dim, int32_t k, float* out);
/* eu_neighbor_top_k_feature into out of out_dtype (see eu_get_dense_feature_out_dtype): the selection is the f32 one, each
 * selected value rounded at the store.  The k and argument refusals come first, then the dtype's. */
int eu_neighbor_top_k_feature_out_dtype(eu_ctx* c, const int64_t* nodes, int64_t B, const int64_t* neighbors, int32_t count, int32_t fid,
                                        int32_t dim, int32_t k, int32_t out_dtype, void* out);
/* tf_euler.get_sparse_feature, one feature (tf_euler/kernels/get_sparse_feature_op.cc:52-130 over Node::GetUint64Feature
 * node.cc:366-379): the uint64 values of slot `fid` for every node, CSR-style: node i owns out_values[out_ptr[i], out_ptr[i+1]).
 * A node without values (absent node, unknown slot, empty slot) owns exactly ONE entry = default_value (the kernel's
 * SparseTensor gets {i, 0} -> default, :96-99).  cap = 0: lengths only (out_values may be NULL); only the first `cap`
 * entries are written.  The SparseTensor of the reference is indices (i, k - out_ptr[i]), dense_shape [M, max row length]. */
int eu_get_sparse_feature(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int64_t default_value, int64_t cap,
                          int64_t* out_ptr, int64_t* out_values);
int eu_get_sparse_feature_host(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int64_t default_value, int64_t cap,
                               int64_t* out_ptr, int64_t* out_values, int64_t* total);
/* tf_euler.get_binary_feature, one feature (tf_euler/kernels/get_binary_feature_op.cc over Node::GetBinaryFeature
 * node.cc:396-409): the bytes of slot `fid` for every node, CSR-style (absent node / unknown slot: empty string). */
int eu_get_binary_feature(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int64_t cap, int64_t* out_ptr, uint8_t* out_bytes);
int eu_get_binary_feature_host(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int64_t cap, int64_t* out_ptr,
                               uint8_t* out_bytes, int64_t* total);
/* SparseEmbedding's lookup from node ids (tf_euler/python/utils/layers.py:152-169: tf.nn.embedding_lookup_sparse(table, sp_ids,
 * None, combiner) over the SparseTensor of get_sparse_feature), fused: row i of out f32[M, dim] combines the rows of
 * table f32[n_rows, dim] named by node i's bag, the uint64 values of slot fid in stored order -- or the single entry
 * default_value when the node has none (absent id, empty or unknown slot), exactly as eu_get_sparse_feature lists them.
 * Fixed order: the sum starts from the bag's first row (a one-entry bag is that row's bits, -0.0 and NaN payloads included)
 * and adds the others left to right, one rounded add each; mean divides once by fl(n), sqrtn once by sqrtf(fl(n)).  Nothing is
 * materialised between the node ids and out; no synchronisation: capturable in a CUDA graph.
 * The backward pass writes grad_table f32[n_rows, dim] (zeros where no entry points): for value v, the sum over the entries
 * with value v of grad_out[i] (sum), grad_out[i] / fl(n_i) (mean) or grad_out[i] / sqrtf(fl(n_i)) (sqrtn), elementwise.  The
 * entries are listed again from the graph and ordered stably by value; each distinct value's entries are summed in chunks of
 * 256 counted from its first entry, each chunk left to right from +0, then the chunk sums in chunk order: deterministic, no
 * atomics.  It synchronises the stream once (to read the entry count E) and uses the ctx scratch: 8 B per node, about 24 B
 * per entry plus cub's sort storage, and (2E/256 + 1) * dim floats of chunk sums -- never O(n_rows) of index data.
 * combiner outside eu_combiner, n_rows or dim < 1, M < 0, a NULL pointer that is needed, default_value outside [0, n_rows),
 * or a slot whose largest value (kept on the graph since its creation) is >= n_rows: EU_ERR_INVALID, before any device work.
 * M or n_rows >= 2^31, or 2^31 or more entries in the backward: EU_ERR_UNSUPPORTED.  Device pointers. */
typedef enum { EU_COMBINE_SUM = 0, EU_COMBINE_MEAN = 1, EU_COMBINE_SQRTN = 2 } eu_combiner;
int eu_sparse_embedding_lookup(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int64_t default_value, const float* table,
                               int64_t n_rows, int32_t dim, int32_t combiner, float* out);
int eu_sparse_embedding_lookup_backward(eu_ctx* c, const float* grad_out, const int64_t* nodes, int64_t M, int32_t fid,
                                        int64_t default_value, int64_t n_rows, int32_t dim, int32_t combiner, float* grad_table);
/* The same gradient as a coalesced COO: rows i64[D] ascending and values f32[D, dim], *n (host) = D, the distinct values the
 * entries name; the arrays must hold min(entries, n_rows) rows (M entries at least, one per node).  No [n_rows, dim] buffer is
 * written.  Synchronises twice (the entry count, then D). */
int eu_sparse_embedding_lookup_backward_sparse(eu_ctx* c, const float* grad_out, const int64_t* nodes, int64_t M, int32_t fid,
                                               int64_t default_value, int64_t n_rows, int32_t dim, int32_t combiner, int64_t* rows,
                                               float* values, int64_t* n);
/* The forward with the table's storage type table_dtype (eu_feat_dtype): table is then read as that type.  Every read widens a
 * bf16 element to f32 exactly and all arithmetic stays f32 in the order above, so a EU_FEAT_BF16 call gives bit for bit what
 * the f32 call gives on the table widened to f32.  The 4-wide loads need dim % 4 == 0, the table 8-byte aligned (bf16) or
 * 16-byte aligned (f32) and out 16-byte aligned; otherwise scalar loads give the same bits.  EU_FEAT_F32 is the call above.
 * An unknown table_dtype: EU_ERR_INVALID, before any device work; every other bound and status as above.  The backward
 * entry points have no _dtype twin: they read grad_out, the graph's bags and the table's shape, never the table. */
int eu_sparse_embedding_lookup_dtype(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int64_t default_value, const void* table,
                                     int64_t n_rows, int32_t dim, int32_t combiner, int32_t table_dtype, float* out);

/* ShallowEncoder's input row, fused (tf_euler/python/utils/encoders.py:32-171): per node an id embedding, the dense feature
 * slots and one SparseEmbedding per uint64 slot, concatenated or added.  Node i of nodes i64[M]:
 *   id part      id_table[nodes[i]] (tf.nn.embedding_lookup: the node id is the row); id_table NULL = no id input
 *   dense part   dense[j]: eu_get_dense_feature(nodes, fid, dim) exactly (padded with zeros, clipped, zeros for an absent
 *                node or an unknown slot); a dim of 0 is allowed
 *   sparse part  sparse[s]: eu_sparse_embedding_lookup(nodes, fid, default_value, table, n_rows, dim, combiner) exactly, by the
 *                same device code (the same adds, in the same order)
 * EU_SHALLOW_CONCAT: out f32[M, W], row i = [id | dense_0 .. dense_{n_dense-1} | sparse_0 .. sparse_{n_sparse-1}], W the sum of
 *   the widths; dense_out unused.
 * EU_SHALLOW_ADD: every embedding (the id table and the slots) has one dim; out f32[M, dim] = id + sparse_0 + .. + sparse_last,
 *   added left to right from the first present term (one rounded add each); dense_out f32[M, sum of dense dims] = the dense
 *   part (the caller maps it through its Dense layer and adds it to out).  With no embedding, out is unused.
 * One lane group per node looks up the node's graph row once and writes its whole row.  No scratch and no synchronisation
 * while the stream is being captured, so the forward is capturable in a CUDA graph; outside capture an id table's ids are
 * checked first (one small kernel and one synchronisation) and one outside [0, n_id_rows) returns EU_ERR_INVALID before out is
 * written.  Under capture that check is skipped: such a row's id columns are NaN and the id is never dereferenced.
 * Backward (the gradient reaches the tables only; features are not trainable): grad_out has out's shape.  Table t (0 = the id
 * table, 1 + s = slot s) gets, for each of its rows, the sum of its entries' gradient rows: the id table's entries are the
 * nodes (row nodes[i]); slot s's are eu_sparse_embedding_lookup_backward's (each value of the node's bag, or the default),
 * with its combiner's division.  The gradient row of an entry of node i is grad_out[i] restricted to the table's columns
 * (CONCAT) or grad_out[i] (ADD).  Every table's entries are listed in one pass over the nodes, ordered stably by row and summed
 * per distinct row in 256-entry chunks (eu_sparse_embedding_lookup_backward's order): no atomics, the same bits on every run.
 *   eu_shallow_encode_backward:        grads[t] dense f32[n_rows_t, dim_t], zero on untouched rows (NULL: no id table)
 *   eu_shallow_encode_backward_sparse: rows[t] i64[D_t] ascending, values[t] f32[D_t, dim_t], counts[t] = D_t (host); arrays of
 *                                      min(entries_t, n_rows_t) rows (M for the id table); no [n_rows, dim] buffer is written
 * Both synchronise once to read the entry counts (the sparse one once more, for D_t).  Scratch: 8 B per node and slot, about
 * 48 B per entry of the largest table, and M dim floats per mean / sqrtn slot; never O(n_rows).
 * Bounds: at most EU_SHALLOW_MAX_SLOTS dense and sparse slots each, W at most EU_SHALLOW_MAX_WIDTH columns, M and table rows
 * below 2^31, and (backward) fewer than 2^31 entries: EU_ERR_UNSUPPORTED beyond them.  A bad combiner, a missing table or
 * output, a dim < 1, ADD with unequal embedding dims, a default outside its table or a slot whose largest value is outside it:
 * EU_ERR_INVALID, before any device work.  Device pointers. */
#define EU_SHALLOW_MAX_SLOTS 8
#define EU_SHALLOW_MAX_WIDTH 16384
enum { EU_SHALLOW_CONCAT = 0, EU_SHALLOW_ADD = 1 };
typedef struct {
  int32_t fid;              /* dense slot id (unknown: zeros) */
  int32_t dim;              /* columns, >= 0 */
} eu_shallow_dense;
typedef struct {
  int32_t fid;              /* uint64 slot id (unknown: every node gets the default) */
  int32_t dim;              /* the table's columns, >= 1 */
  int32_t combiner;         /* eu_combiner */
  int32_t reserved;         /* 0 */
  int64_t default_value;    /* in [0, n_rows) */
  int64_t n_rows;
  const float* table;       /* f32[n_rows, dim]; with the _dtype calls' EU_FEAT_BF16, bf16 storage of that shape */
} eu_shallow_sparse;
typedef struct {
  int32_t combiner;         /* EU_SHALLOW_CONCAT or EU_SHALLOW_ADD */
  int32_t id_dim;
  int64_t M;
  const int64_t* nodes;     /* [M] */
  const float* id_table;    /* f32[n_id_rows, id_dim], or NULL; with the _dtype calls' EU_FEAT_BF16, bf16 storage */
  int64_t n_id_rows;
  int32_t n_dense, n_sparse;
  eu_shallow_dense dense[EU_SHALLOW_MAX_SLOTS];
  eu_shallow_sparse sparse[EU_SHALLOW_MAX_SLOTS];
} eu_shallow_problem;
int eu_shallow_encode(eu_ctx* c, const eu_shallow_problem* p, float* out, float* dense_out);
int eu_shallow_encode_backward(eu_ctx* c, const eu_shallow_problem* p, const float* grad_out, float* const* grads);
int eu_shallow_encode_backward_sparse(eu_ctx* c, const eu_shallow_problem* p, const float* grad_out, int64_t* const* rows,
                                      float* const* values, int64_t* counts);
/* eu_shallow_encode with the tables' storage type table_dtype (eu_feat_dtype): the id table and every slot's table have it,
 * and the problem's table pointers are then read as that type (the struct's layout is unchanged).  As for
 * eu_sparse_embedding_lookup_dtype, every table read widens bf16 to f32 exactly and all arithmetic stays f32 in the order
 * above, so a EU_FEAT_BF16 call gives the f32 call's bits on the widened tables, with f32 or bf16 dense features alike.  A
 * slot's 4-wide loads need its table aligned to four elements (8 bytes of bf16, 16 of f32) and out 16-byte aligned.  An
 * unknown table_dtype: EU_ERR_INVALID, before any device work; every other bound and status as eu_shallow_encode's.  The
 * backward entry points serve both dtypes: they never dereference a table (only its rows and dim). */
int eu_shallow_encode_dtype(eu_ctx* c, const eu_shallow_problem* p, int32_t table_dtype, float* out, float* dense_out);

/* ShallowEncoder's rows pooled over fixed segments: what SageEncoder's first layer needs of the deepest hop of a fanout
 * (tf_euler/python/utils/encoders.py:475-491: the hop's rows reshaped to [R, count, W] reach the mean / gcn aggregator only
 * through a reduction over the count axis).  p is an EU_SHALLOW_CONCAT problem with M = R * count nodes; row r of
 * out f32[R, W] pools the count rows eu_shallow_encode would write for nodes[r * count .. r * count + count - 1], every one
 * of them by eu_shallow_encode's rules (an absent node, sample_fanout's default_node, an empty bag: rows like any other, and
 * they count in the divisor, as tf.reduce_mean(axis=1) counts them).  The [M, W] matrix is never written.
 * Fixed order, per column: acc = row_0's value; acc = __fadd_rn(acc, row_j's value) for j = 1 .. count - 1, where a sparse
 * slot's value is the bag sum after its combiner's division, as eu_sparse_embedding_lookup rounds it.  EU_POOL_SUM: out = acc.
 * EU_POOL_MEAN: out = __fdiv_rn(acc, fl(count)).  The bits do not depend on the alignment of the tables or of out.
 * One lane group per output row looks each node's graph row up once (shared memory) and sums a tile of columns in registers.
 * No scratch, no synchronisation while the stream is being captured; outside capture the id check of eu_shallow_encode.
 * Backward: grad_out f32[R, W]; the gradient row of node k is grad_out[k / count], for EU_POOL_MEAN with every element
 * divided by fl(count) as it is read (one __fdiv_rn, before a mean / sqrtn slot's own division by its bag's divisor, which
 * is a second __fdiv_rn exactly as autograd through eu_shallow_encode and a mean over the segment would do).  Everything else
 * is eu_shallow_encode_backward(_sparse): the same entries, order, chunks, outputs, synchronisations and scratch (the M dim
 * floats of a mean / sqrtn slot included; no [M, W] gradient exists anywhere).
 * Bounds: eu_shallow_encode's, and count at most EU_SHALLOW_POOL_MAX_COUNT; EU_SHALLOW_ADD is EU_ERR_UNSUPPORTED.  count < 1,
 * M % count != 0 or a pool outside the enum: EU_ERR_INVALID.  Device pointers. */
#define EU_SHALLOW_POOL_MAX_COUNT 512
enum { EU_POOL_SUM = 0, EU_POOL_MEAN = 1 };
int eu_shallow_encode_pool(eu_ctx* c, const eu_shallow_problem* p, int32_t count, int32_t pool, float* out);
/* eu_shallow_encode_pool with the tables' storage type table_dtype, by eu_shallow_encode_dtype's rules. */
int eu_shallow_encode_pool_dtype(eu_ctx* c, const eu_shallow_problem* p, int32_t table_dtype, int32_t count, int32_t pool, float* out);
int eu_shallow_encode_pool_backward(eu_ctx* c, const eu_shallow_problem* p, int32_t count, int32_t pool, const float* grad_out,
                                    float* const* grads);
int eu_shallow_encode_pool_backward_sparse(eu_ctx* c, const eu_shallow_problem* p, int32_t count, int32_t pool,
                                           const float* grad_out, int64_t* const* rows, float* const* values, int64_t* counts);

/* Graph-level minibatches (graph classification; reference: euler/core/kernels/sample_graph_label_op.cc,
 * get_graph_by_label_op.cc and Graph::GetGraphLabel, euler/core/graph/graph.cc:439-457).
 * A graph's label table is built on the first graph-label call from its binary feature slot named "graph_label" (the
 * reference's "binary_graph_label"; name a synthetic graph's slot with eu_graph_set_binary_feature_name before that call):
 * the label list is GetGraphLabel's, in its order (an unordered_set of every node's value in node_map_ order, "" for a node
 * without one), and each label's nodes are listed by ascending id (a chosen order: the reference's is its index file's).
 * The label "" lists no nodes, as the converter indexes only the values present.  A graph without the slot or without nodes:
 * every graph-label call returns EU_ERR_STATE ("graph label set is empty!", where the reference aborts).
 * eu_graph_labels reports the list (builds the table: needs the device): n_labels, n_bytes, ptr i64[n_labels + 1] (host, may
 * be NULL) and the concatenated bytes (host, written when n_bytes <= cap).  eu_graph_labels_inspect reports the same list for
 * an Euler directory (shard 0 of 1) without a device.  eu_graph_set_binary_feature_name renames slot fid; EU_ERR_STATE once the
 * label table is built. */
int eu_graph_set_binary_feature_name(eu_graph* g, int32_t fid, const char* name);
int eu_graph_labels(eu_graph* g, int64_t cap, int64_t* n_labels, int64_t* n_bytes, int64_t* ptr, uint8_t* bytes);
int eu_graph_labels_inspect(const char* data_path, int64_t cap, int64_t* n_labels, int64_t* n_bytes, int64_t* ptr,
                            uint8_t* bytes);
/* tf_euler.sample_graph_label: out i32[count] (device) = label indices floor(u * L), u one ThreadLocalRandom() draw each
 * (generate_canonical<double,53>: two minstd_rand0 steps), drawn from the ctx engine and counted in its draws as
 * eu_sample_node's are, so a call followed by any other sampling op reproduces the reference's thread-local stream under
 * EU_RNG_MINSTD; EU_RNG_PHILOX draws one Philox uniform per label.  An index that would round up to L is clamped to L - 1.
 * count = 0 does nothing. */
int eu_sample_graph_label(eu_ctx* c, int32_t count, int32_t* out);
/* tf_euler.get_graph_by_label: labels i32[B] (device; label indices, -1 = a label the graph does not know).  The output is the
 * reference's SparseTensor content: row i lists the node ids of graph i; an unknown label or one without nodes gets the single
 * entry (i, 0) = 0.  Two passes, device pointers:
 *   cap = 0: ptr i64[B + 1] = the row offsets; *total and *max_len (host) = the entries and the longest row (one stream
 *            synchronisation);
 *   cap > 0: from that ptr, indices i64[cap, 2] = (i, j) and values i64[cap] = the ids; entries at or past cap are not written. */
int eu_get_graph_by_label(eu_ctx* c, const int32_t* labels, int64_t B, int64_t cap, int64_t* ptr, int64_t* indices,
                          int64_t* values, int64_t* total, int64_t* max_len);
/* The attention readout of AttentionPool (aggr = 'add') and of one Set2SetPool step (tf_euler/python/graph_pool/), fused.
 * x f32[N, dim], index i32[N] (each row's graph in [0, B)), and exactly one of
 *   logits f32[N]    (AttentionPool's gate), or
 *   q f32[B, dim]    (Set2Set's query: the logit of row n is <x_n, q[index_n]>, in eu_agnn_aggregate's fixed dot order).
 *   alpha[n] = scatter_softmax(logits, index, B)   (running max from -1e9, as scatter_max)
 *   out[b]   = sum over the rows n of graph b of alpha[n] * x[n]     (a graph without rows gets a zero row)
 * A graph's rows are walked in index order (unsorted index: a stable sort first, so the bits are those of the stably sorted
 * rows); its sums (of the exps, and of the weighted rows) are fixed-order chunked segment sums: chunks of 256 rows each added
 * left to right from +0, then the chunk sums in chunk order.  For graphs of at most 256 rows and a non-decreasing index, out
 * and alpha equal scatter_softmax -> multiply -> scatter_add composed from the ops above bit for bit.  alpha f32[N] is
 * required (the backward pass reads it); out f32[B, dim].
 * The backward pass takes grad_out f32[B, dim] and alpha, and writes, with d_n = <x_n, g_b> (the order of the dot above) and
 * S_b = sum over graph b of alpha_n * d_n (chunked):
 *   dl_n = alpha_n * (d_n - S_b),  grad_x f32[N, dim] = alpha_n * g_b (+ dl_n * q_b),
 *   grad_logits f32[N] = dl (logits mode; q NULL) or grad_q f32[B, dim] = sum over graph b of dl_n * x_n (chunked).
 * Deterministic, no atomics.  dim < 1, negative sizes, rows with B = 0, both or neither of logits / q, or a NULL pointer that
 * is needed: EU_ERR_INVALID; 2^31 or more rows or graphs: EU_ERR_UNSUPPORTED.  index is not checked (as eu_gather).  Both calls
 * synchronise the stream once to read whether index is sorted, and use the ctx scratch: 4 B per row and graph, 12 B per
 * graph of segment plan, (B + N / 256) * dim floats of chunk sums, and a sort of 12 B per row when index is unsorted. */
int eu_graph_attention_readout(eu_ctx* c, const float* x, const int32_t* index, int64_t N, int64_t B, int32_t dim,
                               const float* logits, const float* q, float* out, float* alpha);
int eu_graph_attention_readout_backward(eu_ctx* c, const float* grad_out, const float* x, const int32_t* index, int64_t N,
                                        int64_t B, int32_t dim, const float* q, const float* alpha, float* grad_x,
                                        float* grad_logits, float* grad_q);

/* The unsupervised skip-gram step of DeepWalk / node2vec / LINE, fused (reference: UnsuperviseModel.__call__,
 * tf_euler/python/mp_utils/base.py:50-91 and solution/base_unsupervise.py, with PosNegLogits solution/logits.py, xent_loss
 * solution/losses.py and the rank of mrr_score / hitk_score / mr_score utils/metrics.py).  Ids are table rows, as
 * tf.nn.embedding_lookup uses them: src i64[B], pos i64[B, P] (P >= 1), negs i64[B, K] (K >= 0); target and context
 * f32[n_rows, dim] (may be the same table).  Outputs, device pointers:
 *   logits f32[B, P + K]: row b is <target[src_b], context[c]> for c = pos[b, 0 .. P-1], then negs[b, 0 .. K-1], each a dot in
 *                         eu_agnn_aggregate's fixed order (per-lane fma sums over 4-column chunks, then a fixed butterfly;
 *                         the order depends on dim only, never on the launch);
 *   rank i32[B]:          #{j != P-1 : logits[b, j] >= logits[b, P-1]}, the position TF's stable top_k gives the last positive
 *                         in concat([neg, pos], 2) (ties rank it behind);
 *   loss f32[1]:          the mean over the B (P + K) logits of max(x, 0) - x z + log1p(exp(-|x|)), z = 1 for the positives:
 *                         f32 terms summed in f64 in a fixed order, one division (B = 0: NaN).
 * An id outside [0, n_rows) is never dereferenced: EU_ERR_INVALID after the call's one stream synchronisation.
 * The backward passes take grad_loss (a device f32 scalar, read on the device) and the forward's logits, and recompute
 * c_bj = (sigmoid(x) - z) g / (B (P + K)).  The gradient of the target table sums, per distinct src id, the rows
 * sum_j c_bj context[ctx_bj] of its pairs; that of the context table sums, per distinct context id, c_bj target[src_b] over its
 * entries (b, j).  Entries are ordered stably by row (a shared table lists the B src entries first, then the context entries
 * in (b, j) order) and summed in chunks of 256 counted from each row's first entry, left to right from +0, then the chunk sums
 * in chunk order: no atomics, the same bits on every run.  Scratch: O(B (P + K)) of index data plus B dim floats, never
 * O(n_rows); one stream synchronisation per call.
 *   eu_skipgram_loss_backward:        dense grad_target and grad_context f32[n_rows, dim], zero on untouched rows;
 *                                     grad_context == grad_target means one shared table (both gradients summed into it).
 *   eu_skipgram_loss_backward_sparse: the coalesced COO of each table's gradient: rows i64[D] ascending and values f32[D, dim],
 *                                     D (host) = the distinct ids; the arrays must hold min(entries, n_rows) rows (B for the
 *                                     target, B (P + K) for the context, B (P + K + 1) for a shared table).  rows_context
 *                                     NULL means one shared table, written to the target outputs.
 * P < 1, K < 0, B < 0, n_rows or dim < 1, or a NULL pointer that is needed: EU_ERR_INVALID; n_rows >= 2^31, or B (P + K + 1)
 * entries with their 256-entry chunks reaching 2^31: EU_ERR_UNSUPPORTED. */
int eu_skipgram_loss(eu_ctx* c, const int64_t* src, const int64_t* pos, const int64_t* negs, int64_t B, int32_t P, int32_t K,
                     const float* target, const float* context, int64_t n_rows, int32_t dim, float* logits, int32_t* rank,
                     float* loss);
int eu_skipgram_loss_backward(eu_ctx* c, const float* grad_loss, const int64_t* src, const int64_t* pos, const int64_t* negs,
                              int64_t B, int32_t P, int32_t K, const float* target, const float* context, int64_t n_rows,
                              int32_t dim, const float* logits, float* grad_target, float* grad_context);
int eu_skipgram_loss_backward_sparse(eu_ctx* c, const float* grad_loss, const int64_t* src, const int64_t* pos, const int64_t* negs,
                                     int64_t B, int32_t P, int32_t K, const float* target, const float* context, int64_t n_rows,
                                     int32_t dim, const float* logits, int64_t* rows_target, float* values_target,
                                     int64_t* n_target, int64_t* rows_context, float* values_context, int64_t* n_context);
/* The same three with the tables' storage type table_dtype (eu_feat_dtype; both tables have it).  Two rules make a bf16
 * call exact: every read widens a bf16 element to f32 exactly, and all arithmetic stays f32 in the order above.  So a
 * EU_FEAT_BF16 call gives bit for bit what the f32 call gives on the tables widened to f32; logits, rank, loss and the
 * gradients stay f32.  The 4-wide loads need dim % 4 == 0 and the tables 8-byte aligned (bf16) or 16-byte aligned (f32);
 * other tables take scalar loads with the same bits.  An unknown table_dtype: EU_ERR_INVALID. */
int eu_skipgram_loss_dtype(eu_ctx* c, const int64_t* src, const int64_t* pos, const int64_t* negs, int64_t B, int32_t P, int32_t K,
                           const void* target, const void* context, int64_t n_rows, int32_t dim, int32_t table_dtype,
                           float* logits, int32_t* rank, float* loss);
int eu_skipgram_loss_backward_dtype(eu_ctx* c, const float* grad_loss, const int64_t* src, const int64_t* pos, const int64_t* negs,
                                    int64_t B, int32_t P, int32_t K, const void* target, const void* context, int64_t n_rows,
                                    int32_t dim, int32_t table_dtype, const float* logits, float* grad_target,
                                    float* grad_context);
int eu_skipgram_loss_backward_sparse_dtype(eu_ctx* c, const float* grad_loss, const int64_t* src, const int64_t* pos,
                                           const int64_t* negs, int64_t B, int32_t P, int32_t K, const void* target,
                                           const void* context, int64_t n_rows, int32_t dim, int32_t table_dtype,
                                           const float* logits, int64_t* rows_target, float* values_target, int64_t* n_target,
                                           int64_t* rows_context, float* values_context, int64_t* n_context);

/* The reconstruction step of the graph auto-encoders GAE and VGAE (tf_euler/python/mp_utils/base_gae.py, examples/gae/gae.py),
 * fused, over encoder rows.  Three sets of f32 row-major device rows, each 4-byte aligned (16-byte alignment and D % 4 == 0
 * take vector loads, with the same bits): set 0 the sources [B, D], set 1 the positives [B, K, D], set 2 the negatives
 * [B, K, D].  mu[s] are the rows; for the variational form log_var[s] (same shapes) and optionally noise[s] (unit-normal
 * draws, same shapes) are given too, and the op forms z = mu + (radius noise) sqrt(exp(log_var)) itself, element by element in
 * f32, without writing it; noise NULL gives z = mu (VGAE's train=False), log_var NULL the plain GAE (z = mu, no KL).  The
 * pointer arrays mu, log_var, noise (three entries each) are host arrays.  Outputs, device pointers:
 *   logits f32[B, 2K] (may be NULL): row b is <z_src[b], z_pos[b, k]> for k < K, then <z_src[b], z_neg[b, k]>, each dot in
 *                         eu_skipgram_loss's fixed order (per-lane fma sums over 4-column chunks, then a fixed butterfly);
 *   loss f32[1]:          the mean over the 2BK logits of max(x, 0) - x z + log1p(exp(-|x|)), z = 1 for the positives (f32
 *                         terms summed in f64, one division), plus, in the variational form, the mean over the B D (2K + 1)
 *                         elements of kl = -0.5 (log_var - exp(log_var) - mu^2 + 1) (f32 elements summed in f64, one division),
 *                         the two f32 means added in f32 (B = 0: NaN);
 *   correct i64[1]:       #{floor(sigmoid(x) + 0.5) == z} over the 2BK logits, sigmoid(x) = 1 / (1 + exp(-x)) in f32.
 * The backward pass takes grad_loss (a device f32 scalar, read on the device) and the forward's logits, and writes dense
 * gradients of the same shapes as the inputs: grad_mu[s] = dL/dz (+ grad kl / (B D (2K + 1)) mu in the variational form),
 * grad_log_var[s] (required with log_var) = dL/dz (radius noise) 0.5 sqrt(exp(log_var)) + grad (exp(log_var) - 1) / (2 B D
 * (2K + 1)); none goes to noise.  dL/dz_ctx[b, j] = c_bj z_src[b] and dL/dz_src[b] = sum over j of c_bj z_ctx[b, j] (fma from
 * +0 in j order) with c_bj = (sigmoid(x_bj) - z) grad / 2BK.  Every element is written by one thread: no atomics, the same
 * bits on every run, and neither pass synchronises with the host, so both can be captured in a CUDA graph (once the ctx
 * scratch, O(B K) f64, has grown to the batch outside the capture).
 * B < 0, K < 1, D < 1, a non-finite radius, noise without log_var, or a NULL pointer that is needed: EU_ERR_INVALID with
 * nothing written; K >= 2^29 or B (2K + 1) >= 2^34: EU_ERR_UNSUPPORTED. */
int eu_gae_loss(eu_ctx* c, int64_t B, int32_t K, int32_t D, const float* const* mu, const float* const* log_var,
                const float* const* noise, float radius, float* logits, float* loss, int64_t* correct);
int eu_gae_loss_backward(eu_ctx* c, const float* grad_loss, int64_t B, int32_t K, int32_t D, const float* const* mu,
                         const float* const* log_var, const float* const* noise, float radius, const float* logits,
                         float* const* grad_mu, float* const* grad_log_var);

/* The streaming metrics of tf_euler/python/utils/metrics.py (auc_score, f1_score, acc_score), TF 1.x tf.metrics semantics:
 * each call adds one batch's counts to f32 state the caller owns (device) and writes the value of the new state (device f32
 * scalar), as the metric's update op returns it.  Every per-batch count is an exact integer, rounded once to f32 and added to
 * the state with one f32 add: TF's float reduce_sum gives the same counts for batches below 2^24 elements.  Labels and
 * predictions are f32[N] device arrays; a label is positive when nonzero (NaN included).  Neither call synchronises with the
 * host (once the ctx scratch, O(T), has grown) and neither uses float atomics: the bits depend on the inputs only, and both
 * can be captured in a CUDA graph.
 *
 * eu_metric_auc_update: tf.metrics.auc(labels, predictions, num_thresholds=T), trapezoidal ROC.  Thresholds t[0] =
 * fl32(-1e-7), t[i] = fl32(i / (T - 1)) for 0 < i < T - 1 (computed in double), t[T-1] = fl32(1 + 1e-7); prediction p is
 * positive at threshold i iff p > t[i] in f32.  The state is tp, fn, tn, fp f32[T].  Each prediction is bucketed once and
 * counted in integer histograms; prefix sums give the per-threshold counts.  The value, with eps = 1e-6,
 *   rec[i] = (tp + eps) / ((tp + fn) + eps),  fpr[i] = fp / ((fp + tn) + eps),
 *   auc = sum over i < T - 1 of (fpr[i] - fpr[i+1]) ((rec[i] + rec[i+1]) / 2),
 * each op one round-to-nearest f32 op, is summed in this fixed order: lane j of 1024 adds the terms j, j + 1024, .. from +0
 * left to right, then the 1024 lane sums are added by a tree (lane j += lane j + s for s = 512, 256, .., 1); the result is
 * lane 0.  A batch with a prediction outside [0, 1] or NaN (TF asserts) is not counted: the state is untouched and
 * *refused (device i64) += 1.  The value is NaN while *refused > 0.  N = 0 counts nothing and rewrites the value.
 * T < 2 or T > EU_METRIC_AUC_MAX_THRESHOLDS, N < 0, or a NULL pointer that is needed: EU_ERR_INVALID, before any device work.
 *
 * eu_metric_count_update: kind EU_METRIC_F1 (state f32[3] = tp, fn, fp; predictions floor(p + 0.5) in f32 cast to bool,
 * NaN true; value p = tp / ((1e-7 + tp) + fp), r = tp / ((1e-7 + tp) + fn), f1 = ((2 p) r) / ((p + r) + 1e-7)) or
 * EU_METRIC_ACC (state f32[2] = total, count; total += #{floor(p + 0.5) == label}, count += N; value total / count, 0 while
 * count is 0).  With correct (a device i64 scalar) instead of labels and predictions, for EU_METRIC_ACC only, total +=
 * *correct and count += N: a count the caller already has, e.g. eu_gae_loss's, with no second pass.
 * An unknown kind, N < 0, a NULL pointer that is needed, or correct with labels, predictions or EU_METRIC_F1: EU_ERR_INVALID,
 * before any device work. */
#define EU_METRIC_AUC_MAX_THRESHOLDS 16384
enum { EU_METRIC_F1 = 0, EU_METRIC_ACC = 1 };
int eu_metric_auc_update(eu_ctx* c, const float* labels, const float* predictions, int64_t N, int32_t T, float* tp, float* fn,
                         float* tn, float* fp, int64_t* refused, float* value);
int eu_metric_count_update(eu_ctx* c, int32_t kind, const float* labels, const float* predictions, int64_t N,
                           const int64_t* correct, float* state, float* value);

/* tf_euler's optimizers (utils/optimizers.py: sgd and momentum = MomentumOptimizer(lr, 0 / 0.9), AdagradOptimizer,
 * AdamOptimizer) as TF 1.x applies them, in place over var f32[N, D] and its slot tables (accum, or m and v) of the same
 * shape, on the ctx's stream.  All arithmetic is f32, each op rounded once in the order written, no FMA contraction;
 * rsqrt(a) = 1 / sqrt(a).
 * The gradient is dense (R = EU_OPTIM_DENSE: grad f32[N, D]) or sparse (R >= 0: rows i64[R], sorted and unique in [0, N),
 * as a coalesced COO gradient has them, and grad f32[R, D]; TF sums duplicate IndexedSlices first).
 *   Momentum (non-Nesterov): accum = accum * momentum + g; var = var - lr * accum.  Sparse: the R rows only.
 *   Adagrad: accum = accum + g * g; var = var - (lr * g) * rsqrt(accum).  Sparse: the R rows only.
 *   Adam, dense (ApplyAdam): m = m + (g - m) * (1 - b1); v = v + (g * g - v) * (1 - b2);
 *     var = var - (m * alpha) / (sqrt(v) + eps).
 *   Adam, sparse (_apply_sparse_shared), EVERY row: m = m * b1, then on the R rows m = m + g * (1 - b1); v = v * b2, then on
 *     the R rows v = v + (g * g) * (1 - b2); var = var - (alpha * m) / (sqrt(v) + eps).
 *   alpha = (lr * sqrt(1 - beta2_power)) / (1 - beta1_power), computed on the device from powers (device f32[2]:
 *   beta1_power, beta2_power).  The caller multiplies each power by its beta once after every variable of a step (TF's
 *   _finish).
 * Sparse Adam is one pass over the table (24 N D + 4 R (D + 2) bytes); sparse Momentum and Adagrad touch the R rows only.
 * A sparse row outside [0, N) is never written.  No host synchronisation and no float atomics: every call can be captured
 * in a CUDA graph.  N < 0, D < 1, R < EU_OPTIM_DENSE, R > N, or a NULL pointer that is needed: EU_ERR_INVALID, before any
 * device work.  Device pointers. */
#define EU_OPTIM_DENSE (-1)
int eu_optim_momentum(eu_ctx* c, float* var, float* accum, int64_t N, int32_t D, const float* grad, const int64_t* rows,
                      int64_t R, float lr, float momentum);
int eu_optim_adagrad(eu_ctx* c, float* var, float* accum, int64_t N, int32_t D, const float* grad, const int64_t* rows,
                     int64_t R, float lr);
int eu_optim_adam(eu_ctx* c, float* var, float* m, float* v, int64_t N, int32_t D, const float* grad, const int64_t* rows,
                  int64_t R, const float* powers, float lr, float beta1, float beta2, float epsilon);
/* The same three over var and slots of storage type dtype (eu_feat_dtype; the gradient stays f32).  EU_FEAT_F32 is the call
 * above (seed, step and tensor unused).  EU_FEAT_BF16 keeps the skip-gram tables' two rules -- every read widens bf16 to f32
 * exactly, all arithmetic stays f32 in the order above -- so the only new rounding is the store: each value written (var
 * and every slot) is rounded to bf16 by stochastic rounding.  A 16-bit random integer r is added to the low half of the f32
 * bits, which are then truncated: the value rounds up with probability (distance to the bf16 below) / ulp, so a small update
 * survives on average where round to nearest would drop every update below half an ulp.  +-Inf stays; a NaN stays a NaN
 * (its sign and upper payload kept, made quiet).  r is the low 16 bits of word w (0 var, 1 accum or m, 2 v) of the
 * Philox4x32-10 block with key seed and counter (element lo, element hi, *step mod 2^32, tensor): element is the flat index
 * into var (row r, column d: r D + d, for dense and sparse gradients alike), step a device i64 counter the caller advances
 * once per step after every variable (as Adam's powers; read on the device, so a step can be captured in a CUDA graph), and
 * tensor the variable's index among those the caller updates with one seed.  Sparse Adam rounds every row it writes, the
 * decay-only rows included.  The 4-wide form needs D % 4 == 0, var and slots 8-byte aligned and grad 16-byte aligned.  An
 * unknown dtype, or EU_FEAT_BF16 without step: EU_ERR_INVALID, before any device work. */
int eu_optim_momentum_dtype(eu_ctx* c, void* var, void* accum, int64_t N, int32_t D, const float* grad, const int64_t* rows,
                            int64_t R, float lr, float momentum, int32_t dtype, uint64_t seed, const int64_t* step,
                            int32_t tensor);
int eu_optim_adagrad_dtype(eu_ctx* c, void* var, void* accum, int64_t N, int32_t D, const float* grad, const int64_t* rows,
                           int64_t R, float lr, int32_t dtype, uint64_t seed, const int64_t* step, int32_t tensor);
int eu_optim_adam_dtype(eu_ctx* c, void* var, void* m, void* v, int64_t N, int32_t D, const float* grad, const int64_t* rows,
                        int64_t R, const float* powers, float lr, float beta1, float beta2, float epsilon, int32_t dtype,
                        uint64_t seed, const int64_t* step, int32_t tensor);

/* The knowledge-graph embedding step of TransE / TransH / TransR / TransD (examples/TransX) and DistMult (examples/distmult),
 * fused: the mapped id rows of each triple and of its corrupted triples, the scores, the margin loss and the rank.
 * Triple b: src_b, dst_b (entity ids), rel_b (relation id), neg[b, 0 .. K-1] (entity ids); ids are table rows.
 * Tables (device f32; table[t] for t = 0 .. 3): entity [n_ent, ent_dim], relation [n_rel, rel_dim], the entity-side
 * auxiliary (TransD's entity_transfer [n_ent, ent_dim], else NULL) and the relation-side one (TransH's hyper [n_rel, ent_dim],
 * TransR's transfer matrix [n_rel, ent_dim * rel_dim] read as [ent_dim, rel_dim], TransD's relation_transfer [n_rel, rel_dim],
 * else NULL).  With n(x) = x / sqrt(max(sum x^2, 1e-12)) and r = n(relation[rel_b]), an entity row e maps to n(e) (TransE,
 * DistMult), e - (e . h) h with h = n(hyper[rel_b]) (TransH), n(e M) (TransR), n(e + (e . et) rt) (TransD); a triple (a, r, c)
 * scores -||(a + r) - c|| in L1 or L2 (l1) or sum a (r c) (DistMult).  Each relation row is normalised over its own rel_dim.
 * Outputs (device):
 *   scores f32[B, 1 + C K]: the true triple, then (corrupt 1 'front', 2 'tail', 3 'both' = C 2) the K front corruptions
 *                           (neg_k, r, d), then the K tail corruptions (s, r, neg_k);
 *   rank i32[B]:            #{j : neg_j >= pos}, TF's stable top_k position of the last entry of concat([neg, pos]);
 *   loss f32[1]:            mean over b of max((margin + mean_j neg_j) - pos_b, 0): the negative mean a fixed-order f32 sum (see
 *                           csrc/kg.cu), the row losses added in f64 and divided once by B (B = 0: NaN);
 *   src_emb, rel_emb, dst_emb f32[B, rel_dim] (optional, all or none): the mapped rows of the triple.
 * Every reduction has a fixed order that depends on the dims only.  No [B, K, dim] rows are formed: a block maps its triple's
 * rows once, stages TransR's matrix in shared memory and scores a tile of 256 negatives.
 * The backward passes take grad_loss (a device f32 scalar) and the forward's scores.  A row is active when its hinge argument
 * is >= 0 (TF's maximum on equality); L1 differentiates |x| as sign(x) (0 at 0), L2 gives 0 where ||x|| = 0 (TF: NaN), and
 * n(x) passes no gradient to sum x^2 below 1e-12.  One entry per (triple, table row touched): entity entries src, dst, each
 * (b, k) with its front and tail terms summed; one relation and one relation-side entry per triple.  The entries of a table
 * are summed per distinct row in the stable row order in 256-entry chunks (see eu_skipgram_loss_backward): no atomics, the same
 * bits on every run.  Scratch O(B (K + 2) dim) (TransR: plus B ent_dim rel_dim floats), never O(n_rows); one synchronisation.
 *   eu_kg_loss_backward:        grads[t] f32 dense gradient of table t (zero on untouched rows; NULL for an absent table);
 *   eu_kg_loss_backward_sparse: the coalesced COO of table t: rows[t] i64[D] ascending, values[t] f32[D, width], counts[t] = D
 *                               (host); arrays of min(entries, table rows) rows: B (K + 2) for the entity-side tables, B for the
 *                               relation-side ones.
 * K < 1, B < 0, a missing table the model needs, ent_dim != rel_dim outside TransR, or an id outside its table: EU_ERR_INVALID;
 * a dim above 512, a TransR ent_dim * rel_dim above 16384, 2^31 table rows or B (K + 2) entries: EU_ERR_UNSUPPORTED. */
enum { EU_KG_TRANSE = 0, EU_KG_TRANSH = 1, EU_KG_TRANSR = 2, EU_KG_TRANSD = 3, EU_KG_DISTMULT = 4 };
typedef struct {
  int32_t model;            /* EU_KG_* */
  int32_t l1;               /* TransX: 1 = L1 distance, 0 = L2 */
  int32_t corrupt;          /* 1 front, 2 tail, 3 both */
  float margin;
  int64_t B;
  int32_t K;                /* negatives per triple, >= 1 */
  int32_t ent_dim, rel_dim;
  int64_t n_ent, n_rel;     /* rows of the entity-side and the relation-side tables */
  const int64_t* src;       /* [B] */
  const int64_t* dst;       /* [B] */
  const int64_t* rel;       /* [B] */
  const int64_t* neg;       /* [B, K] */
  const float* table[4];    /* entity, relation, entity-side auxiliary, relation-side auxiliary; with the _dtype calls'
                               EU_FEAT_BF16 each points at bf16 storage of the same shape */
} eu_kg_problem;
int eu_kg_loss(eu_ctx* c, const eu_kg_problem* p, float* scores, int32_t* rank, float* loss, float* src_emb, float* rel_emb,
               float* dst_emb);
int eu_kg_loss_backward(eu_ctx* c, const eu_kg_problem* p, const float* grad_loss, const float* scores, float* const* grads);
int eu_kg_loss_backward_sparse(eu_ctx* c, const eu_kg_problem* p, const float* grad_loss, const float* scores, int64_t* const* rows,
                               float* const* values, int64_t* counts);
/* The same three with the tables' storage type table_dtype (eu_feat_dtype; every table of the call has it, and table[t] is
 * then read as that type).  The skip-gram tables' two rules make a bf16 call exact: every read widens a bf16 element to f32
 * exactly (TransR's matrix is staged widened), and all arithmetic stays f32 in the order above.  So a EU_FEAT_BF16 call
 * gives bit for bit what the f32 call gives on the tables widened to f32; scores, rank, loss, the embeddings and every
 * gradient stay f32.  The 4-wide loads need both dims % 4 == 0 and each table 8-byte aligned (bf16) or 16-byte aligned
 * (f32); other tables take scalar loads with the same bits.  EU_FEAT_F32 is the call above.  An unknown table_dtype:
 * EU_ERR_INVALID, before any device work; every other bound and status as above. */
int eu_kg_loss_dtype(eu_ctx* c, const eu_kg_problem* p, int32_t table_dtype, float* scores, int32_t* rank, float* loss,
                     float* src_emb, float* rel_emb, float* dst_emb);
int eu_kg_loss_backward_dtype(eu_ctx* c, const eu_kg_problem* p, int32_t table_dtype, const float* grad_loss, const float* scores,
                              float* const* grads);
int eu_kg_loss_backward_sparse_dtype(eu_ctx* c, const eu_kg_problem* p, int32_t table_dtype, const float* grad_loss,
                                     const float* scores, int64_t* const* rows, float* const* values, int64_t* counts);

/* tf_euler.sample_edge -- TF op SampleEdge (tf_euler/kernels/sample_edge_op.cc; Graph::SampleEdge graph.cc:277-301): `count`
 * edges of ONE type drawn by the alias method over the edge weights, out i64[count,3] = (src, dst, type).  Several types or
 * -1 return EU_ERR_STATE: the reference's edge_type_collection_ is never initialised and it returns nothing for them. */
int eu_sample_edge(eu_ctx* c, int32_t count, const int32_t* types, int32_t n_types, int64_t* out);
/* tf_euler.get_edge_dense_feature / _sparse_ / _binary_ (tf_euler/kernels/get_edge_*_feature_op.cc over
 * euler::GetEdge*Feature api.cc:148-205): edges i64[E,3] = (src, dst, type); unknown edges give zeros / the default entry /
 * the empty string.  Device pointers; the ragged variants follow eu_get_sparse_feature's two-call convention. */
int eu_get_edge_dense_feature(eu_ctx* c, const int64_t* edges, int64_t E, int32_t fid, int32_t dim, float* out);
int eu_get_edge_sparse_feature(eu_ctx* c, const int64_t* edges, int64_t E, int32_t fid, int64_t default_value, int64_t cap,
                               int64_t* out_ptr, int64_t* out_values);
int eu_get_edge_binary_feature(eu_ctx* c, const int64_t* edges, int64_t E, int32_t fid, int64_t cap, int64_t* out_ptr, uint8_t* out_bytes);

/* tf_euler.get_full_neighbor core (euler::GetFullNeighbor api.cc:208-221 over Node::GetFullNeighbor node.cc:176-198):
 * for every node the edges of each requested type, in the order the types are given, as (id, weight, type); a missing
 * node has an empty list.  CSR-style output: out_ptr i64[B+1] (device) -- entries of node i are
 * [out_ptr[i], out_ptr[i+1]); only the first `cap` entries are written (cap = 0: lengths only; out_* may be NULL).
 * The _host variant takes host buffers and also returns *total = out_ptr[B]: call it with cap = 0 to size the
 * outputs, then again with cap >= *total (the reference's kernel sizes its SparseTensor the same way,
 * tf_euler/kernels/get_full_neighbor_op.cc). */
int eu_get_full_neighbor(eu_ctx* c, const int64_t* nodes, int64_t B, const int32_t* etypes, int32_t K,
                         int64_t cap, int64_t* out_ptr, int64_t* out_ids, float* out_w,
                         int32_t* out_t);
int eu_get_full_neighbor_host(eu_ctx* c, const int64_t* nodes, int64_t B, const int32_t* etypes, int32_t K,
                              int64_t cap, int64_t* out_ptr, int64_t* out_ids, float* out_w, int32_t* out_t,
                              int64_t* total);

/* tf_euler.get_sorted_full_neighbor (neighbor_ops.py:100-119; Node::GetSortedFullNeighbor node.cc:210-262; engine
 * "order_by id asc", euler/core/kernels/get_neighbor_op.cc:128-141): eu_get_full_neighbor with every node's entries ordered
 * by neighbor id ascending (ties keep the listing order).  Same convention (cap = 0: lengths only; cap must cover the listing). */
int eu_get_sorted_full_neighbor(eu_ctx* c, const int64_t* nodes, int64_t B, const int32_t* etypes, int32_t K,
                                int64_t cap, int64_t* out_ptr, int64_t* out_ids, float* out_w, int32_t* out_t);
/* tf_euler.get_top_k_neighbor (neighbor_ops.py:44-46; tf_euler/kernels/get_top_k_neighbor_op.cc:54-121; engine "order_by
 * weight desc, limit k"): dense [B,k] outputs, heaviest edge first, default_node / 0.0 / -1 fill.  Device pointers; synchronises
 * the stream once (scratch is sized from the listing length). */
int eu_get_top_k_neighbor(eu_ctx* c, const int64_t* nodes, int64_t B, const int32_t* etypes, int32_t K, int32_t k,
                          int64_t default_node, int64_t* out_ids, float* out_w, int32_t* out_t);
/* tf_euler.sample_neighbor_layerwise (neighbor_ops.py:72-77; tf_euler/kernels/sample_neighbor_layerwise_with_adj_op.cc:54-150 over
 * API_LOCAL_SAMPLE_L, euler/core/kernels/local_sample_layer_op.cc:41-140): nodes i64[batch, n]; per batch row `count` neighbors
 * drawn from the union of the rows' neighbor lists, candidates unique by (dst, type) with summed weights (weight_func 1 = sqrt),
 * out_nb i64[batch, count] (default_node when the union is empty); out_adj (may be NULL) f32[batch, n, count] = 1.0 where
 * out_nb[b, k] is a neighbor of nodes[b, j] -- the dense view of the op's SparseTensor.  Same candidate set, weights and
 * distribution as the reference; the candidate ORDER (an unordered_map<string> artefact upstream) is (dst, type) here.
 * Device pointers; synchronises (scratch is sized from the listing). */
int eu_sample_neighbor_layerwise(eu_ctx* c, const int64_t* nodes, int64_t batch, int32_t n, const int32_t* etypes, int32_t K,
                                 int32_t count, int64_t default_node, int32_t weight_func, int64_t* out_nb, float* out_adj);
/* tf_euler.sparse_get_adj (neighbor_ops.py:33-36; euler/core/kernels/sparse_get_adj_op.cc:34-90): nodes i64[batch, N],
 * nb_nodes i64[batch, M] -> out_adj f32[batch, N, M] = 1.0 where an edge nodes[b, j] -> nb_nodes[b, k] of a listed type exists
 * (dense view of the SparseTensor). */
int eu_sparse_get_adj(eu_ctx* c, const int64_t* nodes, const int64_t* nb_nodes, int64_t batch, int32_t N, int32_t M,
                      const int32_t* etypes, int32_t K, float* out_adj);
/* tf_euler.sparse_get_adj as the reference's SparseTensor itself (tf_euler/kernels/sparse_get_adj_op.cc:84-117): same inputs
 * and membership rule as eu_sparse_get_adj.  Entry (b, j, k) with value 1 iff nb_nodes[b, k] is among the listed neighbors of
 * nodes[b, j]: a neighbor listed several times gives one entry, an id repeated in nb_nodes[b] one entry per position k.  Every
 * batch row without an entry (b, N-1, M-1) gets that entry with value 0 (the reference's filler, which gives the dense shape
 * [batch, N, M]).  Entries in row-major (b, j, k) order:
 *   out_ptr     i64[batch*N + 1]  entries of row (b, j) are [out_ptr[b*N + j], out_ptr[b*N + j + 1])
 *   out_indices i64[nnz, 3]       (b, j, k)
 *   out_values  i64[nnz]          1, or 0 for a filler
 * Two calls, like eu_get_full_neighbor: cap = 0 computes out_ptr only; read nnz = out_ptr[batch*N] and call again with cap = nnz.
 * Cost after the listing: O(listed entries + nnz + M log M) per batch row, balanced by listed entries.  Device pointers;
 * synchronises (scratch is sized from the listing, and the second call checks cap).  2^31 or more listed entries, node rows,
 * neighbor slots or entries return EU_ERR_UNSUPPORTED. */
int eu_sparse_get_adj_coo(eu_ctx* c, const int64_t* nodes, const int64_t* nb_nodes, int64_t batch, int32_t N, int32_t M,
                          const int32_t* etypes, int32_t K, int64_t cap, int64_t* out_ptr, int64_t* out_indices,
                          int64_t* out_values);
/* tf_euler.gen_pair (tf_euler/kernels/gen_pair_op.cc:41-100): skip-gram pairs of walks.  paths i64[B,path_len] ->
 * out i64[B, eu_gen_pair_count(path_len, lw, rw), 2] (device pointers). */
int64_t eu_gen_pair_count(int32_t path_len, int32_t left_win_size, int32_t right_win_size);
int eu_gen_pair(eu_ctx* c, const int64_t* paths, int64_t B, int32_t path_len, int32_t left_win_size, int32_t right_win_size,
                int64_t* out);

/* euler::GetNodeType (euler/core/api/api.cc:50-61; tf_euler get_node_type): type of every node, INT32_MIN
 * (DEFAULT_INT32, euler/common/data_types.cc:23) for ids that are not in the graph. */
int eu_get_node_type(eu_ctx* c, const int64_t* nodes, int64_t B, int32_t* out);
int eu_get_node_type_host(eu_ctx* c, const int64_t* nodes, int64_t B, int32_t* out);
/* Node::GetWeight (euler/core/graph/node.h:78) of every node, 0.0 for ids that are not in the graph (host buffers). */
int eu_get_node_weight_host(eu_ctx* c, const int64_t* nodes, int64_t B, float* out);

/* tf.unique on the device (UniqueDataFlow / SageDataFlow, tf_euler/python/dataflow/neighbor_dataflow.py:84-109): the
 * distinct values of ids in order of FIRST occurrence and, per input, the index of its value in that list.
 * uniq: device i64[n] (first *n_unique valid), inverse: device i32[n], n_unique: device i64[1] (may be NULL). */
int eu_unique(eu_ctx* c, const int64_t* ids, int64_t n, int64_t* uniq, int32_t* inverse, int64_t* n_unique);

/* One full-neighbor hop of the full-neighborhood minibatch constructions, fused: list every neighbor of the n frontier
 * nodes (eu_get_full_neighbor's listing: E entries, row-major, types in the order given), renumber the listed ids by
 * first occurrence (tf.unique) and emit the hop's edges in the new numbering.
 *   GCNDataFlow (tf_euler/python/dataflow/gcn_dataflow.py:34-48 + neighbor_dataflow.py:84-110):
 *       flags = EU_HOP_APPEND_FRONTIER [| EU_HOP_SELF_LOOPS]
 *   RelationDataFlow (relation_dataflow.py:31-71): flags = EU_HOP_APPEND_FRONTIER, out_t = the block's e_id
 *   get_multi_hop_neighbor (tf_euler/python/euler_ops/neighbor_ops.py:209-242): flags = EU_HOP_SORT, out_w = the values
 * EU_HOP_APPEND_FRONTIER: the unique runs over concat(listing, nodes) instead of the listing alone.
 * EU_HOP_SELF_LOOPS (needs APPEND, excludes SORT): n self-loop edges (k, position of nodes[k]) follow the E entries.
 * EU_HOP_SORT: within each node's row the entries (cols, weights) are ordered by column, ties in listing order
 *   (tf.sparse_reorder of the (row, col) SparseTensor); rows are unchanged.
 * Device pointers; W = E + n with SELF_LOOPS, E otherwise:
 *   out_ptr  i64[n+1]  listing offsets: the entries of node i are [out_ptr[i], out_ptr[i+1])
 *   out_uniq i64[E (+n with APPEND)]  the next frontier, first *n_unique valid; n_unique i64[1]
 *   out_rows i64[W]    each edge's row (index into nodes)                                  (may be NULL)
 *   out_cols i64[W]    each edge's column (index into out_uniq)
 *   out_w    f32[E]    each entry's weight                                                 (may be NULL)
 *   out_t    i32[E]    each entry's edge type, not with SORT                               (may be NULL)
 *   out_res  i64[n]    APPEND only: the position of every frontier node in out_uniq       (may be NULL)
 * Two calls, like eu_get_full_neighbor: with cap = 0 and out_uniq = NULL only out_ptr is computed; read E = out_ptr[n],
 * size the outputs and call again with cap = E (cap must equal the listing's total; the second call recomputes out_ptr).
 * No host synchronisation.  A hop whose E (+ n with APPEND) reaches 2^31 returns EU_ERR_UNSUPPORTED (the reference's
 * tf.unique and row indices are int32). */
enum { EU_HOP_APPEND_FRONTIER = 1, EU_HOP_SELF_LOOPS = 2, EU_HOP_SORT = 4 };
int eu_full_neighbor_hop(eu_ctx* c, const int64_t* nodes, int64_t n, const int32_t* etypes, int32_t K, int32_t flags,
                         int64_t cap, int64_t* out_ptr, int64_t* out_uniq, int64_t* n_unique, int64_t* out_rows,
                         int64_t* out_cols, float* out_w, int32_t* out_t, int64_t* out_res);

/* ------------------------------------------------------------------ message-passing ops ------ */
/* MPGather / MPScatterAdd / MPScatterMax (tf_euler/ops/mp_ops.cc:22-81; kernels
 * tf_euler/kernels/gather_op.cc:31-52, scatter_op.cc:32-92).  f32 data, i32 indices, as registered. */
int eu_gather(eu_ctx* c, const float* params, int64_t N, int64_t D, const int32_t* idx, int64_t E,
              float* out);
/* scatter_add (and scatter_mean): a non-decreasing idx sums each row in index order, bit for bit the reference's result.  Any
 * other idx sums with float atomics in no fixed order, within 1e-5 of the sum of |updates| per entry, plus an absolute error
 * below 2 * 2^-126 per update: the atomics flush subnormal updates and partial sums to zero. */
int eu_scatter_add(eu_ctx* c, const float* updates, int64_t D, const int32_t* idx, int64_t E,
                   int64_t size, float* out);
/* scatter_max: out initialised to -1e9 and raised by strict `upd > out`, so NaN never wins and values at or below -1e9 leave
 * -1e9.  A non-decreasing idx gives the reference's result bit for bit.  Any other idx gives the same bits except among equal
 * zeros: there +0.0 wins over -0.0 whatever their order (the reference keeps the first); -0.0 beats every negative value. */
int eu_scatter_max(eu_ctx* c, const float* updates, int64_t D, const int32_t* idx, int64_t E,
                   int64_t size, float* out);
/* scatter_mean (tf_euler/python/euler_ops/mp_ops.py:65-69): add / (add(ones) + 1e-7) */
int eu_scatter_mean(eu_ctx* c, const float* updates, int64_t D, const int32_t* idx, int64_t E,
                    int64_t size, float* out);
/* Fused SAGE aggregation for fixed-fanout blocks (sage_dataflow.py:43-46 edge_src = repeat(range(B),count)):
 * out[r,:] = mean_{j<count} x(nbr_ids[r*count+j]) with scatter_mean's (count + 1e-7) divisor, summed in ascending j, where
 * x(id) f32[dim] is columns [0, min(dim, feat_dim)) of id's whole stored feature row (every slot, concatenated), zeros beyond,
 * and all zeros for an id not in the graph (default fill).  x(id) equals get_dense_feature(id, slot 0, dim) when the graph has
 * one slot or dim <= slot 0's width; otherwise it reads the later slots' columns where get_dense_feature zero-fills. */
int eu_sage_mean_aggregate(eu_ctx* c, const int64_t* nbr_ids, int64_t rows, int32_t count,
                           int32_t dim, float* out);
int eu_sage_mean_aggregate_host(eu_ctx* c, const int64_t* nbr_ids, int64_t rows, int32_t count,
                                int32_t dim, float* out);
/* the same block with aggr = 'add' (scatter_add, tf_euler/kernels/scatter_op.cc:44-55): out[r,:] = sum_j x(nbr_ids[r*count+j]),
 * x as above */
int eu_sage_add_aggregate(eu_ctx* c, const int64_t* nbr_ids, int64_t rows, int32_t count, int32_t dim, float* out);
/* the three above into out of out_dtype (the rule of eu_get_dense_feature_out_dtype): sums and the (count + 1e-7) division in
 * f32 as the f32 calls do them, each value rounded once at the store; a repeated segment's copies and the zero rows of
 * segments without a neighbour are the same bits as its own row / +0.0 */
int eu_sage_mean_aggregate_out_dtype(eu_ctx* c, const int64_t* nbr_ids, int64_t rows, int32_t count, int32_t dim, int32_t out_dtype,
                                     void* out);
int eu_sage_mean_aggregate_host_out_dtype(eu_ctx* c, const int64_t* nbr_ids, int64_t rows, int32_t count, int32_t dim,
                                          int32_t out_dtype, void* out);
int eu_sage_add_aggregate_out_dtype(eu_ctx* c, const int64_t* nbr_ids, int64_t rows, int32_t count, int32_t dim, int32_t out_dtype,
                                    void* out);
/* GATConv's attention aggregation (tf_euler/python/convolution/gat_conv.py:53-78, aggr = 'add', after its `fc`), fused.
 * H = heads, C = head_dim; inputs h_src f32[n_src, H*C] (heads concatenated per row), s_dst f32[n_dst, H] and
 * s_src f32[n_src, H] (the per-node scores att_i(x), att_j(x)), dst / src i32[E] (edge_index[0] / [1]).  For head h:
 *   u[e,h]     = leaky_relu(s_dst[dst_e,h] + s_src[src_e,h], 0.2)
 *   alpha[e,h] = scatter_softmax(u, dst, n_dst)        (running max from -1e9, as scatter_max: a target whose logits are
 *                                                       all below -1e9 gets NaN alphas)
 *   out[i, h*C:(h+1)*C] = sum over the edges e with dst_e = i of alpha[e,h] * h_src[src_e, h*C:(h+1)*C]
 * out f32[n_dst, H*C] (a target without edges gets a zero row); alpha f32[E, H] may be NULL (not written).
 * For non-decreasing dst, out and alpha equal bit for bit gather -> add -> leaky_relu -> scatter_softmax -> multiply ->
 * scatter_add composed from the ops above: every sum runs left to right in edge order.  Unsorted dst is ordered by a stable
 * sort first: the result is bit-identical to the call on the stably sorted edge list.
 * The backward pass takes the forward's alpha and the gradient of out, grad_out f32[n_dst, H*C], and writes
 *   grad_h_src f32[n_src, H*C], grad_s_dst f32[n_dst, H], grad_s_src f32[n_src, H]
 * with d_alpha = <grad_out[dst_e, h-slice], h_src[src_e, h-slice]> and du = alpha * (d_alpha - sum_seg alpha * d_alpha) *
 * (u > 0 ? 1 : 0.2); per-target sums run over the dst order, per-source sums over a stable sort of the edges by src, each
 * in edge order: deterministic, no atomics.  Rows without edges get zeros.
 * heads < 1, head_dim < 1, negative sizes, edges with n_dst or n_src = 0, or a NULL pointer that is needed: EU_ERR_INVALID;
 * 2^31 or more edges, rows or H*C columns: EU_ERR_UNSUPPORTED.  Indices are not checked (as eu_gather).  Device pointers;
 * both calls synchronise the stream once to read whether dst is sorted (an unsorted dst costs a radix sort, a sorted one
 * nothing more), and they use the ctx scratch. */
int eu_gat_aggregate(eu_ctx* c, const float* h_src, const float* s_dst, const float* s_src, const int32_t* dst, const int32_t* src,
                     int64_t E, int64_t n_dst, int64_t n_src, int32_t heads, int32_t head_dim, float* out, float* alpha);
int eu_gat_aggregate_backward(eu_ctx* c, const float* grad_out, const float* h_src, const float* alpha, const float* s_dst,
                              const float* s_src, const int32_t* dst, const int32_t* src, int64_t E, int64_t n_dst, int64_t n_src,
                              int32_t heads, int32_t head_dim, float* grad_h_src, float* grad_s_dst, float* grad_s_src);
/* AGNNConv's cosine-attention aggregation (tf_euler/python/convolution/agnn_conv.py:32-54, aggr = 'add'), fused.
 * Inputs x_src f32[n_src, dim] (the rows summed), nrm_dst f32[n_dst, dim] and nrm_src f32[n_src, dim] (the l2-normalized
 * target and source rows; the op does not require them to be normalized), beta f32[1] (a device pointer: the trainable
 * scalar is never read on the host), dst / src i32[E] (edge_index[0] / [1]):
 *   cos[e]   = <nrm_dst[dst_e], nrm_src[src_e]>   (fixed order: lane l of a power-of-two group G = min(32, pow2 >=
 *              ceil(dim/4)) accumulates its 4-column chunks l, l + G, ... left to right with one fused multiply-add per
 *              column, then a butterfly over the lanes at xor distances G/2 .. 1; the same on every path)
 *   u[e]     = beta * cos[e]                      (one rounded multiply)
 *   alpha[e] = scatter_softmax(u, dst, n_dst)     (running max from -1e9, as scatter_max: a target whose logits are all
 *                                                  below -1e9 gets NaN alphas)
 *   out[i]   = sum over the edges e with dst_e = i of alpha[e] * x_src[src_e]
 * out f32[n_dst, dim] (a target without edges gets a zero row); alpha f32[E] and cos f32[E] may each be NULL (not written).
 * Given u, the softmax and the sum are those of eu_gat_aggregate with one head: for non-decreasing dst, out and alpha equal
 * bit for bit beta * cos -> scatter_softmax -> multiply -> scatter_add composed from the ops above, fed this op's cos.  Unsorted
 * dst is ordered by a stable sort first: bit-identical to the call on the stably sorted edge list.
 * The backward pass takes the forward's alpha and cos and grad_out f32[n_dst, dim], and writes grad_x_src f32[n_src, dim],
 * grad_nrm_dst f32[n_dst, dim], grad_nrm_src f32[n_src, dim] and grad_beta f32[1] (device):
 *   d_alpha[e] = <grad_out[dst_e], x_src[src_e]> (the order of cos), du[e] = alpha[e] * (d_alpha[e] - sum_seg alpha * d_alpha),
 *   grad_nrm_dst[i] = sum_{dst_e = i} (beta * du[e]) * nrm_src[src_e],  grad_nrm_src[j] = sum_{src_e = j} (beta * du[e]) * nrm_dst[dst_e],
 *   grad_x_src[j]   = sum_{src_e = j} alpha[e] * grad_out[dst_e],      grad_beta = sum_i (sum_{dst_e = i} du[e] * cos[e]);
 * per-target sums run over the dst order, per-source sums over a stable sort of the edges by src, each in edge order, and
 * grad_beta adds the per-target sums in a fixed order: deterministic, no atomics.  Rows without edges get zeros.
 * dim < 1, negative sizes, edges with n_dst or n_src = 0, or a NULL pointer that is needed: EU_ERR_INVALID; 2^31 or more
 * edges or rows: EU_ERR_UNSUPPORTED.  Indices are not checked (as eu_gather).  Device pointers; both calls synchronise the
 * stream once to read whether dst is sorted (an unsorted dst costs a radix sort), and they use the ctx scratch: forward
 * 4 B per edge when alpha is NULL; backward 4 B per edge + 4 B per target + a sort by src (12 B per edge + cub's temporary
 * storage), and a sort by dst as well when dst is unsorted. */
int eu_agnn_aggregate(eu_ctx* c, const float* x_src, const float* nrm_dst, const float* nrm_src, const float* beta,
                      const int32_t* dst, const int32_t* src, int64_t E, int64_t n_dst, int64_t n_src, int32_t dim, float* out,
                      float* alpha, float* cos);
int eu_agnn_aggregate_backward(eu_ctx* c, const float* grad_out, const float* x_src, const float* nrm_dst, const float* nrm_src,
                               const float* beta, const float* alpha, const float* cos, const int32_t* dst, const int32_t* src,
                               int64_t E, int64_t n_dst, int64_t n_src, int32_t dim, float* grad_x_src, float* grad_nrm_dst,
                               float* grad_nrm_src, float* grad_beta);
/* RelationConv's typed mean aggregation (tf_euler/python/convolution/relation_conv.py:53-70, aggr = 'mean', up to
 * apply_node), fused.  R = num_relations, D = dim, F = fea_dim; inputs x_src f32[n_src, F], matrix f32[R, D, F],
 * rel i32[E] (each edge's relation, edge_attr upstream), dst / src i32[E] (edge_index[0] / [1]):
 *   out[i] = (sum over the edges e with dst_e = i of matrix[rel_e] . x_src[src_e]) / fl(cnt_i + 1e-7)
 * out f32[n_dst, D]; the divisor is scatter_mean's (the f32 edge count plus 1e-7f, one rounded division), so a target without
 * edges gets a zero row.  The edges are summed by pair p = (target, relation) before the transform, which runs once per pair:
 *   S_p = sum over the edges of p of x_src[src_e]   (fixed order: the pair's edges in key order, in chunks of 256 counted from
 *                                                    its first edge, each chunk left to right from +0, then the chunk sums in
 *                                                    chunk order)
 *   out[i, d] = (one fused multiply-add chain over the pairs of i in key order and f ascending of matrix[r_p, d, f] * S_p[f])
 *               / fl(cnt_i + 1e-7)
 * so the result differs from a per-edge matvec only in rounding (it is equal on inputs whose sums are exact).  Keys (dst, rel)
 * that are non-decreasing (as RelationDataFlow lists them) are walked as given; otherwise a stable radix sort on
 * dst * R + rel orders the edges first: the result is bit-identical to the call on the stably sorted edge list.
 * The backward pass takes grad_out f32[n_dst, D] and writes grad_x_src f32[n_src, F] and grad_matrix f32[R, D, F]; rel gets
 * no gradient.  With gm_i = grad_out[i] / fl(cnt_i + 1e-7):
 *   gS_p = matrix[r_p]^T . gm_i(p) (a chain over d ascending),  grad_x_src[j] = sum over the edges e with src_e = j of gS_pair(e)
 *   (a stable sort of the edges by src, each source's edges in order),  grad_matrix[r] = sum over the pairs p with r_p = r of
 *   gm_i(p) (x) S_p (the pairs in stable relation order, chunks of 256 pairs, the chunk sums in chunk order).
 * Deterministic, no atomics; sources and relations without edges get zeros.
 * num_relations, dim or fea_dim < 1, negative sizes, edges with n_dst or n_src = 0, a NULL pointer that is needed, or a
 * relation outside [0, R): EU_ERR_INVALID (the relations are checked in the pass that checks the order: a bad one would read
 * outside matrix).  2^31 or more edges, rows or matrix entries: EU_ERR_UNSUPPORTED.  dst and src are not checked (as eu_gather).
 * Device pointers; each call synchronises the stream once to read the order flags and P (the number of pairs), twice when
 * the keys are unsorted, and uses the ctx scratch: O(E) index data (8 B per edge; the backward adds 8 B per edge and a sort
 * by src of 12 B per edge plus cub's temporary storage; unsorted keys add a sort of 24 B per edge plus cub's) plus
 * O(P * (F + D)) floats, (P + E / 256) * F floats of chunk sums, and for grad_matrix one D x F block per 256 pairs of a
 * relation; never O(E * D). */
int eu_relation_aggregate(eu_ctx* c, const float* x_src, const float* matrix, const int32_t* rel, const int32_t* dst,
                          const int32_t* src, int64_t E, int64_t n_dst, int64_t n_src, int32_t num_relations, int32_t dim,
                          int32_t fea_dim, float* out);
int eu_relation_aggregate_backward(eu_ctx* c, const float* grad_out, const float* x_src, const float* matrix, const int32_t* rel,
                                   const int32_t* dst, const int32_t* src, int64_t E, int64_t n_dst, int64_t n_src,
                                   int32_t num_relations, int32_t dim, int32_t fea_dim, float* grad_x_src, float* grad_matrix);
/* DNAConv's attention aggregation (tf_euler/python/convolution/dna_conv.py:115-170, aggr = 'mean'), fused, after the
 * per-node linear maps.  H = heads, C = head_dim, dim = H * C; inputs q f32[n_dst, dim] (lin_q(in_fc(x_target))), k and v
 * f32[n_src, dim] (lin_k / lin_v(in_fc(x_source))), n0 f32[n_dst] and n1 f32[n_src] (gcn_norm's deg^-1/2 of both sides),
 * dst / src i32[E] (edge_index[0] / [1]).  For edge e = (i, j) = (dst_e, src_e) and heads h, h':
 *   s[e,h,h']  = <q_i[h], k_j[h']> / sqrtf(C)   (every query head against every key head; the dot in a fixed order: lane l
 *                of a power-of-two group G = min(32, pow2 >= ceil(C/4)) accumulates its 4-column chunks l, l + G, ... left
 *                to right with one fused multiply-add per column, then a butterfly over the lanes at xor distances G/2 .. 1,
 *                as eu_agnn_aggregate's cos; then one rounded division)
 *   m[e,h]     = max(0, max_h' s[e,h,h'])
 *   a[e,h,h']  = expf(s - m) / (sum over h'' ascending of expf(s[e,h,h''] - m) + expf(-m))   (restricted_softmax)
 *   msg[e,h,:] = fl(n0_i * n1_j) * (sum over h' ascending of a[e,h,h'] * v_j[h']: one multiply, then fused multiply-adds)
 *   out_i      = (sum over the edges of i of msg_e) / fl(fl(cnt_i) + 1e-7f)   (scatter_mean's divisor; no edge: a zero row)
 * A target's edges are summed in order (dst order; unsorted dst is ordered by a stable sort first, so the result is
 * bit-identical to the call on the stably sorted edge list) in chunks of 256 counted from its first edge, each chunk left to
 * right from +0, then the chunk sums in chunk order.  For H = 1 and targets of at most 256 edges, given alpha, out equals
 * gather -> multiply by alpha -> multiply by the norm product -> scatter_mean composed from the ops above, bit for bit.
 * out f32[n_dst, dim]; alpha f32[E, H, H] may be NULL (not written).
 * The backward pass takes the forward's alpha and grad_out f32[n_dst, dim], and writes grad_q f32[n_dst, dim], grad_k and
 * grad_v f32[n_src, dim]; n0 and n1 get no gradient.  With gm_i = grad_out[i] / fl(cnt_i + 1e-7) and w_e = fl(n0_i * n1_j):
 *   da = w_e * <gm_i[h], v_j[h']> (the order of s),  t = a * (da - sum_h'' a * da) / sqrtf(C),
 *   grad_q_i[h] = sum_{dst_e = i} sum_h' t * k_j[h'],  grad_k_j[h'] = sum_{src_e = j} sum_h t * q_i[h],
 *   grad_v_j[h'] = sum_{src_e = j} w_e * sum_h a * gm_i[h]
 * each segment sum chunked as the forward's, per-target over the dst order, per-source over a stable sort of the edges by
 * src: deterministic, no atomics.  Rows without edges get zeros.
 * heads or head_dim < 1, negative sizes, edges with n_dst or n_src = 0, or a NULL pointer that is needed: EU_ERR_INVALID.
 * heads > 8 (one edge's scores of a head are held in registers), 2^31 or more edges, rows or dim columns: EU_ERR_UNSUPPORTED.
 * Indices are not checked (as eu_gather).  Device pointers; both calls synchronise the stream once to read whether dst is
 * sorted (an unsorted dst costs a radix sort, a sorted one nothing more), and they use the ctx scratch: forward 4 H^2 B per
 * edge when alpha is NULL, 12 B per target and (n_dst + E / 256) * dim floats of chunk sums; backward n_dst * dim floats,
 * 4 H^2 B per edge, a sort by src (12 B per edge plus cub's temporary storage) and the chunk sums of both sides; never
 * O(E * dim). */
int eu_dna_aggregate(eu_ctx* c, const float* q, const float* k, const float* v, const float* n0, const float* n1, const int32_t* dst,
                     const int32_t* src, int64_t E, int64_t n_dst, int64_t n_src, int32_t heads, int32_t head_dim, float* out,
                     float* alpha);
int eu_dna_aggregate_backward(eu_ctx* c, const float* grad_out, const float* q, const float* k, const float* v, const float* n0,
                              const float* n1, const float* alpha, const int32_t* dst, const int32_t* src, int64_t E, int64_t n_dst,
                              int64_t n_src, int32_t heads, int32_t head_dim, float* grad_q, float* grad_k, float* grad_v);
/* The neighbour mean over a CSR adjacency: what GCNAggregator and MeanAggregator of the sparse aggregators compute before
 * their dense layers (tf_euler/python/utils/sparse_aggregators.py:37-84: the weights replaced by ones, sparse_reduce_sum,
 * sparse_tensor_dense_matmul, maximum(degree, 1e-7)).  Inputs x_neigh f32[m, dim] and the adjacency of n rows as
 * eu_full_neighbor_hop's EU_HOP_SORT outputs give it, indptr i64[n+1] (indptr[0] = 0, indptr[n] = nnz) and cols i64[nnz]
 * (the weights are not read).  For row i with deg_i = indptr[i+1] - indptr[i] entries (multi-edges counted):
 *   S_i    = sum over k in [indptr[i], indptr[i+1]) of x_neigh[cols[k], :]   (fixed order: the row cut into chunks of 256
 *            entries counted from its first one, each chunk summed left to right from +0, the chunk sums of a row of
 *            several chunks added in chunk order from +0)
 *   out[i] = __fdiv_rn(S_i, max(fl(deg_i), 1e-7f))   (one IEEE-rounded division; a row without entries gives a zero row)
 * out f32[n, dim].  A row of at most 256 entries thus gets the bits of the plain left-to-right float32 sum.  The float4 and
 * scalar paths (dim % 4 == 0 with x_neigh and out 16-byte aligned, or not) give the same bits.  No host synchronisation;
 * ctx scratch of 12 B per row and (n + nnz / 256) * dim floats of chunk sums, which grows only with the sizes (a forward
 * at sizes already seen is capturable in a CUDA graph).
 * The backward pass takes grad_out f32[n, dim] and writes grad_x f32[m, dim] (zeroed first; columns without entries stay
 * zero): with gs_i = __fdiv_rn(grad_out[i], max(fl(deg_i), 1e-7f)),
 *   grad_x[j] = sum over the entries k with cols[k] = j of gs[row of k]
 * summed as the id-table gradients of eu_sparse_embedding_lookup_backward are: the entries of column j in stable row
 * order, chunks of 256 from +0, the chunk sums in chunk order.  Deterministic, no atomics, no host synchronisation; ctx
 * scratch of n * dim floats, 8 B per entry and a stable sort of the entries by column (O(nnz)).
 * Negative sizes, dim < 1, entries with n or m = 0, or a NULL pointer that is needed: EU_ERR_INVALID; n, m or nnz of 2^31
 * or more (or nnz entries whose 256-entry chunks reach 2^31): EU_ERR_UNSUPPORTED.  indptr and cols are not checked (as
 * eu_gather): indptr must be non-decreasing from 0 to nnz and cols must lie in [0, m).  Device pointers. */
int eu_adjacency_mean(eu_ctx* c, const float* x_neigh, int64_t m, const int64_t* indptr, const int64_t* cols, int64_t n,
                      int64_t nnz, int32_t dim, float* out);
int eu_adjacency_mean_backward(eu_ctx* c, const float* grad_out, const int64_t* indptr, const int64_t* cols, int64_t n,
                               int64_t nnz, int64_t m, int32_t dim, float* grad_x);
/* The adjacency of the resident graph, with engine rows as columns (layer-by-layer inference of GCNEncoder and
 * GenieEncoder: every layer one pass over the graph's edges).  Output row i lists engine row r0 + i, or rows[r0 + i] when
 * rows (i64, device) is given -- a value outside [0, n) lists nothing -- for i in [0, r1 - r0): eu_get_full_neighbor's
 * listing of that row's node (the K types in the order given, repeats repeat, multi-edges kept; an unknown type lists
 * nothing), each neighbour id replaced by its engine row (arithmetic on synthetic and sharded layouts, the id table
 * otherwise).  A listed id that is not a node of the graph gets column n + k (n = eu_graph_num_nodes), k numbering the
 * distinct such ids in first-occurrence order over THIS call's listing: each call, and so each chunk of a chunked build,
 * numbers its own; out_extra[k] is the id.
 * Two calls, like eu_get_full_neighbor:
 *   cap = 0:             out_ptr i64[r1 - r0 + 1] and counts[0] = the listed entries whose id is not a node
 *   cap = nnz = out_ptr[r1 - r0], extra_cap = counts[0]:   out_ptr again, out_cols i64[nnz], out_w f32[nnz] (optional:
 *                        cum_w differences as eu_get_full_neighbor's weights), out_extra i64[extra_cap] (the first
 *                        counts[1] hold the distinct absent ids)
 * counts is i64[2] on the device.  No host synchronisation; entries are spread over threads by entry (a hub row does not
 * serialise), the first call reads every listed id once more to count the absent ones.  ctx scratch: the scan temp, and
 * O(extra_cap) for the absent ids.  r0 > r1, r1 > n without rows, K outside [0, 32], a NULL pointer that is needed:
 * EU_ERR_INVALID; 2^31 rows or absent entries or more: EU_ERR_UNSUPPORTED.  Device pointers.
 * eu_graph_node_ids: the node ids in engine-row order, out i64[n].
 * eu_graph_node_rows: the engine row of every id, -1 for ids that are not nodes, out i64[B]. */
int eu_graph_adjacency(eu_ctx* c, const int32_t* etypes, int32_t K, const int64_t* rows, int64_t r0, int64_t r1, int64_t cap,
                       int64_t extra_cap, int64_t* out_ptr, int64_t* out_cols, float* out_w, int64_t* out_extra,
                       int64_t* counts);
int eu_graph_node_ids(eu_ctx* c, int64_t* out);
int eu_graph_node_rows(eu_ctx* c, const int64_t* nodes, int64_t B, int64_t* out);
/* The per-layer embedding stores of ScalableSageEncoder / ScalableGCNEncoder (tf_euler/python/utils/encoders.py:294-408,
 * 629-748): a store f32[n_rows, dim] and its gradient store f32[n_rows, dim], updated in place with fixed meanings for
 * repeated ids.  ids i64[M] must lie in [0, n_rows).
 * eu_store_exchange: rows f32[M, dim] in, taken f32[M, dim] out:
 *   store[ids[i]]   = rows[the LAST i with that id]      (tf.scatter_update, whose winner is unspecified upstream)
 *   taken[i]        = grad_store[ids[i]] as it was before this call, for every i (repeats included)
 *   grad_store[v]   = 0 for every id v of ids
 *   The ids are ordered stably and planned once (the id-table gradient path's plan); one lane group per distinct id then
 *   reads, copies, writes and clears its row: no atomics.  Rows no id names are untouched.
 * eu_store_accumulate: grad f32[M / count, dim]; count >= 1 divides M; pool EU_POOL_SUM or EU_POOL_MEAN:
 *   grad_store[v] = __fadd_rn(grad_store[v], S_v),  S_v = sum over the i with ids[i] = v of grad[i / count] (EU_POOL_MEAN:
 *   each element __fdiv_rn'd by fl(count) as it is read), summed as eu_shallow_encode_pool_backward sums a table gradient
 *   (stable id order, chunks of 256 from +0, the chunk sums in chunk order); S_v is the gradient of eu_shallow_encode_pool
 *   over the store as id table (count = 1: of eu_shallow_encode), added to the stored row with one rounding.
 * Both calls first check the ids (one small kernel, one stream synchronisation): an id outside [0, n_rows) returns
 * EU_ERR_INVALID before either table is written.  Under CUDA-graph capture the check is skipped and such an id touches no
 * table row (exchange: its taken row is NaN).  No other synchronisation; ctx scratch O(M) index data (plus M * dim floats
 * for eu_store_accumulate), never O(n_rows).  M = 0 does nothing.  dim < 1, n_rows < 1, negative M, a bad count or pool or a
 * NULL pointer that is needed: EU_ERR_INVALID; n_rows of 2^31 - 1 or more, or M ids whose 256-entry chunks reach 2^31:
 * EU_ERR_UNSUPPORTED.  Device pointers. */
int eu_store_exchange(eu_ctx* c, float* store, float* grad_store, int64_t n_rows, int32_t dim, const int64_t* ids, int64_t M,
                      const float* rows, float* taken);
int eu_store_accumulate(eu_ctx* c, float* grad_store, int64_t n_rows, int32_t dim, const int64_t* ids, int64_t M, int32_t count,
                        int32_t pool, const float* grad);
/* The same two over a store pair of storage type dtype (eu_feat_dtype; store and grad_store both have it; rows, taken and
 * grad stay f32).  EU_FEAT_F32 is the call above (seed, step and tensor unused).  With EU_FEAT_BF16 every read widens a
 * stored element exactly to f32 and only the writes round:
 *   exchange:    store[v] = the round to nearest even of rows[the last i with that id] (an overwrite: no seed); taken[i] =
 *                the pre-clear gradient row widened, f32; the cleared rows are exact zeros.
 *   accumulate:  grad_store[v] = SR(__fadd_rn(widen(grad_store[v]), S_v)), S_v the f32 call's sum, SR the stochastic
 *                rounding of eu_optim_*_dtype: the low 16 bits of word 0 of Philox4x32-10 with counter (element lo,
 *                element hi, *step mod 2^32, tensor) and key seed, element = v * dim + f (64-bit), are added to the low half
 *                of the f32 bits, which are then dropped.  step is a device int64 read on the device, so a captured graph
 *                replays with the live counter.  Rows no id names keep their bits.
 * The 4-wide path needs dim % 4 == 0, the bf16 tables 8-byte aligned and rows / taken 16-byte aligned; otherwise scalar
 * accesses give the same bits.  An unknown dtype, or eu_store_accumulate_dtype with EU_FEAT_BF16 and no step:
 * EU_ERR_INVALID before any device work; every other bound and status as above. */
int eu_store_exchange_dtype(eu_ctx* c, void* store, void* grad_store, int64_t n_rows, int32_t dim, const int64_t* ids, int64_t M,
                            const float* rows, float* taken, int32_t dtype);
int eu_store_accumulate_dtype(eu_ctx* c, void* grad_store, int64_t n_rows, int32_t dim, const int64_t* ids, int64_t M,
                              int32_t count, int32_t pool, const float* grad, int32_t dtype, uint64_t seed, const int64_t* step,
                              int32_t tensor);
int eu_gather_host(eu_ctx* c, const float* params, int64_t N, int64_t D, const int32_t* idx,
                   int64_t E, float* out);
int eu_scatter_add_host(eu_ctx* c, const float* updates, int64_t D, const int32_t* idx, int64_t E,
                        int64_t size, float* out);
int eu_scatter_max_host(eu_ctx* c, const float* updates, int64_t D, const int32_t* idx, int64_t E,
                        int64_t size, float* out);

/* ------------------------------------------------------------------ sharding (multi-GPU) ----- */
/* Replace ID_SPLIT / IDX_MERGE / DATA_MERGE (euler/core/kernels/id_split_op.cc:46-99, idx_merge_op.cc:32-78)
 * either side of an all-to-all.  eu_shard_bucket: stable counting sort of ids by owner
 * (id % num_partitions) % shard_num; sorted_ids[k] came from ids[src_index[k]]; counts[o] / offsets[o]
 * (device, i64[shard_num] / [shard_num+1]) delimit owner o's segment.  eu_shard_merge_sample: replies in
 * sorted order -> original row order + TF packing + engine-id frontier.  eu_shard_merge_rows: the same for
 * fixed-width f32 rows (features). */
int eu_shard_bucket(eu_ctx* c, const int64_t* ids, int64_t rows, int32_t num_partitions, int32_t shard_num,
                    int32_t self_shard, int64_t* sorted_ids, int32_t* src_index, int64_t* counts, int64_t* offsets);
/* ids 0 and 2^64-1 (placeholder / default fill) exist nowhere and are routed to self_shard.
 * eu_shard_pack_sample: (ids, w, t)[n] -> n 16-byte records {id, w | t << 32} so one all-to-all carries a reply;
 * eu_shard_merge_sample consumes records in sorted order. */
int eu_shard_pack_sample(eu_ctx* c, const int64_t* ids, const float* w, const int32_t* t, int64_t n, int64_t* packed);
int eu_shard_merge_sample(eu_ctx* c, const int64_t* packed, const int32_t* src_index, int64_t rows, int32_t count,
                          int64_t default_node, int64_t* eng_ids, int64_t* out_ids, float* out_w, int32_t* out_t);
int eu_shard_merge_rows(eu_ctx* c, const float* rows_in, const int32_t* src_index, int64_t rows, int64_t D,
                        float* out);

/* Peer-memory exchange (csrc/p2p.cu): the all-to-all of a hop / feature fetch done by the kernels themselves over
 * NVLink peer mappings -- no NCCL call, no host sync, CUDA-graph capturable.  One eu_sym per (ctx, rank): a symmetric
 * region exported with cudaIpc; all_gather the 64-byte handles (any out-of-band channel) and eu_sym_connect.
 * Results land in the rank's own symmetric output arrays (eu_sym_outputs), already in request order. */
typedef struct eu_sym eu_sym;
int eu_sym_create(eu_ctx* c, int32_t rank, int32_t world, int64_t max_rows, int32_t max_count, int64_t max_feat_rows,
                  int32_t max_dim, eu_sym** out, void* handle_out /* 64 bytes */);
int eu_sym_connect(eu_sym* s, const void* handles /* world x 64 bytes, rank order */);
int eu_sym_destroy(eu_sym* s);
int eu_sym_outputs(eu_sym* s, int64_t** eng, int64_t** ids, float** w, int32_t** t, float** rows);
int eu_sym_error(eu_sym* s, int* err);   /* 1 if a bounded wait timed out (synchronises) */
int eu_sym_sample_hop(eu_sym* s, const int64_t* seeds, int64_t rows, const int32_t* etypes, int32_t K, int32_t count,
                      int64_t default_node, int32_t num_partitions, int32_t want_packed);
/* nb independent batches per exchange: seeds i64[nb][rows], outputs [nb][rows][count]; batch g is sampled by every
 * shard's engine g (eu_ctx_set_engines) over the requests of rank 0..N-1 for that batch, its own dedup scope. */
int eu_sym_sample_hop_batched(eu_sym* s, const int64_t* seeds, int32_t nb, int64_t rows, const int32_t* etypes, int32_t K,
                              int32_t count, int64_t default_node, int32_t num_partitions, int32_t want_packed);
int eu_sym_get_dense_feature(eu_sym* s, const int64_t* ids, int64_t rows, int32_t fid, int32_t dim, int32_t num_partitions);
/* Sharded eu_sage_mean_aggregate: REMOTE get_dense_feature (euler/core/kernels/remote_op.cc:60-146) fused with the
 * scatter_mean that follows it (tf_euler/python/euler_ops/mp_ops.py:65-69 over sage_dataflow.py:43-46's edge_src).
 * Each owner sums the rows of ITS ids per destination (j ascending) and stores one partial row per destination in the
 * requester's region; the requester adds the partials in rank order and divides by (count + 1e-7).  rows*count ids must
 * fit the inbox (max(max_rows, max_feat_rows)) and world*rows*dim floats the feature region.  out: device f32[rows*dim]. */
int eu_sym_sage_mean(eu_sym* s, const int64_t* nbr_ids, int64_t rows, int32_t count, int32_t dim, int32_t num_partitions,
                     float* out);

/* ------------------------------------------------------------------ reference entry point ---- */
/* bool InitQueryProxy(const char* conf) -- tf_euler/utils/init_query_proxy.cc:19-36.  "k=v;k=v";
 * keys of euler/client/query_proxy.cc:41-160 that apply here: mode (local only), data_path,
 * sampler_type, data_type, shard_num(=1); new keys: device, seed, rng (minstd|philox).
 * Returns false only for an empty / malformed list (as the reference does, :22-33); load errors are
 * logged.  Creates the process-wide default graph + ctx used by the *_default accessors. */
bool InitQueryProxy(const char* conf);
eu_graph* eu_default_graph(void);
eu_ctx* eu_default_ctx(void);
int eu_set_default_graph(eu_graph* g, eu_rng_kind rng, uint64_t seed);

#ifdef __cplusplus
}
#endif
#endif /* EULER_B200_H_ */
