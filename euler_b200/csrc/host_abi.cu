// The host-buffer C ABI: every `eu_*_host` entry point.  Each one lays its caller buffers out in the ctx's staging buffers,
// uploads the inputs, runs the device entry point on the staged copies, downloads the outputs and returns once they have
// landed.  How a caller buffer reaches the device and comes back is decided in one place, HostIO.
#include <string.h>

#include <algorithm>
#include <initializer_list>
#include <vector>

#include "internal.h"

namespace eu {

// Grows the ctx's staging buffers (they never shrink).  The pinned host side is only needed for pageable caller buffers.
static int ctx_stage(eu_ctx* c, int64_t host_bytes, int64_t dev_bytes) {
  if (host_bytes > c->pin_bytes) {
    if (c->h_pin) cudaFreeHost(c->h_pin);
    c->h_pin = nullptr; c->pin_bytes = 0;
    EU_CUDA(cudaHostAlloc(&c->h_pin, (size_t)host_bytes, cudaHostAllocDefault));
    c->pin_bytes = host_bytes;
  }
  if (dev_bytes > c->stage_bytes) {
    EU_CUDA(cudaStreamSynchronize(c->stream));   // the stream may still read the old buffer
    cudaFree(c->d_stage);
    c->d_stage = nullptr; c->stage_bytes = 0;
    EU_CUDA(cudaMalloc(&c->d_stage, (size_t)dev_bytes));
    c->stage_bytes = dev_bytes;
  }
  return EU_OK;
}

// A caller's host buffer that is already page-locked (cudaHostAlloc / cudaHostRegister -- e.g. a framework's pinned
// tensor) is DMA'd directly; only pageable memory goes through the ctx's pinned staging buffer (a pageable
// cudaMemcpyAsync would serialise against the host, and the extra memcpy costs more than PCIe for wide feature rows).
static bool host_is_pinned(const void* p) {
  if (!p) return false;
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return a.type == cudaMemoryTypeHost;
}

// Host-buffer staging of one call, on the ctx stream.  in() / out() lay out one slot each, at the same offset on the
// device stage and on the pinned host stage, and register the caller buffer that goes with it (null or empty: nothing is
// copied, the slot is device-only).  Usage: lay out, begin, upload, device call, download, finish.
struct HostIO {
  eu_ctx* c;
  struct Buf { void* user; int64_t off, bytes; bool pinned; };
  std::vector<Buf> ins, outs;
  int64_t size = 0;        // bytes laid out, each slot 256-byte aligned
  bool pageable = false;   // some registered buffer is pageable: the pinned host stage is needed

  int64_t in(const void* user, int64_t bytes) { return take(ins, const_cast<void*>(user), bytes); }
  int64_t out(void* user, int64_t bytes) { return take(outs, user, bytes); }
  int begin() { return ctx_stage(c, pageable ? size : 0, size); }
  template <typename T> T* dev(int64_t off) const { return (T*)((char*)c->d_stage + off); }
  char* pin(int64_t off) const { return (char*)c->h_pin + off; }
  int upload() {
    for (const Buf& b : ins) {
      if (!b.pinned) memcpy(pin(b.off), b.user, (size_t)b.bytes);
      EU_CUDA(cudaMemcpyAsync(dev<char>(b.off), b.pinned ? b.user : pin(b.off), (size_t)b.bytes, cudaMemcpyHostToDevice, c->stream));
    }
    return EU_OK;
  }
  int download() {
    for (const Buf& b : outs)
      EU_CUDA(cudaMemcpyAsync(b.pinned ? b.user : pin(b.off), dev<char>(b.off), (size_t)b.bytes, cudaMemcpyDeviceToHost, c->stream));
    return EU_OK;
  }
  // the call's one synchronise, then the pageable outputs leave the pinned stage
  int finish() {
    EU_CUDA(cudaStreamSynchronize(c->stream));
    for (const Buf& b : outs)
      if (!b.pinned) memcpy(b.user, pin(b.off), (size_t)b.bytes);
    return EU_OK;
  }

 private:
  int64_t take(std::vector<Buf>& list, void* user, int64_t bytes) {
    const int64_t off = size;
    size += (int64_t)a256((size_t)std::max<int64_t>(bytes, 0));
    if (user && bytes > 0) {
      const bool pinned = host_is_pinned(user);
      pageable = pageable || !pinned;
      list.push_back({user, off, bytes, pinned});
    }
    return off;
  }
};

// The ragged entry points (CSR-style out_ptr + value arrays) in two HostIO rounds.  Phase 1: the nodes go up, out_ptr
// comes down, and *total = out_ptr[M].  Phase 2, only when n = min(cap, total) > 0: the first n entries of every value
// array.  It uploads the nodes again because the stage does not keep its contents when it grows, and the device call
// recomputes the lengths.  fetch(d_nodes, cap, d_ptr, d_vals) runs the device entry point on at most three value arrays;
// d_vals are all null in phase 1.
struct RaggedOut { void* user; int64_t elem_bytes; };
template <typename Fetch>
static int ragged_host(eu_ctx* c, const int64_t* nodes, int64_t M, int64_t cap, int64_t* out_ptr, int64_t* total,
                       std::initializer_list<RaggedOut> vals, const char* what, Fetch fetch) {
  if (!c || M < 0 || cap < 0 || !out_ptr || (M > 0 && !nodes)) { set_error("%s: bad argument", what); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  char* d_vals[3] = {nullptr, nullptr, nullptr};
  int rc;
  {
    HostIO io{c};
    const int64_t o_nodes = io.in(nodes, 8 * M), o_ptr = io.out(out_ptr, 8 * (M + 1));
    if ((rc = io.begin()) || (rc = io.upload())) return rc;
    if ((rc = fetch(io.dev<const int64_t>(o_nodes), 0, io.dev<int64_t>(o_ptr), d_vals))) return rc;
    if ((rc = io.download()) || (rc = io.finish())) return rc;
  }
  const int64_t tot = out_ptr[M];
  if (total) *total = tot;
  const int64_t n = std::min(cap, tot);
  if (n <= 0) return EU_OK;
  for (const RaggedOut& v : vals)
    if (!v.user) { set_error("%s: null output", what); return EU_ERR_INVALID; }
  HostIO io{c};
  const int64_t o_nodes = io.in(nodes, 8 * M), o_ptr = io.out(nullptr, 8 * (M + 1));
  int64_t o_vals[3];
  int nv = 0;
  for (const RaggedOut& v : vals) o_vals[nv++] = io.out(v.user, v.elem_bytes * n);
  if ((rc = io.begin()) || (rc = io.upload())) return rc;
  for (int k = 0; k < nv; ++k) d_vals[k] = io.dev<char>(o_vals[k]);
  if ((rc = fetch(io.dev<const int64_t>(o_nodes), n, io.dev<int64_t>(o_ptr), d_vals))) return rc;
  if ((rc = io.download())) return rc;
  return io.finish();
}

}  // namespace eu

using namespace eu;

extern "C" {

int eu_sample_fanout_batched_host(eu_ctx* c, const int64_t* nodes, int32_t nb, int64_t B, const int32_t* etypes,
                                  int32_t K, const int32_t* counts, int32_t L, int64_t default_node,
                                  int64_t* const* out_ids, float* const* out_w, int32_t* const* out_t) {
  if (!c || nb < 1 || B < 0 || L < 0 || L > 16 || !counts || (B > 0 && !nodes)) { set_error("eu_sample_fanout_host: bad argument"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  HostIO io{c};
  const int64_t o_nodes = io.in(nodes, 8 * B * nb);
  int64_t o_ids[16], o_w[16], o_t[16];
  int64_t rows = B * nb;
  for (int l = 0; l < L; ++l) {
    if (counts[l] < 0) { set_error("negative count"); return EU_ERR_INVALID; }
    rows *= counts[l];
    o_ids[l] = io.out(out_ids ? out_ids[l] : nullptr, 8 * rows);
    o_w[l] = io.out(out_w ? out_w[l] : nullptr, 4 * rows);
    o_t[l] = io.out(out_t ? out_t[l] : nullptr, 4 * rows);
  }
  int rc;
  if ((rc = io.begin()) || (rc = io.upload())) return rc;
  int64_t* d_ids[16]; float* d_w[16]; int32_t* d_t[16];
  for (int l = 0; l < L; ++l) { d_ids[l] = io.dev<int64_t>(o_ids[l]); d_w[l] = io.dev<float>(o_w[l]); d_t[l] = io.dev<int32_t>(o_t[l]); }
  if ((rc = eu_sample_fanout_batched(c, io.dev<const int64_t>(o_nodes), nb, B, etypes, K, counts, L, default_node, d_ids, d_w, d_t))) return rc;
  if ((rc = io.download())) return rc;
  return io.finish();
}

int eu_sample_fanout_host(eu_ctx* c, const int64_t* nodes, int64_t B, const int32_t* etypes,
                          int32_t K, const int32_t* counts, int32_t L, int64_t default_node,
                          int64_t* const* out_ids, float* const* out_w, int32_t* const* out_t) {
  return eu_sample_fanout_batched_host(c, nodes, 1, B, etypes, K, counts, L, default_node, out_ids, out_w, out_t);
}

int eu_sample_neighbor_host(eu_ctx* c, const int64_t* nodes, int64_t B, const int32_t* etypes,
                            int32_t K, int32_t count, int64_t default_node, int64_t* out_ids,
                            float* out_w, int32_t* out_t) {
  return eu_sample_fanout_host(c, nodes, B, etypes, K, &count, 1, default_node, &out_ids, &out_w, &out_t);
}

int eu_sample_neighbor_raw_host(eu_ctx* c, const int64_t* nodes, int64_t B, const int32_t* etypes, int32_t K, int32_t count,
                                int64_t* out_ids, float* out_w, int32_t* out_t) {
  if (!c || B < 0 || count < 0 || (B > 0 && (!nodes || (count > 0 && (!out_ids || !out_w || !out_t))))) { set_error("eu_sample_neighbor_raw_host: bad argument"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  HostIO io{c};
  const int64_t n = B * count;
  const int64_t o_nodes = io.in(nodes, 8 * B), o_ids = io.out(out_ids, 8 * n), o_w = io.out(out_w, 4 * n), o_t = io.out(out_t, 4 * n);
  int rc;
  if ((rc = io.begin()) || (rc = io.upload())) return rc;
  if ((rc = eu_sample_neighbor_raw(c, io.dev<const int64_t>(o_nodes), B, etypes, K, count, io.dev<int64_t>(o_ids), io.dev<float>(o_w), io.dev<int32_t>(o_t)))) return rc;
  if ((rc = io.download())) return rc;
  return io.finish();
}

int eu_sample_node_host(eu_ctx* c, int32_t count, const int32_t* types, int32_t n_types, int64_t* out) {
  if (!c || count < 0 || (count > 0 && !out)) { set_error("eu_sample_node_host: bad argument"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  HostIO io{c};
  const int64_t o_out = io.out(out, 8 * (int64_t)count);
  int rc;
  if ((rc = io.begin()) || (rc = io.upload())) return rc;
  if ((rc = eu_sample_node(c, count, types, n_types, io.dev<int64_t>(o_out)))) return rc;
  if ((rc = io.download())) return rc;
  return io.finish();
}

int eu_random_walk_host(eu_ctx* c, const int64_t* nodes, int64_t B, const int32_t* etypes,
                        int32_t K, int32_t L, float p, float q, int64_t default_node, int64_t* out) {
  if (!c || B < 0 || L < 0 || (B > 0 && (!nodes || !out))) { set_error("eu_random_walk_host: bad argument"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  HostIO io{c};
  const int64_t o_nodes = io.in(nodes, 8 * B), o_out = io.out(out, 8 * B * (L + 1));
  int rc;
  if ((rc = io.begin()) || (rc = io.upload())) return rc;
  if ((rc = eu_random_walk(c, io.dev<const int64_t>(o_nodes), B, etypes, K, L, p, q, default_node, io.dev<int64_t>(o_out)))) return rc;
  if ((rc = io.download())) return rc;
  return io.finish();
}

// bytes of one output element of a checked eu_feat_dtype code
static int64_t out_elem_bytes(int32_t dtype) { return dtype == EU_FEAT_BF16 ? 2 : 4; }

static int dense_feature_host(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int32_t dim, int32_t out_dtype, void* out,
                              const char* who) {
  if (!c || M < 0 || dim < 0 || (M > 0 && (!nodes || !out))) { set_error("%s: bad argument", who); return EU_ERR_INVALID; }
  if (int rc = dtype_check(out_dtype, who, "output")) return rc;
  EU_CUDA(cudaSetDevice(c->g->device));
  HostIO io{c};
  const int64_t o_nodes = io.in(nodes, 8 * M), o_out = io.out(out, out_elem_bytes(out_dtype) * M * dim);
  int rc;
  if ((rc = io.begin()) || (rc = io.upload())) return rc;
  if ((rc = out_dtype == EU_FEAT_F32
                ? eu_get_dense_feature(c, io.dev<const int64_t>(o_nodes), M, fid, dim, io.dev<float>(o_out))
                : eu_get_dense_feature_out_dtype(c, io.dev<const int64_t>(o_nodes), M, fid, dim, out_dtype, io.dev<void>(o_out)))) return rc;
  if ((rc = io.download())) return rc;
  return io.finish();
}

// eu_sage_mean_aggregate with host buffers: only the neighbor ids go up and only the [rows, dim] means come down -- the
// rows*count feature rows the unfused composition (get_dense_feature_host + scatter_mean) would move never leave HBM.
static int sage_mean_aggregate_host(eu_ctx* c, const int64_t* nbr_ids, int64_t rows, int32_t count, int32_t dim, int32_t out_dtype,
                                    void* out, const char* who) {
  if (!c || rows < 0 || count < 0 || dim <= 0 || (rows > 0 && (!nbr_ids || !out))) { set_error("%s: bad argument", who); return EU_ERR_INVALID; }
  if (int rc = dtype_check(out_dtype, who, "output")) return rc;
  EU_CUDA(cudaSetDevice(c->g->device));
  HostIO io{c};
  const int64_t o_ids = io.in(nbr_ids, 8 * rows * count), o_out = io.out(out, out_elem_bytes(out_dtype) * rows * dim);
  int rc;
  if ((rc = io.begin()) || (rc = io.upload())) return rc;
  if ((rc = out_dtype == EU_FEAT_F32
                ? eu_sage_mean_aggregate(c, io.dev<const int64_t>(o_ids), rows, count, dim, io.dev<float>(o_out))
                : eu_sage_mean_aggregate_out_dtype(c, io.dev<const int64_t>(o_ids), rows, count, dim, out_dtype, io.dev<void>(o_out)))) return rc;
  if ((rc = io.download())) return rc;
  return io.finish();
}

int eu_get_dense_feature_host(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int32_t dim, float* out) {
  return dense_feature_host(c, nodes, M, fid, dim, EU_FEAT_F32, out, "eu_get_dense_feature_host");
}
int eu_get_dense_feature_host_out_dtype(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int32_t dim, int32_t out_dtype, void* out) {
  return dense_feature_host(c, nodes, M, fid, dim, out_dtype, out, "eu_get_dense_feature_host_out_dtype");
}
int eu_sage_mean_aggregate_host(eu_ctx* c, const int64_t* nbr_ids, int64_t rows, int32_t count, int32_t dim, float* out) {
  return sage_mean_aggregate_host(c, nbr_ids, rows, count, dim, EU_FEAT_F32, out, "eu_sage_mean_aggregate_host");
}
int eu_sage_mean_aggregate_host_out_dtype(eu_ctx* c, const int64_t* nbr_ids, int64_t rows, int32_t count, int32_t dim, int32_t out_dtype,
                                          void* out) {
  return sage_mean_aggregate_host(c, nbr_ids, rows, count, dim, out_dtype, out, "eu_sage_mean_aggregate_host_out_dtype");
}

int eu_gather_host(eu_ctx* c, const float* params, int64_t N, int64_t D, const int32_t* idx, int64_t E, float* out) {
  if (!c || N < 0 || D <= 0 || E < 0) { set_error("eu_gather_host: bad argument"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  HostIO io{c};
  const int64_t o_p = io.in(params, 4 * N * D), o_i = io.in(idx, 4 * E), o_o = io.out(out, 4 * E * D);
  int rc;
  if ((rc = io.begin()) || (rc = io.upload())) return rc;
  if ((rc = eu_gather(c, io.dev<const float>(o_p), N, D, io.dev<const int32_t>(o_i), E, io.dev<float>(o_o)))) return rc;
  if ((rc = io.download())) return rc;
  return io.finish();
}

static int scatter_host(int op, eu_ctx* c, const float* u, int64_t D, const int32_t* idx, int64_t E, int64_t size, float* out) {
  if (!c || D <= 0 || E < 0 || size < 0) { set_error("scatter_host: bad argument"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  HostIO io{c};
  const int64_t o_u = io.in(u, 4 * E * D), o_i = io.in(idx, 4 * E), o_o = io.out(out, 4 * size * D);
  int rc;
  if ((rc = io.begin()) || (rc = io.upload())) return rc;
  const float* du = io.dev<const float>(o_u); const int32_t* di = io.dev<const int32_t>(o_i); float* dout = io.dev<float>(o_o);
  if ((rc = op == 0 ? eu_scatter_add(c, du, D, di, E, size, dout) : eu_scatter_max(c, du, D, di, E, size, dout))) return rc;
  if ((rc = io.download())) return rc;
  return io.finish();
}
int eu_scatter_add_host(eu_ctx* c, const float* u, int64_t D, const int32_t* idx, int64_t E, int64_t size, float* out) { return scatter_host(0, c, u, D, idx, E, size, out); }
int eu_scatter_max_host(eu_ctx* c, const float* u, int64_t D, const int32_t* idx, int64_t E, int64_t size, float* out) { return scatter_host(1, c, u, D, idx, E, size, out); }

int eu_get_node_type_host(eu_ctx* c, const int64_t* nodes, int64_t B, int32_t* out) {
  if (!c || B < 0 || (B > 0 && (!nodes || !out))) { set_error("eu_get_node_type_host: bad argument"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  HostIO io{c};
  const int64_t o_nodes = io.in(nodes, 8 * B), o_out = io.out(out, 4 * B);
  int rc;
  if ((rc = io.begin()) || (rc = io.upload())) return rc;
  if ((rc = eu_get_node_type(c, io.dev<const int64_t>(o_nodes), B, io.dev<int32_t>(o_out)))) return rc;
  if ((rc = io.download())) return rc;
  return io.finish();
}

int eu_get_node_weight_host(eu_ctx* c, const int64_t* nodes, int64_t B, float* out) {
  if (!c || B < 0 || (B > 0 && (!nodes || !out))) { set_error("eu_get_node_weight_host: bad argument"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  HostIO io{c};
  const int64_t o_nodes = io.in(nodes, 8 * B), o_out = io.out(out, 4 * B);
  int rc;
  if ((rc = io.begin()) || (rc = io.upload())) return rc;
  if ((rc = get_node_weight(c, io.dev<const int64_t>(o_nodes), B, io.dev<float>(o_out)))) return rc;
  if ((rc = io.download())) return rc;
  return io.finish();
}

// Call with cap = 0 to learn *total (out_ptr is filled), then with cap >= *total for the entries.
int eu_get_full_neighbor_host(eu_ctx* c, const int64_t* nodes, int64_t B, const int32_t* etypes, int32_t K,
                              int64_t cap, int64_t* out_ptr, int64_t* out_ids, float* out_w, int32_t* out_t,
                              int64_t* total) {
  return ragged_host(c, nodes, B, cap, out_ptr, total, {{out_ids, 8}, {out_w, 4}, {out_t, 4}}, "eu_get_full_neighbor_host",
                     [&](const int64_t* d_nodes, int64_t n, int64_t* d_ptr, char* const* v) {
                       return eu_get_full_neighbor(c, d_nodes, B, etypes, K, n, d_ptr, (int64_t*)v[0], (float*)v[1], (int32_t*)v[2]);
                     });
}

int eu_get_sparse_feature_host(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int64_t default_value, int64_t cap, int64_t* out_ptr,
                               int64_t* out_values, int64_t* total) {
  return ragged_host(c, nodes, M, cap, out_ptr, total, {{out_values, 8}}, "eu_get_sparse_feature_host",
                     [&](const int64_t* d_nodes, int64_t n, int64_t* d_ptr, char* const* v) {
                       return eu_get_sparse_feature(c, d_nodes, M, fid, default_value, n, d_ptr, (int64_t*)v[0]);
                     });
}

int eu_get_binary_feature_host(eu_ctx* c, const int64_t* nodes, int64_t M, int32_t fid, int64_t cap, int64_t* out_ptr, uint8_t* out_bytes,
                               int64_t* total) {
  return ragged_host(c, nodes, M, cap, out_ptr, total, {{out_bytes, 1}}, "eu_get_binary_feature_host",
                     [&](const int64_t* d_nodes, int64_t n, int64_t* d_ptr, char* const* v) {
                       return eu_get_binary_feature(c, d_nodes, M, fid, n, d_ptr, (uint8_t*)v[0]);
                     });
}

}  // extern "C"
