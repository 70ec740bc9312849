// Contexts (scratch, engines, profiling), the default graph and the reference's InitQueryProxy entry.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <mutex>
#include <string>

#include "internal.h"

namespace eu {

// engine e is seeded with seeds[e] (or seed0 + e when seeds == nullptr)
__global__ void k_seed(EuRngState* rs, int n, unsigned long long seed0, const unsigned long long* seeds) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const unsigned long long seed = seeds ? seeds[e] : seed0 + (unsigned long long)e;
  EuRngState* r = rs + e;
  // std::minstd_rand0::seed(s): x = s mod m, 1 if that is 0 (SURVEY.md Appendix A-13)
  unsigned long long x = seed % 2147483647ull;
  r->x = x == 0 ? 1u : (uint32_t)x;
  r->x_prev = r->x;
  r->draws = 0;
  r->calls = 0;
  r->blocks_done = 0;
  r->key = seed * 0x9E3779B97F4A7C15ull;
}

template <typename T>
static int regrow(T** p, int64_t count) {
  if (*p) cudaFree(*p);
  *p = nullptr;
  void* q = nullptr;
  size_t bytes = (size_t)(count > 0 ? count : 1) * sizeof(T);
  cudaError_t e = cudaMalloc(&q, bytes);
  if (e != cudaSuccess) { set_error("cudaMalloc(%zu) -> %s", bytes, cudaGetErrorString(e)); return EU_ERR_CUDA; }
  *p = (T*)q;
  return EU_OK;
}

// growing scratch frees and re-allocates under a stream synchronise: impossible while the stream is being captured into
// a CUDA graph -- fail loudly and say what to do instead of invalidating the capture
int refuse_growth_in_capture(eu_ctx* c, const char* what) {
  cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(c->stream, &st) == cudaSuccess && st != cudaStreamCaptureStatusNone) {
    set_error("%s must grow while the ctx stream is being captured: run the op once (or call eu_ctx_reserve) before the capture", what);
    return EU_ERR_STATE;
  }
  cudaGetLastError();
  return EU_OK;
}

int ctx_reserve(eu_ctx* c, int64_t rows, int64_t table_slots) {
  int rc;
  if ((table_slots > c->tab_set_slots || rows > c->cap_rows) && (rc = refuse_growth_in_capture(c, "the sampling scratch"))) return rc;
  if (table_slots > c->tab_set_slots) {
    EU_CUDA(cudaStreamSynchronize(c->stream));  // growing while the stream still uses the old buffers would be a race
    const int64_t slots = table_slots + 64;
    if ((rc = regrow(&c->d_dedup, 2 * slots))) return rc;  // two table sets: hop l uses set l & 1
    c->tab_set_slots = slots;
    // all-free tables: key 0, row = kEmptyRow (see hop() invariant)
    for (int64_t off = 0; off < 2 * slots; off += (int64_t)1 << 20) {
      int64_t n = std::min<int64_t>((int64_t)1 << 20, 2 * slots - off);
      EU_CUDA(cudaMemset2DAsync(&c->d_dedup[off].key, sizeof(HashSlot), 0x00, 8, (size_t)n, c->stream));
      EU_CUDA(cudaMemset2DAsync(&c->d_dedup[off].row, sizeof(HashSlot), 0xFF, 8, (size_t)n, c->stream));
    }
  }
  if (rows <= c->cap_rows) return EU_OK;
  EU_CUDA(cudaStreamSynchronize(c->stream));
  if ((rc = regrow(&c->d_first, rows))) return rc;
  if ((rc = regrow(&c->d_rowof, rows))) return rc;
  if ((rc = regrow(&c->d_elig, rows))) return rc;
  if ((rc = regrow(&c->d_state, rows))) return rc;
  if ((rc = regrow(&c->d_emask, rows / 32 + 2))) return rc;
  if ((rc = regrow(&c->d_woff, rows / 32 + 2))) return rc;
  if ((rc = regrow(&c->d_blkpre, rows / 256 + 66))) return rc;
  if ((rc = regrow(&c->d_blkmul, rows / 256 + 66))) return rc;
  if ((rc = regrow(&c->d_live, rows))) return rc;
  if ((rc = regrow(&c->d_dup, rows))) return rc;
  if (!c->d_nlive && (rc = regrow(&c->d_nlive, 4))) return rc;
  if ((rc = regrow(&c->d_front[0], rows))) return rc;
  if ((rc = regrow(&c->d_front[1], rows))) return rc;
  c->cap_rows = rows;
  return EU_OK;
}

int ctx_misc(eu_ctx* c, int64_t bytes) {
  if (bytes <= c->misc_bytes) return EU_OK;
  if (int rc0 = refuse_growth_in_capture(c, "the op scratch")) return rc0;
  EU_CUDA(cudaStreamSynchronize(c->stream));
  char* p = (char*)c->d_misc;
  int rc = regrow(&p, bytes);
  c->d_misc = p;
  if (rc) { c->misc_bytes = 0; return rc; }
  c->misc_bytes = bytes;
  return EU_OK;
}

int agg_reserve(eu_ctx* c, int64_t rows, int64_t table_slots) {
  if (rows <= c->agg_rows && table_slots <= c->agg_slots) return EU_OK;
  int rc;
  if ((rc = refuse_growth_in_capture(c, "the aggregation scratch"))) return rc;
  EU_CUDA(cudaStreamSynchronize(c->stream));
  if (table_slots > c->agg_slots) {
    c->agg_slots = 0;
    if ((rc = regrow(&c->d_agg_tab, table_slots))) return rc;
    EU_CUDA(cudaMemsetAsync(c->d_agg_tab, 0, sizeof(unsigned long long) * (size_t)table_slots, c->stream));   // all free
    c->agg_slots = table_slots;
  }
  if (rows > c->agg_rows) {
    c->agg_rows = 0;
    if ((rc = regrow(&c->d_agg_src, rows))) return rc;
    if ((rc = regrow(&c->d_agg_rep, rows))) return rc;
    if ((rc = regrow(&c->d_agg_slot, rows))) return rc;
    if (!c->d_agg_nrep && (rc = regrow(&c->d_agg_nrep, 1))) return rc;
    c->agg_rows = rows;
  }
  return EU_OK;
}

static std::mutex g_default_mu;
static eu_graph* g_default_graph = nullptr;
static eu_ctx* g_default_ctx = nullptr;

}  // namespace eu

using namespace eu;

extern "C" {

int eu_ctx_create(eu_graph* g, eu_rng_kind rng, uint64_t seed, void* stream, eu_ctx** out) {
  if (!g || !out || (rng != EU_RNG_MINSTD && rng != EU_RNG_PHILOX)) { set_error("eu_ctx_create: bad argument"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(g->device));
  eu_ctx* c = new eu_ctx();
  c->g = g; c->rng = rng; c->seed = seed; c->stream = (cudaStream_t)stream;
  cudaError_t e = cudaMalloc(&c->d_rng, sizeof(EuRngState));
  if (e != cudaSuccess) { set_error("cudaMalloc rng -> %s", cudaGetErrorString(e)); delete c; return EU_ERR_CUDA; }
  k_seed<<<1, 64, 0, c->stream>>>(c->d_rng, 1, seed, nullptr);
  g_launches++;
  *out = c;
  return EU_OK;
}

int eu_ctx_destroy(eu_ctx* c) {
  if (!c) return EU_OK;
  cudaSetDevice(c->g->device);
  cudaStreamSynchronize(c->stream);
  cudaFree(c->d_rng); cudaFree(c->d_dedup); cudaFree(c->d_first); cudaFree(c->d_rowof);
  cudaFree(c->d_elig); cudaFree(c->d_state); cudaFree(c->d_emask); cudaFree(c->d_woff); cudaFree(c->d_blkpre); cudaFree(c->d_blkmul); cudaFree(c->d_live); cudaFree(c->d_dup); cudaFree(c->d_nlive); cudaFree(c->d_front[0]); cudaFree(c->d_front[1]);
  cudaFree(c->d_misc); cudaFree(c->d_stage); cudaFree(c->d_walkv);
  cudaFree(c->d_agg_tab); cudaFree(c->d_agg_src); cudaFree(c->d_agg_rep); cudaFree(c->d_agg_slot); cudaFree(c->d_agg_nrep);
  for (int i = 0; i < 2; ++i) { if (c->aux[i]) cudaStreamDestroy(c->aux[i]); if (c->ev_join[i]) cudaEventDestroy(c->ev_join[i]); }
  if (c->ev_fork) cudaEventDestroy(c->ev_fork);
  if (c->h_pin) cudaFreeHost(c->h_pin);
  delete c;
  return EU_OK;
}

int eu_ctx_set_stream(eu_ctx* c, void* stream) {
  if (!c) { set_error("null ctx"); return EU_ERR_INVALID; }
  c->stream = (cudaStream_t)stream;
  return EU_OK;
}

int eu_ctx_seed(eu_ctx* c, uint64_t seed) {
  if (!c) { set_error("null ctx"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  c->seed = seed;
  k_seed<<<1, 64, 0, c->stream>>>(c->d_rng, c->n_eng, seed, nullptr);
  EU_LAUNCHED();
  return EU_OK;
}

// n engines, engine e seeded with seeds[e] (seeds == NULL: seed + e).  Batch b of a *_batched call uses engine b.
int eu_ctx_set_engines(eu_ctx* c, int32_t n, const uint64_t* seeds) {
  if (!c || n < 1 || n > 64) { set_error("eu_ctx_set_engines: 1..64 engines"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  EU_CUDA(cudaStreamSynchronize(c->stream));
  EuRngState* r = nullptr;
  EU_CUDA(cudaMalloc(&r, sizeof(EuRngState) * n));
  unsigned long long* d_seeds = nullptr;
  if (seeds) {
    EU_CUDA(cudaMalloc(&d_seeds, sizeof(unsigned long long) * n));
    EU_CUDA(cudaMemcpy(d_seeds, seeds, sizeof(unsigned long long) * n, cudaMemcpyHostToDevice));
    c->seed = seeds[0];
  }
  cudaFree(c->d_rng);
  c->d_rng = r;
  c->n_eng = n;
  k_seed<<<1, 64, 0, c->stream>>>(c->d_rng, n, c->seed, d_seeds);
  EU_LAUNCHED();
  EU_CUDA(cudaStreamSynchronize(c->stream));
  if (d_seeds) cudaFree(d_seeds);
  return EU_OK;
}

int eu_ctx_reserve(eu_ctx* c, int64_t max_rows) {
  if (!c || max_rows < 0) { set_error("eu_ctx_reserve: bad argument"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  const int nb = c->n_eng;
  int rc = ctx_reserve(c, max_rows + 256 * nb, 4 * max_rows + 65 * nb);
  if (rc) return rc;
  return ctx_misc(c, 256 + 4 * max_rows);
}

int eu_ctx_sync(eu_ctx* c) {
  if (!c) { set_error("null ctx"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  EU_CUDA(cudaStreamSynchronize(c->stream));
  return EU_OK;
}

int eu_ctx_draws(eu_ctx* c, uint64_t* draws) {
  if (!c || !draws) { set_error("eu_ctx_draws: bad argument"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  EuRngState h;
  EU_CUDA(cudaMemcpyAsync(&h, c->d_rng, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
  EU_CUDA(cudaStreamSynchronize(c->stream));
  *draws = h.draws;
  return EU_OK;
}

int eu_ctx_profile(eu_ctx* c, int enable) {
  if (!c) { set_error("null ctx"); return EU_ERR_INVALID; }
  c->prof = enable != 0;
  return EU_OK;
}

// Synchronises, then writes "name,rows,launches,total_ms\n" lines (aggregated) into buf and clears the log.
int eu_ctx_profile_read(eu_ctx* c, char* buf, int64_t cap) {
  if (!c || !buf || cap <= 0) { set_error("eu_ctx_profile_read: bad argument"); return EU_ERR_INVALID; }
  EU_CUDA(cudaSetDevice(c->g->device));
  EU_CUDA(cudaStreamSynchronize(c->stream));
  std::map<std::pair<std::string, int64_t>, std::pair<int64_t, double>> agg;
  for (auto& r : c->prof_recs) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, r.e0, r.e1);
    auto& a = agg[std::make_pair(std::string(r.name), r.rows)];
    a.first += 1; a.second += ms;
    cudaEventDestroy(r.e0); cudaEventDestroy(r.e1);
  }
  c->prof_recs.clear();
  std::string out;
  char line[256];
  for (auto& kv : agg) {
    snprintf(line, sizeof(line), "%s,%lld,%lld,%.6f\n", kv.first.first.c_str(), (long long)kv.first.second,
             (long long)kv.second.first, kv.second.second);
    out += line;
  }
  if ((int64_t)out.size() + 1 > cap) { set_error("profile buffer too small"); return EU_ERR_INVALID; }
  memcpy(buf, out.c_str(), out.size() + 1);
  return EU_OK;
}

// ------------------------------------------------------------------------------ InitQueryProxy
eu_graph* eu_default_graph(void) { std::lock_guard<std::mutex> l(g_default_mu); return g_default_graph; }
eu_ctx* eu_default_ctx(void) { std::lock_guard<std::mutex> l(g_default_mu); return g_default_ctx; }

int eu_set_default_graph(eu_graph* g, eu_rng_kind rng, uint64_t seed) {
  std::lock_guard<std::mutex> l(g_default_mu);
  if (g_default_ctx) { eu_ctx_destroy(g_default_ctx); g_default_ctx = nullptr; }
  g_default_graph = g;
  if (!g) return EU_OK;
  return eu_ctx_create(g, rng, seed, nullptr, &g_default_ctx);
}

// tf_euler/utils/init_query_proxy.cc:19-36: split on ';' then '=', false only when the list is
// empty or an item is not exactly k=v; the graph-load status is NOT propagated (:34).
bool InitQueryProxy(const char* conf) {
  if (!conf) return false;
  std::map<std::string, std::string> kv;
  std::string s(conf);
  size_t pos = 0;
  int items = 0;
  while (pos <= s.size()) {
    size_t end = s.find(';', pos);
    if (end == std::string::npos) end = s.size();
    std::string item = s.substr(pos, end - pos);
    pos = end + 1;
    if (item.empty()) continue;
    size_t eq = item.find('=');
    if (eq == std::string::npos || item.find('=', eq + 1) != std::string::npos) return false;
    kv[item.substr(0, eq)] = item.substr(eq + 1);
    ++items;
  }
  if (items == 0) return false;
  std::string mode = kv.count("mode") ? kv["mode"] : "local";
  if (mode != "local") {
    fprintf(stderr, "[euler_b200] ERROR InitQueryProxy: mode=%s is not on this path (only mode=local; sharding is eu_* over NCCL)\n", mode.c_str());
    return true;
  }
  int device = kv.count("device") ? atoi(kv["device"].c_str()) : 0;
  uint64_t seed = kv.count("seed") ? strtoull(kv["seed"].c_str(), nullptr, 10) : 1;
  eu_rng_kind rng = (kv.count("rng") && kv["rng"] == "philox") ? EU_RNG_PHILOX : EU_RNG_MINSTD;
  // feature_dtype: the dense node feature table's storage type (eu_graph_load_dtype); float32 when absent
  const std::string fdt = kv.count("feature_dtype") ? kv["feature_dtype"] : "float32";
  if (fdt != "float32" && fdt != "bfloat16") {
    fprintf(stderr, "[euler_b200] ERROR InitQueryProxy: feature_dtype=%s is not float32 or bfloat16\n", fdt.c_str());
    return true;
  }
  // feature_place=device|host and feature_cache_rows=C: where the table lives (eu_feat_storage); device and 0 when absent
  const std::string fpl = kv.count("feature_place") ? kv["feature_place"] : "device";
  const std::string fcr = kv.count("feature_cache_rows") ? kv["feature_cache_rows"] : "0";
  if ((fpl != "device" && fpl != "host") || fcr.empty() || fcr.find_first_not_of("0123456789") != std::string::npos) {
    fprintf(stderr, "[euler_b200] ERROR InitQueryProxy: feature_place=%s / feature_cache_rows=%s: the place is device or host, "
            "the rows an integer >= 0\n", fpl.c_str(), fcr.c_str());
    return true;
  }
  const eu_feat_storage st{fdt == "bfloat16" ? EU_FEAT_BF16 : EU_FEAT_F32, fpl == "host" ? EU_FEAT_HOST : EU_FEAT_DEVICE,
                           (int64_t)strtoll(fcr.c_str(), nullptr, 10)};
  eu_graph* g = nullptr;
  int rc = eu_graph_load_storage(kv["data_path"].c_str(), 0, 1, device, 1, &st, &g);
  if (rc != EU_OK) {
    fprintf(stderr, "[euler_b200] ERROR InitQueryProxy: graph load failed: %s\n", eu_last_error());
    return true;
  }
  rc = eu_set_default_graph(g, rng, seed);
  if (rc != EU_OK) fprintf(stderr, "[euler_b200] ERROR InitQueryProxy: %s\n", eu_last_error());
  return true;
}

}  // extern "C"
