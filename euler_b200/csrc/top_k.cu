// LGCEncoder's input block: a node's dense feature row followed, column by column, by the k largest values of that column
// over the node's sampled neighbours -- one pass from the ids to f32[B, k + 1, dim], with no [B, count, dim] intermediate.
//
// Reference semantics (file:line in the upstream alibaba/euler tree):
//   LGCEncoder.call   tf_euler/python/utils/encoders.py:895-922  get_dense_feature of the nodes and of their sample_neighbor
//                     rows, tf.nn.top_k(k) over the transposed [B, D, nb_num] neighbour block, transposed back, the node row
//                     concatenated first
//   tf.nn.top_k       (TF's TopKV2) "If two elements are equal, the lower-index element appears first"
// Every value is read under k_feature's rule (mp_ops.cu): the slot's stored columns, zeros past them, zeros for an absent
// id.  NaN ranks above every number, as torch.sort orders it.  The selection only compares and copies, so the output is
// bit-exact against a stable descending sort of the fetched rows.
//
// One warp per batch row.  The lanes resolve 32 neighbour ids at a time (one lookup_row each) and pass the rows round by
// shuffle; lane l walks columns d0 + 32 c + l (c < C), so each neighbour row is read in coalesced 128-byte lines, and keeps
// each column's KMAX best values sorted in registers.  The rows are resolved again for every further 32 C columns (a
// lookup per 32 neighbours, against 32 C columns of each).
#include <algorithm>
#include <math.h>

#include "internal.h"

namespace eu {

// a ranks strictly above b: NaN above every number; equal values (+0.0 and -0.0, two NaNs) do not
__device__ __forceinline__ bool ranks_above(float a, float b) { return a > b || (isnan(a) && !isnan(b)); }

// t: descending, equal values in arrival order.  v arrives after every entry, so it goes below each one it does not rank
// above; the last entry drops out.
template <int KMAX>
__device__ __forceinline__ void top_k_insert(float (&t)[KMAX], float v) {
#pragma unroll
  for (int i = KMAX - 1; i > 0; --i)
    if (ranks_above(v, t[i])) t[i] = ranks_above(v, t[i - 1]) ? t[i - 1] : v;
  if (ranks_above(v, t[0])) t[0] = v;
}

// out[b, 0, :] = the node's row, out[b, 1 + j, d] = the j-th of column d over the count neighbours (j < k <= KMAX).  The
// slots start at -inf: a slot no value ranks above keeps -inf, which is the value it would have selected (k <= count).  The
// selection is f32; O, the output's element type, only decides how each selected value is stored (a bf16 one rounded once).
template <typename T, typename O, int KMAX, int C, int P>
__global__ void __launch_bounds__(256, 4) k_neighbor_top_k(DevGraph g, const unsigned long long* __restrict__ nodes, int64_t B,
                                                           const unsigned long long* __restrict__ nbrs, int32_t count, int32_t soff,
                                                           int32_t width, int32_t dim, int32_t k, O* __restrict__ out) {
  const int lane = (int)(threadIdx.x & 31);
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int32_t w = min(width, dim);   // columns read from the graph; the rest are zeros
  for (int64_t b = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; b < B; b += nwarps) {
    const unsigned long long* nb = nbrs + b * count;
    const int64_t self = w > 0 ? lookup_row(g, nodes[b]) : -1;
    const T* fs = self >= 0 ? feat_row<T, P>(g, self) + soff : nullptr;
    O* o = out + b * (int64_t)(k + 1) * dim;
    for (int32_t d0 = 0; d0 < dim; d0 += 32 * C) {
      float t[C][KMAX];
#pragma unroll
      for (int c = 0; c < C; ++c)
#pragma unroll
        for (int i = 0; i < KMAX; ++i) t[c][i] = -INFINITY;
      for (int32_t j0 = 0; j0 < count; j0 += 32) {
        const int32_t n = min(32, count - j0);
        const int64_t mine = (w > 0 && lane < n) ? lookup_row(g, nb[j0 + lane]) : -1;
        for (int32_t j = 0; j < n; ++j) {
          const int64_t row = __shfl_sync(0xffffffffu, mine, j);
          const T* f = feat_row_if<T, P>(g, row >= 0, row, soff);
          float v[C];
#pragma unroll
          for (int c = 0; c < C; ++c) {
            const int32_t d = d0 + 32 * c + lane;
            v[c] = (row >= 0 && d < w) ? feat_ld(f + d) : 0.f;
          }
#pragma unroll
          for (int c = 0; c < C; ++c) top_k_insert<KMAX>(t[c], v[c]);
        }
      }
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const int32_t d = d0 + 32 * c + lane;
        if (d >= dim) continue;
        o[d] = feat_st<O>((fs && d < w) ? feat_ld(fs + d) : 0.f);
#pragma unroll
        for (int i = 0; i < KMAX; ++i)
          if (i < k) o[(int64_t)(1 + i) * dim + d] = feat_st<O>(t[c][i]);
      }
    }
  }
}

template <int KMAX, int C>
static int launch_top_k(eu_ctx* c, const int64_t* nodes, int64_t B, const int64_t* neighbors, int32_t count, int32_t soff,
                        int32_t width, int32_t dim, int32_t k, int32_t out_dtype, void* out) {
  const unsigned blocks = (unsigned)std::min<int64_t>(ceil_div(B, 8), (int64_t)kSMs * 32);
  EuProfScope ps(c, "k_neighbor_top_k", B);
  // a bf16 table widens exactly and order-preservingly (+-0 and NaN included): the selection is the f32 one's on the widened rows
  const auto* nd = (const unsigned long long*)nodes;
  const auto* nb = (const unsigned long long*)neighbors;
  const DevGraph& g = c->g->d;
  with_feat(g, [&](auto t, auto p) {
    with_dtype(out_dtype, [&](auto o) {
      using O = typename decltype(o)::type;
      k_neighbor_top_k<typename decltype(t)::type, O, KMAX, C, decltype(p)::value><<<blocks, 256, 0, c->stream>>>(g, nd, B, nb, count, soff,
                                                                                                                width, dim, k, (O*)out);
    });
  });
  EU_LAUNCHED();
  return EU_OK;
}

static int neighbor_top_k(eu_ctx* c, const int64_t* nodes, int64_t B, const int64_t* neighbors, int32_t count, int32_t fid, int32_t dim,
                          int32_t k, int32_t out_dtype, void* out, const char* who) {
  if (!c || B < 0 || dim < 0 || (B > 0 && (!nodes || !neighbors || (dim > 0 && !out)))) {
    set_error("%s: bad argument", who);
    return EU_ERR_INVALID;
  }
  if (k < 1 || k > count) {
    set_error("%s: k = %d must lie in [1, count = %d]", who, k, count);
    return EU_ERR_INVALID;
  }
  if (k > EU_NEIGHBOR_TOP_K_MAX) {
    set_error("%s: k = %d is above the bound %d", who, k, EU_NEIGHBOR_TOP_K_MAX);
    return EU_ERR_UNSUPPORTED;
  }
  if (int rc = dtype_check(out_dtype, who, "output")) return rc;
  EU_CUDA(cudaSetDevice(c->g->device));
  if (B == 0 || dim == 0) return EU_OK;
  int32_t soff, width;
  dense_slot(c->g->d, fid, &soff, &width);
  if (k <= 4) return launch_top_k<4, 4>(c, nodes, B, neighbors, count, soff, width, dim, k, out_dtype, out);
  if (k <= 8) return launch_top_k<8, 2>(c, nodes, B, neighbors, count, soff, width, dim, k, out_dtype, out);
  return launch_top_k<EU_NEIGHBOR_TOP_K_MAX, 1>(c, nodes, B, neighbors, count, soff, width, dim, k, out_dtype, out);
}

}  // namespace eu

using namespace eu;

extern "C" {

int eu_neighbor_top_k_feature(eu_ctx* c, const int64_t* nodes, int64_t B, const int64_t* neighbors, int32_t count, int32_t fid,
                              int32_t dim, int32_t k, float* out) {
  return neighbor_top_k(c, nodes, B, neighbors, count, fid, dim, k, EU_FEAT_F32, out, "eu_neighbor_top_k_feature");
}
int eu_neighbor_top_k_feature_out_dtype(eu_ctx* c, const int64_t* nodes, int64_t B, const int64_t* neighbors, int32_t count, int32_t fid,
                                        int32_t dim, int32_t k, int32_t out_dtype, void* out) {
  return neighbor_top_k(c, nodes, B, neighbors, count, fid, dim, k, out_dtype, out, "eu_neighbor_top_k_feature_out_dtype");
}

}  // extern "C"
