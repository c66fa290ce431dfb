// VAE tile stitch: the seam blending of diffusers' tiled VAE encode / decode, from the raw tile outputs in one pass.
//
// The reference blends in place, tile by tile in row-major order: tile (i, j) first takes blend_v from the already blended
// tile (i-1, j), then blend_h from the already blended tile (i, j-1), and keeps its first row_limit x row_limit pixels.
// Blended values therefore feed later blends.  The chain is short, though.  Along an axis, the seam of tile k reads its
// neighbour k-1 at rows t_{k-1} - e + y >= t_{k-1} - blend, and every tile but the last is at least 2 * blend long (checked
// on the host), so the rows read lie past the neighbour's own blended band (y < e <= blend): a neighbour is only ever read
// where it carries no blend along that axis.  Output element (y, x) of tile (i, j) thus depends on at most four raw tiles:
//   U  = (i-1, j) at (yu, x),   with yu = t_{i-1} - ev + y;  if x < eh:  U = blend_h(UL, U)
//   L  = (i, j-1) at (y, xl),   with xl = t_{j-1} - eh + x;  if y < ev:  L = blend_v(UL, L)
//   UL = (i-1, j-1) at (yu, xl), raw (outside both of its bands)
//   out = raw (i, j);  if y < ev: out = blend_v(U, out);  if x < eh: out = blend_h(L, out)
// Each blend is evaluated with torch's fp16 rounding sequence for `a * (1 - y/e) + b * (y/e)` (fp16 tensor x Python
// float): the weights are computed in double and rounded to fp32, each product and the sum round to fp16, with fp32
// arithmetic in between and no FMA contraction.  So the result is bit-identical to the sequential loop.
//
// One thread per output element, channels innermost (the VAE's channels-last layout), gathers through the tile table.
// The work is a copy of the output with a few extra reads at the seams; nothing here is compute-bound.
#include <cuda_fp16.h>

#include "host_util.cuh"

namespace av2v {
namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ int extent(int k, int L, int tile, int step) { return min(tile, L - k * step); }

__device__ __forceinline__ float raw(const av2v_tile_desc& d, int c, int y, int x) {
  const __half* p = static_cast<const __half*>(d.ptr) + c * d.sc + y * d.sy + x * d.sx;
  return __half2float(__ldg(p));
}

// b[pos] <- a * (1 - pos/e) + b[pos] * (pos/e), as torch evaluates it on fp16 tensors
__device__ __forceinline__ float blend(float a, float b, int pos, int e) {
  const double r = static_cast<double>(pos) / static_cast<double>(e);
  const float pa = __half2float(__float2half_rn(__fmul_rn(a, static_cast<float>(1.0 - r))));
  const float pb = __half2float(__float2half_rn(__fmul_rn(b, static_cast<float>(r))));
  return __half2float(__float2half_rn(__fadd_rn(pa, pb)));
}

__global__ void __launch_bounds__(kThreads)
tile_stitch_kernel(const av2v_tile_desc* __restrict__ tiles, __half* __restrict__ out, av2v_tile_stitch_args a,
                   long long total) {
  for (long long idx = blockIdx.x * static_cast<long long>(kThreads) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * kThreads) {
    long long t = idx;
    const int c = static_cast<int>(t % a.C);
    t /= a.C;
    const int X = static_cast<int>(t % a.W);
    t /= a.W;
    const int Y = static_cast<int>(t % a.H);
    const int n = static_cast<int>(t / a.H);
    const int i = Y / a.row_limit, j = X / a.row_limit;
    const int y = Y - i * a.row_limit, x = X - j * a.row_limit;
    const av2v_tile_desc* row = tiles + (static_cast<long long>(n) * a.tile_rows + i) * a.tile_cols;

    int ev = 0, eh = 0, yu = 0, xl = 0;
    if (i > 0) {
      const int tu = extent(i - 1, a.H, a.tile, a.step);
      ev = min(min(tu, extent(i, a.H, a.tile, a.step)), a.blend);
      yu = tu - ev + y;
    }
    if (j > 0) {
      const int tl = extent(j - 1, a.W, a.tile, a.step);
      eh = min(min(tl, extent(j, a.W, a.tile, a.step)), a.blend);
      xl = tl - eh + x;
    }
    const bool bv = y < ev, bh = x < eh;

    float v = raw(row[j], c, y, x);
    if (bv) {
      const av2v_tile_desc* up = row - a.tile_cols;
      float u = raw(up[j], c, yu, x);
      if (bh) u = blend(raw(up[j - 1], c, yu, xl), u, x, eh);
      v = blend(u, v, y, ev);
    }
    if (bh) {
      float l = raw(row[j - 1], c, y, xl);
      if (bv) l = blend(raw(row[j - 1 - a.tile_cols], c, yu, xl), l, y, ev);
      v = blend(l, v, x, eh);
    }
    out[n * a.on + c * a.oc + Y * a.oy + X * a.ox] = __float2half_rn(v);
  }
}

// the kept parts of the tiles cover [0, L) exactly, and every tile but the last is long enough for the closed form
int check_axis(const char* axis, int L, int n_tiles, const av2v_tile_stitch_args* a) {
  const int want = (L + a->step - 1) / a->step;
  AV2V_REQUIRE(n_tiles == want, AV2V_EINVAL, "tile_stitch: %d tiles along %s, expected ceil(%d / %d) = %d", n_tiles, axis, L,
               a->step, want);
  long long kept = 0;
  for (int k = 0; k < n_tiles; ++k) {
    const int t = L - k * a->step < a->tile ? L - k * a->step : a->tile;
    if (k + 1 < n_tiles) {
      AV2V_REQUIRE(t >= a->row_limit && t >= 2 * a->blend, AV2V_EINVAL,
                   "tile_stitch: tile %d along %s is %d long, shorter than row_limit %d or 2 x blend %d", k, axis, t,
                   a->row_limit, a->blend);
      kept += a->row_limit;
    } else {
      kept += t < a->row_limit ? t : a->row_limit;
    }
  }
  AV2V_REQUIRE(kept == L, AV2V_EINVAL,
               "tile_stitch: the kept parts along %s cover %lld pixels, not %d (tile %d, step %d, row_limit %d)", axis, kept,
               L, a->tile, a->step, a->row_limit);
  return AV2V_OK;
}

}  // namespace
}  // namespace av2v

using namespace av2v;

extern "C" int av2v_tile_stitch_f16(const av2v_tile_stitch_args* a, av2v_stream_t stream) {
  AV2V_REQUIRE(a != nullptr, AV2V_EINVAL, "tile_stitch: null args");
  AV2V_REQUIRE(a->N >= 0 && a->C >= 1 && a->H >= 1 && a->W >= 1, AV2V_EINVAL, "tile_stitch: bad shape N=%d C=%d H=%d W=%d",
               a->N, a->C, a->H, a->W);
  AV2V_REQUIRE(a->tile >= 1 && a->step >= 1 && a->row_limit >= 1 && a->blend >= 0, AV2V_EINVAL,
               "tile_stitch: bad grid tile=%d step=%d blend=%d row_limit=%d", a->tile, a->step, a->blend, a->row_limit);
  if (int rc = check_axis("H", a->H, a->tile_rows, a)) return rc;
  if (int rc = check_axis("W", a->W, a->tile_cols, a)) return rc;
  if (a->N == 0) return AV2V_OK;
  AV2V_REQUIRE(a->tiles && a->out, AV2V_EINVAL, "tile_stitch: null tiles / out");
  const long long total = static_cast<long long>(a->N) * a->C * a->H * a->W;
  const long long blocks = (total + kThreads - 1) / kThreads;
  const int grid = static_cast<int>(blocks < 16LL * sm_count_cached() ? blocks : 16LL * sm_count_cached());
  tile_stitch_kernel<<<grid, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(a->tiles, static_cast<__half*>(a->out), *a,
                                                                               total);
  AV2V_CHECK_CUDA(cudaGetLastError());
  return AV2V_OK;
}
