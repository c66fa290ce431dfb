// Shared by the two GEMM kernels: the launch parameters av2v_gemm_f16 validates and fills, the GEGLU activation and the
// staged epilogue.
//   gemm_ws.cu         : persistent and warp-specialized, TMA-fed: the LINEAR mode, and the conv modes (3 x 3 stride 1, up2
//                        phase, temporal (3, 1, 1)) whose 128-row tiles are each one box of the input (conv_ws_box)
//   gemm_wgmma.cu      : the other conv geometries (stride 2, widths that do not divide 128, ...), cp.async-gathered, two
//                        CTAs per SM
#pragma once
#include "host_util.cuh"
#include "ptx.cuh"

namespace av2v {

struct GemmP {
  int mode;
  const __half* a;
  const __half* a2;
  const __half* w;
  int M, N, K;
  int lda, lda2, k_split;  // LINEAR (k_split = K for one source)
  int Hin, Win, chan;      // CONV3X3: input image, channels present (row stride of A)
  int Ho, Wo, stride;      // CONV3X3: output pixels of the GEMM rows
  int taps_w, up2, py, px; // CONV3X3: taps per kernel row (3, or 2 for an up2 phase), phase offsets
  int Cin;                 // CONV3X3 / TCONV3: K per tap
  int F, HW;               // TCONV3
  const __half* bias;
  const __half* rowbias;
  int rows_per_rowbias;
  const __half* residual;
  __half* out;
  int ldo;
  int n_slots;
  long long slot_stride;
  int geglu;
  int n_tiles, num_kb;
};

// Exact-erf GELU, branch-free: gelu(g) = g/2 * erfc(-g/sqrt 2).  With E = erfc(z), z = |g|/sqrt 2:
//   g < 0: gelu = g/2 * E;   g >= 0: gelu = g - g/2 * E   ->   gelu = max(g, 0) - |g/2| * E.
// E has the form of the erfcc routine of Numerical Recipes, t = 1 / (1 + z/2), E = t * exp(-z^2 + P(t)), with a degree-5 P
// fitted in tools/erfc_poly_fit.py: its error is RELATIVE (< 1.4e-5 on z in [0, 5.6], fp32 evaluation included), so the
// small negative-gate side keeps full fp16 precision.  (An absolute-error erf — A&S 7.1.25, 2.5e-5 — was 20 fp16 ulps off at
// gates in [-4, -3], where gelu is ~1e-3.)  MUFU rcp + ex2 and ~9 FMAs per element; libdevice erfcf costs more and diverges.
__device__ __forceinline__ float gelu_erf_fast(float g) {
  const float z = fabsf(g) * 0.70710678118654752f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.5f, z, 1.0f)));
  float p = fmaf(t, 0.22427836f, -0.69402432f);
  p = fmaf(p, t, 0.45475456f);
  p = fmaf(p, t, 0.26681793f);
  p = fmaf(p, t, 1.01429605f);
  p = fmaf(p, t, -1.26611602f);
  const float e = t * ex2_approx(fmaf(-z, z, p) * 1.4426950408889634f);
  return fmaf(-fabsf(0.5f * g), e, fmaxf(g, 0.0f));
}

// ---- staged epilogue.  A 128 x 128 output tile is packed in fp16 into a staging tile in shared memory (128 rows x 256
// bytes, 16-byte chunk c of row r at chunk c ^ (r & 7): the 8 rows x 4 lanes of a fragment store and the 8 chunks a quarter
// warp copies out both cover the 32 banks once) and leaves it in 16-byte stores along the output rows.  A 128 x 160 tile
// (gemm_ws_kernel's 160-column tiles) keeps that layout for its first 128 columns and puts its last 32 (chunks 16 .. 19) in
// a second part of 128 rows x 64 bytes behind the first, chunk 16 + c of row r at chunk c ^ ((r >> 1) & 3): 8 consecutive
// rows of a fragment store again cover the 32 banks once, and the tail's copy-out and residual fetch, 8 rows x 4 chunks
// per warp instruction, read and write 2 whole rows = 128 bytes per quarter warp.  A warp's unit of work is a band: the 16
// tile rows r0 .. r0 + 15 it holds in one m64nBN accumulator (float[BN / 2]); a warp with kBands accumulators owns the bands
// r0 + 64 b.  A warp fetches, writes and copies out only its own bands' rows, so the kernels order these steps with
// __syncwarp.  N, ldo and slot_stride are multiples of 8, so every chunk is whole: it is stored iff its row < M and its
// first column < N.  A value is rounded once: acc + bias + rowbias + residual in fp32, packed over the residual's place in
// the tile.
template <int kBN = 128>
__device__ __forceinline__ uint32_t stage_offset(int row, int chunk) {
  static_assert(kBN == 128 || kBN == 160, "staging tiles are 128 or 160 columns wide");
  if (kBN == 128 || chunk < 16) return static_cast<uint32_t>(row * 256 + ((chunk ^ (row & 7)) << 4));
  return static_cast<uint32_t>(128 * 256 + row * 64 + (((chunk - 16) ^ ((row >> 1) & 3)) << 4));
}

// The row mapping and the output tile differ by A mode, fixed at compile time so that neither instantiation carries the
// other's: kConv (gemm_wgmma.cu, gemm_ws_kernel<true>): the rows of an up2 phase are its pixels of the 2x output; otherwise
// (LINEAR, gemm_ws_kernel<false>) row m is out row m and a GEGLU tile is 128 x 64.

// element offset of output row m inside a slot of out / residual
template <bool kConv>
__device__ __forceinline__ long long out_row_offset(const GemmP& p, int m) {
  if (!kConv || !p.up2) return static_cast<long long>(m) * p.ldo;
  // low-resolution pixel (n, i, j) -> (n, 2 i + py, 2 j + px) of the [NF][2H][2W] output
  const int j = m % p.Wo, t = m / p.Wo, i = t % p.Ho, n = t / p.Ho;
  return ((static_cast<long long>(n) * 2 * p.Ho + 2 * i + p.py) * (2 * p.Wo) + 2 * j + p.px) * p.ldo;
}

// the band at tile rows r0 .. r0 + 15 of the residual tile of `slot` -> staging tile by cp.async: per instruction 2 rows x
// 16 chunks (a 160-wide tile's last 32 columns: 8 rows x 4 chunks), zero-filled past M / N
template <bool kConv, int kBN = 128>
__device__ __forceinline__ void fetch_residual_band(const GemmP& p, int slot, int m0, int n0, int r0, uint32_t tile) {
  const int lane = threadIdx.x & 31, ch = lane & 15;
  const int c = n0 + 8 * ch;
  const __half* src = p.residual + slot * p.slot_stride + c;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int r = r0 + 2 * i + (lane >> 4);
    const bool v = m0 + r < p.M && c < p.N;
    cp_async16(tile + stage_offset<kBN>(r, ch), v ? src + out_row_offset<kConv>(p, m0 + r) : p.residual, v);
  }
  if constexpr (kBN == 160) {
    const int ct = 16 + (lane & 3), c1 = n0 + 8 * ct;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = r0 + 8 * i + (lane >> 2);
      const bool v = m0 + r < p.M && c1 < p.N;
      cp_async16(tile + stage_offset<kBN>(r, ct),
                 v ? p.residual + slot * p.slot_stride + c1 + out_row_offset<kConv>(p, m0 + r) : p.residual, v);
    }
  }
}

// acc + bias + rowbias (+ the residual the tile holds) of the warp's bands -> fp16 pairs in fragment order in the staging
// tile.  Column pair j is the outer loop, so its bias is loaded once for every band (st.shared clobbers memory).
template <int kBands, int kAcc>
__device__ __forceinline__ void epilogue_bands(const GemmP& p, const float (&d)[kBands][kAcc], int m0, int n0, int r0,
                                               uint32_t tile) {
  constexpr int kBN = 2 * kAcc;  // m64nBN: BN / 2 accumulators per thread
  const int fr = r0 + ((threadIdx.x & 31) >> 2);  // the thread's rows fr + 64 b + 8 h (accumulator layout, acc_row)
  const int cq = 2 * (threadIdx.x & 3);
  const __half* rb[kBands][2];
#pragma unroll
  for (int b = 0; b < kBands; ++b)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = m0 + fr + 64 * b + 8 * h;
      rb[b][h] = p.rowbias && m < p.M ? p.rowbias + static_cast<long long>(m / p.rows_per_rowbias) * p.N : nullptr;
    }
#pragma unroll
  for (int j = 0; j < kBN / 8; ++j) {
    const int c = n0 + 8 * j + cq;
    if (c >= p.N) continue;
    float2 bias = make_float2(0.f, 0.f);
    if (p.bias) bias = __half22float2(*reinterpret_cast<const __half2*>(p.bias + c));
#pragma unroll
    for (int b = 0; b < kBands; ++b)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t at = tile + stage_offset<kBN>(fr + 64 * b + 8 * h, j) + 2 * cq;
        float o0 = d[b][4 * j + 2 * h], o1 = d[b][4 * j + 2 * h + 1];
        if (p.bias) {
          o0 += bias.x;
          o1 += bias.y;
        }
        if (rb[b][h]) {
          const float2 t = __half22float2(*reinterpret_cast<const __half2*>(rb[b][h] + c));
          o0 += t.x;
          o1 += t.y;
        }
        if (p.residual) {
          const uint32_t rr = ld_shared_u32(at);
          const float2 r = __half22float2(*reinterpret_cast<const __half2*>(&rr));
          o0 += r.x;
          o1 += r.y;
        }
        st_shared_u32(at, pack_half2(o0, o1));
      }
  }
}

// the band at tile rows r0 .. r0 + 15 of the staging tile -> slot `slot` of out: lane -> 16-byte chunk of a row, a warp
// instruction covers 2 rows x 256 bytes (GEGLU: 4 rows x 128 bytes; a 160-wide tile's last 32 columns: 8 rows x 64 bytes)
template <bool kConv, int kBN = 128>
__device__ __forceinline__ void copy_out_band(const GemmP& p, int slot, int m0, int n0, int r0, uint32_t tile) {
  const int lane = threadIdx.x & 31;
  const bool geglu = kBN == 128 && !kConv && p.geglu;  // GEGLU tiles are 128 wide
  const int lg = geglu ? 3 : 4;  // log2(chunks per output row of the tile)
  const int col0 = geglu ? n0 / 2 : n0, n_out = geglu ? p.N / 2 : p.N;
  __half* out = p.out + slot * p.slot_stride + col0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int idx = 32 * i + lane;
    const int r = r0 + (idx >> lg), ch = idx & ((1 << lg) - 1);
    if ((idx >> lg) < 16 && m0 + r < p.M && col0 + 8 * ch < n_out)
      st_global_v4(out + out_row_offset<kConv>(p, m0 + r) + 8 * ch, ld_shared_v4(tile + stage_offset<kBN>(r, ch)));
  }
  if constexpr (kBN == 160) {
    const int ct = 16 + (lane & 3);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = r0 + 8 * i + (lane >> 2);
      if (m0 + r < p.M && n0 + 8 * ct < p.N)
        st_global_v4(out + out_row_offset<kConv>(p, m0 + r) + 8 * ct, ld_shared_v4(tile + stage_offset<kBN>(r, ct)));
    }
  }
}

// Launches of gemm_ws.cu's persistent kernel on `tiles` output tiles; p is validated and filled by av2v_gemm_f16.
// LINEAR mode; a conv mode whose tiles are each one box of its input (conv_ws_box returns true and the box).  ws_tile_n is
// the column tile of both (128 or 160): av2v_gemm_f16 counts p.n_tiles in it.
int ws_tile_n(const GemmP& p);
int gemm_linear_ws(const GemmP& p, int tiles, cudaStream_t stream);
bool conv_ws_box(const GemmP& p, unsigned (&box)[3]);
int gemm_conv_ws(const GemmP& p, const unsigned (&box)[3], int tiles, cudaStream_t stream);

}  // namespace av2v
