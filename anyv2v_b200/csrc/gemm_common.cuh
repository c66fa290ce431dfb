// Shared by the two GEMM kernels: the launch parameters av2v_gemm_f16 validates and fills, and the GEGLU activation.
//   gemm_wgmma.cu      : the conv modes (3 x 3, stride 2, up2 phase, temporal (3, 1, 1)), two CTAs per SM
//   gemm_linear_ws.cu  : the LINEAR mode, persistent and warp-specialized
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

// LINEAR-mode launch (gemm_linear_ws.cu); p is validated and filled by av2v_gemm_f16
int gemm_linear_ws(const GemmP& p, cudaStream_t stream);

}  // namespace av2v
