// HBM-bound row kernels of the hot path: fused CFG + DDIM step (K7, eta = 0 and eta > 0), fused CFG + DPM-Solver++(2M) step
// and LayerNorm.  GroupNorm(+SiLU) (K6) is groupnorm.cu.
#include "host_util.cuh"
#include "ptx.cuh"

namespace av2v {
namespace {

// ---------------------------------------------------------------------------------------------------- K7
// Every arithmetic result is rounded to fp16 separately, in the order the reference's chain of PyTorch ops
// produces them (pipeline_i2vgen_xl.py:1162, consisti2v/ddim_inverse_scheduler.py:346-369): fp32 multiply by the
// fp32 scalar, round; fp32 add of two fp16 values, round.  __fmul_rn/__fadd_rn forbid FMA contraction.
__device__ __forceinline__ float r16(float x) { return __half2float(__float2half_rn(x)); }

__device__ __forceinline__ float ddim_one(float x, float vn, float ve, bool cfg, float g, float ca, float cb,
                                          float cc, float cd) {
  float v = vn;
  if (cfg) {
    const float d0 = r16(__fsub_rn(ve, vn));
    const float d1 = r16(__fmul_rn(g, d0));
    v = r16(__fadd_rn(vn, d1));
  }
  const float x0 = r16(__fsub_rn(r16(__fmul_rn(ca, x)), r16(__fmul_rn(cb, v))));
  const float ep = r16(__fadd_rn(r16(__fmul_rn(ca, v)), r16(__fmul_rn(cb, x))));
  const float dir = r16(__fmul_rn(cd, ep));
  return r16(__fadd_rn(r16(__fmul_rn(cc, x0)), dir));
}

// kNoise: stochastic DDIM (eta > 0).  diffusers' step adds std_dev_t * variance_noise to the eta = 0 update as two more
// PyTorch ops (fp32 0-dim scalar times fp16 tensor, then fp16 + fp16), so the kernel rounds twice more:
// out = r16(ddim_one(...) + r16(cs * z)), with cd = sqrt(1 - a_prev - cs^2) passed in by the host.
template <bool kNoise>
__global__ void __launch_bounds__(256)
ddim_step_kernel(const __half* __restrict__ x, const __half* __restrict__ vn, const __half* __restrict__ ve,
                 const __half* __restrict__ z, __half* __restrict__ out, long long n, float g, float ca, float cb,
                 float cc, float cd, float cs, const float* __restrict__ coef_dev) {
  if (coef_dev != nullptr) {
    ca = coef_dev[0];
    cb = coef_dev[1];
    cc = coef_dev[2];
    cd = coef_dev[3];
    g = coef_dev[4];
    if (kNoise) cs = coef_dev[5];
  }
  const bool cfg = ve != nullptr;
  const long long nvec = n >> 3;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += stride) {
    const uint4 xv = reinterpret_cast<const uint4*>(x)[i];
    const uint4 nv = reinterpret_cast<const uint4*>(vn)[i];
    uint4 ev = nv;
    if (cfg) ev = reinterpret_cast<const uint4*>(ve)[i];
    uint4 zv = nv;
    if (kNoise) zv = reinterpret_cast<const uint4*>(z)[i];
    const __half* xh = reinterpret_cast<const __half*>(&xv);
    const __half* nh = reinterpret_cast<const __half*>(&nv);
    const __half* eh = reinterpret_cast<const __half*>(&ev);
    const __half* zh = reinterpret_cast<const __half*>(&zv);
    uint4 ov;
    __half* oh = reinterpret_cast<__half*>(&ov);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float y = ddim_one(__half2float(xh[e]), __half2float(nh[e]), __half2float(eh[e]), cfg, g, ca, cb, cc, cd);
      if (kNoise) y = r16(__fadd_rn(y, r16(__fmul_rn(cs, __half2float(zh[e])))));
      oh[e] = __float2half_rn(y);
    }
    reinterpret_cast<uint4*>(out)[i] = ov;
  }
  // tail (n not a multiple of 8)
  const long long tail0 = nvec << 3;
  for (long long i = tail0 + static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    float y = ddim_one(__half2float(x[i]), __half2float(vn[i]), cfg ? __half2float(ve[i]) : 0.f, cfg, g, ca, cb, cc, cd);
    if (kNoise) y = r16(__fadd_rn(y, r16(__fmul_rn(cs, __half2float(z[i])))));
    out[i] = __float2half_rn(y);
  }
}

unsigned ddim_blocks(long long n) {
  const long long nvec = (n + 7) >> 3;
  long long blocks = (nvec + 255) / 256;
  const long long cap = static_cast<long long>(sm_count_cached()) * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return static_cast<unsigned>(blocks);
}

int ddim_launch(const av2v_ddim_args* a, cudaStream_t stream) {
  AV2V_REQUIRE(a != nullptr, AV2V_EINVAL, "ddim: null args");
  AV2V_REQUIRE(a->n >= 0, AV2V_EINVAL, "ddim: negative element count");
  if (a->n == 0) return AV2V_OK;  // empty latents: nothing to do (pointers may be null)
  AV2V_REQUIRE(a->x && a->v_neg && a->out, AV2V_EINVAL, "ddim: null x / v_neg / out");
  AV2V_REQUIRE(aligned16(a->x) && aligned16(a->v_neg) && aligned16(a->out) && (!a->v_edit || aligned16(a->v_edit)),
               AV2V_EALIGN, "ddim: pointers must be 16-byte aligned");
  ddim_step_kernel<false><<<ddim_blocks(a->n), 256, 0, stream>>>(
      static_cast<const __half*>(a->x), static_cast<const __half*>(a->v_neg), static_cast<const __half*>(a->v_edit),
      nullptr, static_cast<__half*>(a->out), a->n, a->guidance, a->ca, a->cb, a->cc, a->cd, 0.f, a->coef_dev);
  AV2V_CHECK_CUDA(cudaGetLastError());
  return AV2V_OK;
}

int ddim_eta_launch(const av2v_ddim_eta_args* a, cudaStream_t stream) {
  AV2V_REQUIRE(a != nullptr, AV2V_EINVAL, "ddim_eta: null args");
  AV2V_REQUIRE(a->n >= 0, AV2V_EINVAL, "ddim_eta: negative element count");
  if (a->n == 0) return AV2V_OK;
  AV2V_REQUIRE(a->x && a->v_neg && a->noise && a->out, AV2V_EINVAL, "ddim_eta: null x / v_neg / noise / out");
  AV2V_REQUIRE(aligned16(a->x) && aligned16(a->v_neg) && aligned16(a->noise) && aligned16(a->out) &&
                   (!a->v_edit || aligned16(a->v_edit)),
               AV2V_EALIGN, "ddim_eta: pointers must be 16-byte aligned");
  ddim_step_kernel<true><<<ddim_blocks(a->n), 256, 0, stream>>>(
      static_cast<const __half*>(a->x), static_cast<const __half*>(a->v_neg), static_cast<const __half*>(a->v_edit),
      static_cast<const __half*>(a->noise), static_cast<__half*>(a->out), a->n, a->guidance, a->ca, a->cb, a->cc, a->cd,
      a->cs, a->coef_dev);
  AV2V_CHECK_CUDA(cudaGetLastError());
  return AV2V_OK;
}

// ---------------------------------------------------------------------------------------------------- DPM-Solver++(2M)
// One step t -> s of the multistep solver (anyv2v_b200/schedulers.py DPMSolverMultistepScheduler), v-prediction:
//   v   = v_edit ? r16(v_neg + r16(g * r16(v_edit - v_neg))) : v_neg      (the CFG combine, rounded as ddim_one rounds it)
//   x0  = r16(alpha * x - sigma * v)                                     (stored to x0_prev for the next step)
//   D   = c != 0 ? x0 + c * (x0 - x0_prev) : x0                          (c = 0: first-order step; x0_prev is not read)
//   out = r16(a * x + b * D)
// Pinned rounding points: x0 and out are rounded to fp16 once each; everything between is fp32, one IEEE rounding per
// operation in the order written (__fmul_rn / __fadd_rn / __fsub_rn, no FMA contraction), so a CPU restatement in fp32
// tensor ops gives the same bits.  The kernel reads x0_prev before it overwrites the same element with x0.
__device__ __forceinline__ void dpm_one(float x, float vn, float ve, float p, bool cfg, bool second, float g, float al,
                                        float si, float a, float b, float c, float& x0_out, float& y_out) {
  float v = vn;
  if (cfg) {
    const float d0 = r16(__fsub_rn(ve, vn));
    const float d1 = r16(__fmul_rn(g, d0));
    v = r16(__fadd_rn(vn, d1));
  }
  const float x0 = r16(__fsub_rn(__fmul_rn(al, x), __fmul_rn(si, v)));
  const float d = second ? __fadd_rn(x0, __fmul_rn(c, __fsub_rn(x0, p))) : x0;
  x0_out = x0;
  y_out = __fadd_rn(__fmul_rn(a, x), __fmul_rn(b, d));
}

__global__ void __launch_bounds__(256)
dpm_step_kernel(const __half* __restrict__ x, const __half* __restrict__ vn, const __half* __restrict__ ve,
                __half* __restrict__ x0p, __half* __restrict__ out, long long n, float g, float al, float si, float a,
                float b, float c, const float* __restrict__ coef_dev) {
  if (coef_dev != nullptr) {
    al = coef_dev[0];
    si = coef_dev[1];
    a = coef_dev[2];
    b = coef_dev[3];
    c = coef_dev[4];
    g = coef_dev[5];
  }
  const bool cfg = ve != nullptr;
  const bool second = c != 0.f;
  const long long nvec = n >> 3;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += stride) {
    const uint4 xv = reinterpret_cast<const uint4*>(x)[i];
    const uint4 nv = reinterpret_cast<const uint4*>(vn)[i];
    uint4 ev = nv;
    if (cfg) ev = reinterpret_cast<const uint4*>(ve)[i];
    uint4 pv = nv;
    if (second) pv = reinterpret_cast<const uint4*>(x0p)[i];
    const __half* xh = reinterpret_cast<const __half*>(&xv);
    const __half* nh = reinterpret_cast<const __half*>(&nv);
    const __half* eh = reinterpret_cast<const __half*>(&ev);
    const __half* ph = reinterpret_cast<const __half*>(&pv);
    uint4 ov, qv;
    __half* oh = reinterpret_cast<__half*>(&ov);
    __half* qh = reinterpret_cast<__half*>(&qv);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float x0, y;
      dpm_one(__half2float(xh[e]), __half2float(nh[e]), __half2float(eh[e]), __half2float(ph[e]), cfg, second, g, al, si, a,
              b, c, x0, y);
      qh[e] = __float2half_rn(x0);
      oh[e] = __float2half_rn(y);
    }
    reinterpret_cast<uint4*>(x0p)[i] = qv;
    reinterpret_cast<uint4*>(out)[i] = ov;
  }
  // tail (n not a multiple of 8)
  const long long tail0 = nvec << 3;
  for (long long i = tail0 + static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    float x0, y;
    dpm_one(__half2float(x[i]), __half2float(vn[i]), cfg ? __half2float(ve[i]) : 0.f, second ? __half2float(x0p[i]) : 0.f,
            cfg, second, g, al, si, a, b, c, x0, y);
    x0p[i] = __float2half_rn(x0);
    out[i] = __float2half_rn(y);
  }
}

int dpmpp2m_launch(const av2v_dpmpp2m_args* a, cudaStream_t stream) {
  AV2V_REQUIRE(a != nullptr, AV2V_EINVAL, "dpmpp2m: null args");
  AV2V_REQUIRE(a->n >= 0, AV2V_EINVAL, "dpmpp2m: negative element count");
  if (a->n == 0) return AV2V_OK;
  AV2V_REQUIRE(a->x && a->v_neg && a->x0_prev && a->out, AV2V_EINVAL, "dpmpp2m: null x / v_neg / x0_prev / out");
  AV2V_REQUIRE(a->x0_prev != a->x && a->x0_prev != a->out && a->x0_prev != a->v_neg && a->x0_prev != a->v_edit,
               AV2V_EINVAL, "dpmpp2m: x0_prev must not alias x / v_neg / v_edit / out");
  AV2V_REQUIRE(aligned16(a->x) && aligned16(a->v_neg) && aligned16(a->x0_prev) && aligned16(a->out) &&
                   (!a->v_edit || aligned16(a->v_edit)),
               AV2V_EALIGN, "dpmpp2m: pointers must be 16-byte aligned");
  dpm_step_kernel<<<ddim_blocks(a->n), 256, 0, stream>>>(
      static_cast<const __half*>(a->x), static_cast<const __half*>(a->v_neg), static_cast<const __half*>(a->v_edit),
      static_cast<__half*>(a->x0_prev), static_cast<__half*>(a->out), a->n, a->guidance, a->alpha, a->sigma, a->a, a->b,
      a->c, a->coef_dev);
  AV2V_CHECK_CUDA(cudaGetLastError());
  return AV2V_OK;
}

// ---------------------------------------------------------------------------------------------------- LayerNorm
// Fallback for widths that are not a multiple of 320 (none in I2VGen-XL; tiny test configs): one warp per row; the row
// (C <= 2048) lives in registers: sum -> mean, centred sum of squares -> rstd, normalise.
template <int kVecPerLane>
__global__ void __launch_bounds__(256)
layernorm_kernel(const __half* __restrict__ x, __half* __restrict__ y, const __half* __restrict__ gamma,
                 const __half* __restrict__ beta, long long rows, int C, float eps) {
  const int lane = threadIdx.x & 31;
  const long long row = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int vpr = C >> 3;
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * C);
  uint4 v[kVecPerLane];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < kVecPerLane; ++i) {
    const int vi = lane + i * 32;
    if (vi < vpr) {
      v[i] = __ldg(xr + vi);
      const __half2* h2 = reinterpret_cast<const __half2*>(&v[i]);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(h2[e]);
        s += f.x + f.y;
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / static_cast<float>(C);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < kVecPerLane; ++i) {
    const int vi = lane + i * 32;
    if (vi < vpr) {
      const __half2* h2 = reinterpret_cast<const __half2*>(&v[i]);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(h2[e]);
        q += (f.x - mean) * (f.x - mean) + (f.y - mean) * (f.y - mean);
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / static_cast<float>(C) + eps);
  uint4* yr = reinterpret_cast<uint4*>(y + row * C);
#pragma unroll
  for (int i = 0; i < kVecPerLane; ++i) {
    const int vi = lane + i * 32;
    if (vi < vpr) {
      const uint4 gv = __ldg(reinterpret_cast<const uint4*>(gamma) + vi);
      const uint4 bv = __ldg(reinterpret_cast<const uint4*>(beta) + vi);
      const __half2* h2 = reinterpret_cast<const __half2*>(&v[i]);
      const __half2* g2 = reinterpret_cast<const __half2*>(&gv);
      const __half2* b2 = reinterpret_cast<const __half2*>(&bv);
      uint4 ov;
      uint32_t* ow = reinterpret_cast<uint32_t*>(&ov);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(h2[e]);
        const float2 g = __half22float2(g2[e]);
        const float2 b = __half22float2(b2[e]);
        ow[e] = pack_half2((f.x - mean) * rstd * g.x + b.x, (f.y - mean) * rstd * g.y + b.y);
      }
      yr[vi] = ov;
    }
  }
}


// ---------------------------------------------------------------------------------------------------- LayerNorm, C = 40 * LPR vectors
// The product path.  Every I2VGen-XL width is a multiple of 320 = 40 vectors, so LPR = C / 40 lanes (8, 16 or 32) share a row with exactly FIVE 16-byte vectors each: 32 / LPR rows per warp
// per iteration, all lanes busy; warps are persistent (grid-stride over rows), gamma / beta are staged in shared memory once
// per CTA, and the next iteration's vectors are loaded before the current ones are reduced.
template <int LPR>
__global__ void __launch_bounds__(256, 3)  // <= 85 registers: three CTAs (24 warps, 10 vector loads each in flight) per SM
layernorm5_kernel(const __half* __restrict__ x, __half* __restrict__ y, const __half* __restrict__ gamma,
                  const __half* __restrict__ beta, long long rows, int C, float eps) {
  constexpr int RPW = 32 / LPR;  // rows per warp iteration
  const int lane = threadIdx.x & 31;
  const int sub = lane / LPR;     // which of the warp's rows
  const int l = lane % LPR;       // lane inside the row group
  const long long warp_g = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long stride = static_cast<long long>(gridDim.x) * (blockDim.x >> 5) * RPW;
  __shared__ uint4 gb[2][5 * LPR];  // gamma / beta staged once per CTA (kept out of the register file)
  for (int i = threadIdx.x; i < 5 * LPR; i += blockDim.x) {
    gb[0][i] = __ldg(reinterpret_cast<const uint4*>(gamma) + i);
    gb[1][i] = __ldg(reinterpret_cast<const uint4*>(beta) + i);
  }
  __syncthreads();
  const float inv_c = 1.0f / static_cast<float>(C);
  long long row = warp_g * RPW + sub;
  uint4 v[5], vn[5];
  // rows are walked BACK TO FRONT (logical row r -> physical row rows-1-r): the producing GEMM wrote x front to back, so the
  // tail is what L2 still holds when x is about L2-sized, and the head of y — written last here — is what the next GEMM,
  // which reads front to back, finds resident
  auto load = [&](long long r, uint4 (&dst)[5]) {
    if (r < rows) {
      const uint4* xr = reinterpret_cast<const uint4*>(x + (rows - 1 - r) * C);
#pragma unroll
      for (int i = 0; i < 5; ++i) dst[i] = __ldg(xr + l + i * LPR);
    } else {
#pragma unroll
      for (int i = 0; i < 5; ++i) dst[i] = make_uint4(0, 0, 0, 0);
    }
  };
  load(row, v);
  // the loop bound is warp-uniform (row - sub): every lane takes part in the shuffles of every iteration
  for (; row - sub < rows; row += stride) {
    load(row + stride, vn);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      const __half2* h2 = reinterpret_cast<const __half2*>(&v[i]);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(h2[e]);
        s += f.x + f.y;
      }
    }
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s * inv_c;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      const __half2* h2 = reinterpret_cast<const __half2*>(&v[i]);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(h2[e]);
        q += (f.x - mean) * (f.x - mean) + (f.y - mean) * (f.y - mean);
      }
    }
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = rsqrtf(q * inv_c + eps);
    if (row < rows) {
      uint4* yr = reinterpret_cast<uint4*>(y + (rows - 1 - row) * C);
#pragma unroll
      for (int i = 0; i < 5; ++i) {
        const __half2* h2 = reinterpret_cast<const __half2*>(&v[i]);
        const uint4 gvi = gb[0][l + i * LPR], bvi = gb[1][l + i * LPR];
        const __half2* g2 = reinterpret_cast<const __half2*>(&gvi);
        const __half2* b2 = reinterpret_cast<const __half2*>(&bvi);
        uint4 ov;
        uint32_t* ow = reinterpret_cast<uint32_t*>(&ov);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 f = __half22float2(h2[e]);
          const float2 g = __half22float2(g2[e]);
          const float2 b = __half22float2(b2[e]);
          ow[e] = pack_half2((f.x - mean) * rstd * g.x + b.x, (f.y - mean) * rstd * g.y + b.y);
        }
        yr[l + i * LPR] = ov;
      }
    }
#pragma unroll
    for (int i = 0; i < 5; ++i) v[i] = vn[i];
  }
}

template <int LPR>
int layernorm5_launch(const av2v_layernorm_args* a, cudaStream_t stream) {
  constexpr int RPW = 32 / LPR;
  const int warps = 8;
  long long blocks = (a->rows + warps * RPW - 1) / (warps * RPW);
  const long long cap = static_cast<long long>(sm_count_cached()) * 3;
  if (blocks > cap) blocks = cap;
  layernorm5_kernel<LPR><<<static_cast<unsigned>(blocks), warps * 32, 0, stream>>>(
      static_cast<const __half*>(a->x), static_cast<__half*>(a->y), static_cast<const __half*>(a->gamma),
      static_cast<const __half*>(a->beta), a->rows, a->C, a->eps);
  AV2V_CHECK_CUDA(cudaGetLastError());
  return AV2V_OK;
}
}  // namespace
}  // namespace av2v

using namespace av2v;

extern "C" int av2v_layernorm_f16(const av2v_layernorm_args* a, av2v_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  AV2V_REQUIRE(a != nullptr, AV2V_EINVAL, "layernorm: null args");
  AV2V_REQUIRE(a->rows >= 0 && a->C > 0, AV2V_EINVAL, "layernorm: bad shape");
  if (a->rows == 0) return AV2V_OK;
  AV2V_REQUIRE(a->x && a->y && a->gamma && a->beta, AV2V_EINVAL, "layernorm: null pointer");
  AV2V_REQUIRE(a->C % 8 == 0 && a->C <= 2048, AV2V_ENOSUP, "layernorm: C must be a multiple of 8 and <= 2048 (got %d)", a->C);
  AV2V_REQUIRE(aligned16(a->x) && aligned16(a->y) && aligned16(a->gamma) && aligned16(a->beta), AV2V_EALIGN,
               "layernorm: pointers must be 16-byte aligned");
  if (a->C % 40 == 0) {
    const int lpr = a->C / 40;
    if (lpr == 8) return layernorm5_launch<8>(a, stream);
    if (lpr == 16) return layernorm5_launch<16>(a, stream);
    if (lpr == 32) return layernorm5_launch<32>(a, stream);
  }
  const int warps = 8;
  const long long blocks = (a->rows + warps - 1) / warps;
  AV2V_REQUIRE(blocks <= 0x7fffffffll, AV2V_EINVAL, "layernorm: too many rows");
  const int vpl = (a->C / 8 + 31) / 32;
  const __half* x = static_cast<const __half*>(a->x);
  __half* y = static_cast<__half*>(a->y);
  const __half* g = static_cast<const __half*>(a->gamma);
  const __half* b = static_cast<const __half*>(a->beta);
  const unsigned grid = static_cast<unsigned>(blocks);
#define AV2V_LN_LAUNCH(V) layernorm_kernel<V><<<grid, warps * 32, 0, stream>>>(x, y, g, b, a->rows, a->C, a->eps)
  if (vpl <= 1) AV2V_LN_LAUNCH(1);
  else if (vpl <= 2) AV2V_LN_LAUNCH(2);
  else if (vpl <= 3) AV2V_LN_LAUNCH(3);
  else if (vpl <= 5) AV2V_LN_LAUNCH(5);
  else AV2V_LN_LAUNCH(8);
#undef AV2V_LN_LAUNCH
  AV2V_CHECK_CUDA(cudaGetLastError());
  return AV2V_OK;
}

extern "C" int av2v_ddim_step_cfg_f16(const av2v_ddim_args* a, av2v_stream_t stream) {
  return ddim_launch(a, static_cast<cudaStream_t>(stream));
}
extern "C" int av2v_ddim_inverse_step_f16(const av2v_ddim_args* a, av2v_stream_t stream) {
  return ddim_launch(a, static_cast<cudaStream_t>(stream));
}
extern "C" int av2v_ddim_step_eta_f16(const av2v_ddim_eta_args* a, av2v_stream_t stream) {
  return ddim_eta_launch(a, static_cast<cudaStream_t>(stream));
}
extern "C" int av2v_dpmpp2m_step_f16(const av2v_dpmpp2m_args* a, av2v_stream_t stream) {
  return dpmpp2m_launch(a, static_cast<cudaStream_t>(stream));
}
