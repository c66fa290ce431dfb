// FreeU (arXiv:2309.11497) at the skip connections of the first two up blocks: the backbone half of the hidden
// states is scaled by b, and the skip features go through diffusers' `fourier_filter(x, threshold=1, scale=s)`.
//
// The filter scales the centred 2 x 2 window of the shifted spectrum, i.e. the frequencies {0, -1} of each axis
// (only {0} when the axis has size 1).  For a real plane x[h, w] with th = 2 pi h / H and ph = 2 pi w / W that is,
// without any FFT,
//   y = x + (s - 1) / (H W) * ( Sx + [H>1] (Sx.cos th * cos th_h + Sx.sin th * sin th_h)
//                                  + [W>1] (Sx.cos ph * cos ph_w + Sx.sin ph * sin ph_w)
//                                  + [H>1 and W>1] (Sx.cos(th+ph) * cos(th_h+ph_w) + Sx.sin(th+ph) * sin(th_h+ph_w)) )
// where S. are seven sums over the plane.  One CTA owns one frame and 64 channels (8 lanes x 16-byte vectors, 32
// pixels in flight): pass 1 accumulates the 7 x 8 sums per lane in fp32 over the pixels, the CTA reduces them in a
// fixed order (deterministic), and pass 2 re-reads the plane (L1 / L2 resident) and writes y with one rounding to fp16.
// Further CTAs of the same grid scale hidden[..., :Ch/2] in place: fp16(fp32(x) * b), torch's fp16 `x * b`.
#include "host_util.cuh"
#include "ptx.cuh"

namespace av2v {
namespace {

constexpr int kLanes = 8;                  // 16-byte channel vectors per pixel row of a CTA (64 channels)
constexpr int kThreads = 256;
constexpr int kSlots = kThreads / kLanes;  // pixels in flight per CTA
constexpr int kWarps = kThreads / 32;
constexpr int kSums = 7;                   // per channel: Sx, Sx.cos th, Sx.sin th, Sx.cos ph, Sx.sin ph, Sx.cos(th+ph), Sx.sin(th+ph)
constexpr int kAcc = 8 * kSums;

// the six twiddles of pixel p: cos / sin of th_h, ph_w and th_h + ph_w (sincospif keeps the angle exact up to the
// rounding of 2h/H; the sum angle comes from the addition theorem)
__device__ __forceinline__ void twiddles(int p, int H, int W, float (&t)[6]) {
  const int h = p / W, w = p - h * W;
  sincospif(2.f * static_cast<float>(h) / static_cast<float>(H), &t[1], &t[0]);
  sincospif(2.f * static_cast<float>(w) / static_cast<float>(W), &t[3], &t[2]);
  t[4] = t[0] * t[2] - t[1] * t[3];
  t[5] = t[1] * t[2] + t[0] * t[3];
}

__global__ void __launch_bounds__(kThreads)
freeu_kernel(__half* __restrict__ hidden, const __half* __restrict__ skip, __half* __restrict__ out, int H, int W,
             int Ch, int Cs, int skip_blocks, float b, float s) {
  const int HW = H * W;
  const int lane = threadIdx.x % kLanes;
  const int slot = threadIdx.x / kLanes;
  const long long frame = blockIdx.y;

  if (static_cast<int>(blockIdx.x) >= skip_blocks) {  // backbone half of hidden, in place
    const int half_c = Ch / 2;
    const int v = (blockIdx.x - skip_blocks) * kLanes + lane;
    if (v * 8 >= half_c) return;
    for (int p = slot; p < HW; p += kSlots) {
      uint4* ptr = reinterpret_cast<uint4*>(hidden + (frame * HW + p) * Ch) + v;
      uint4 xv = *ptr;
      __half* xh = reinterpret_cast<__half*>(&xv);
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (v * 8 + e < half_c) xh[e] = __float2half_rn(__fmul_rn(__half2float(xh[e]), b));
      *ptr = xv;
    }
    return;
  }

  __shared__ float red[kWarps][kLanes][kAcc];
  __shared__ float fin[kLanes][kAcc];
  const int v = blockIdx.x * kLanes + lane;
  const bool active = v * 8 < Cs;
  const uint4* src = reinterpret_cast<const uint4*>(skip + frame * HW * Cs) + v;
  const int vpp = Cs / 8;  // vectors per pixel

  float acc[kAcc];
#pragma unroll
  for (int i = 0; i < kAcc; ++i) acc[i] = 0.f;
  for (int p = slot; p < HW; p += kSlots) {
    if (!active) continue;
    const uint4 xv = __ldg(src + static_cast<long long>(p) * vpp);
    const __half* xh = reinterpret_cast<const __half*>(&xv);
    float t[6];
    twiddles(p, H, W, t);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float f = __half2float(xh[e]);
      acc[e * kSums] += f;
#pragma unroll
      for (int j = 0; j < 6; ++j) acc[e * kSums + 1 + j] = fmaf(f, t[j], acc[e * kSums + 1 + j]);
    }
  }
  // the 4 pixel slots of a warp share a lane index: fold them (lane bits 3 and 4), then the warps in a fixed order
#pragma unroll
  for (int i = 0; i < kAcc; ++i) {
    acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], 8);
    acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], 16);
  }
  const int warp = threadIdx.x / 32;
  if ((threadIdx.x & 31) < kLanes) {
#pragma unroll
    for (int i = 0; i < kAcc; ++i) red[warp][lane][i] = acc[i];
  }
  __syncthreads();
  const float k = (s - 1.f) / static_cast<float>(HW);
  for (int i = threadIdx.x; i < kLanes * kAcc; i += kThreads) {
    const int l = i / kAcc, j = (i % kAcc) % kSums;
    float sum = 0.f;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) sum += red[w][l][i % kAcc];
    // modes of a size-1 axis are the same frequency as mode 0: drop them
    const bool keep = j == 0 || (j <= 2 ? H > 1 : j <= 4 ? W > 1 : (H > 1 && W > 1));
    fin[l][i % kAcc] = keep ? k * sum : 0.f;
  }
  __syncthreads();
  if (!active) return;
  float c[kAcc];
#pragma unroll
  for (int i = 0; i < kAcc; ++i) c[i] = fin[lane][i];
  uint4* dst = reinterpret_cast<uint4*>(out + frame * HW * Cs) + v;
  for (int p = slot; p < HW; p += kSlots) {
    const uint4 xv = __ldg(src + static_cast<long long>(p) * vpp);
    const __half* xh = reinterpret_cast<const __half*>(&xv);
    float t[6];
    twiddles(p, H, W, t);
    uint4 ov;
    __half* oh = reinterpret_cast<__half*>(&ov);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float corr = c[e * kSums];
#pragma unroll
      for (int j = 0; j < 6; ++j) corr = fmaf(c[e * kSums + 1 + j], t[j], corr);
      oh[e] = __float2half_rn(__half2float(xh[e]) + corr);
    }
    dst[static_cast<long long>(p) * vpp] = ov;
  }
}

}  // namespace
}  // namespace av2v

using namespace av2v;

extern "C" int av2v_freeu_f16(const av2v_freeu_args* a, av2v_stream_t stream) {
  AV2V_REQUIRE(a != nullptr, AV2V_EINVAL, "freeu: null args");
  AV2V_REQUIRE(a->NF >= 0 && a->H >= 1 && a->W >= 1, AV2V_EINVAL, "freeu: bad shape NF=%d H=%d W=%d", a->NF, a->H, a->W);
  AV2V_REQUIRE(a->Ch > 0 && a->Cs > 0 && a->Ch % 8 == 0 && a->Cs % 8 == 0, AV2V_EINVAL,
               "freeu: Ch and Cs must be positive multiples of 8 (got %d, %d)", a->Ch, a->Cs);
  AV2V_REQUIRE(static_cast<long long>(a->H) * a->W <= 0x7fffffffll, AV2V_EINVAL, "freeu: plane too large");
  AV2V_REQUIRE(a->NF <= 65535, AV2V_EINVAL, "freeu: at most 65535 frames per call (got %d)", a->NF);
  if (a->NF == 0) return AV2V_OK;
  AV2V_REQUIRE(a->hidden && a->skip && a->out, AV2V_EINVAL, "freeu: null hidden / skip / out");
  AV2V_REQUIRE(aligned16(a->hidden) && aligned16(a->skip) && aligned16(a->out), AV2V_EALIGN,
               "freeu: pointers must be 16-byte aligned");
  const int skip_blocks = (a->Cs / 8 + kLanes - 1) / kLanes;
  const int hidden_blocks = ((a->Ch / 2 + 7) / 8 + kLanes - 1) / kLanes;
  freeu_kernel<<<dim3(skip_blocks + hidden_blocks, a->NF), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<__half*>(a->hidden), static_cast<const __half*>(a->skip), static_cast<__half*>(a->out), a->H, a->W, a->Ch,
      a->Cs, skip_blocks, a->b, a->s);
  AV2V_CHECK_CUDA(cudaGetLastError());
  return AV2V_OK;
}
