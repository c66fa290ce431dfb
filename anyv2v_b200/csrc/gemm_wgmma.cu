// wgmma GEMM core of the I2VGen-XL UNet hot path (sm_90a): the convolutions gemm_ws.cu's persistent kernel does not
// take.  av2v_gemm_f16 validates every call the same way whichever kernel runs it, then sends the LINEAR mode, and every
// conv whose 128-row tiles are each one TMA box of its input (conv_ws_box: 3 x 3 stride 1 and up2 phases at widths that
// divide 128, temporal convs whose tiles hold whole frames of one clip), to gemm_ws.cu; the rest (stride 2, widths
// such as 27 or 88, temporal convs whose frame count the box does not divide) run here.
//
//   out[slot][m, n] = sum_k A[m, k] * W[n, k] + bias[n] + rowbias[m / rows_per_rowbias, n] + residual[slot][m, n]
//
// One CTA computes a 128 x 128 output tile with two warpgroups (rows 0-63 / 64-127), each issuing wgmma.m64n128k16 with
// both operands in shared memory.  All 256 threads gather the operand tiles with 16-byte cp.async straight from the
// channels-last activations — the A row of output pixel m for K block kb is the (tap, channel block) the block names, so the
// 3 x 3 conv (plain, stride 2, one phase of nearest-up x 2) and the temporal (3, 1, 1) conv are implicit GEMMs without an im2col buffer; out-of-image taps, ragged rows and the K tail are zero-filled by cp.async.
// kStages = 3 stage ring (32 KB per stage), prefetch distance 1, one wgmma group in flight behind the current one:
//   top of K block kb: cp.async of block kb landed (wait_group) -> fence.proxy.async -> __syncthreads (also: every warpgroup
//   retired wgmma kb-2)
//   -> issue the loads of block kb + 1 into the slot of kb - 2 -> wgmma kb -> wait_group 1 (kb - 1 retired).
// Two CTAs per SM (2 x 97 KB of shared memory, <= 128 registers per thread): one CTA's prologue loads, K-loop gathers and
// epilogue run while the other's wgmma keep the tensor cores busy.  A tile's K loop is short (5 blocks at K = 320), so
// this overlap between tiles is worth more than a deeper ring inside one: with 4 stages only one CTA fits.
// Epilogue: gemm_common.cuh's staged epilogue, each warp on one band (the 16 tile rows its accumulators hold), so it needs
// no block barrier.  The staging tile of slot 0 takes the ring slot that block num_kb - 3 left, free from the top of the
// last K block, and the residual tile of slot 0 is fetched there by cp.async as soon as the last wgmma are issued, so it
// lands under them.  (Issued from inside the K loop, ptxas serializes the wgmma.)  The residual tiles of further slots go
// to the other two ring slots once every warpgroup has retired its wgmma.  All of a warp's residual reads complete before
// its first store, so a residual that aliases out stays safe.
#include "gemm_common.cuh"

namespace av2v {
namespace {

constexpr int BM = 128, BN = 128, BK = 64;
constexpr int kStages = 3;
constexpr int kThreads = 256;
constexpr int kTileBytes = BM * BK * 2;  // 16 KB, A and B alike (BM == BN)
constexpr int kSmemBytes = kStages * 2 * kTileBytes + 1024;

// Per-thread view of the A rows it gathers (rows r0 + 32 i, i = 0..3, of the tile): what the K loop needs to address them.
struct ARows {
  long long base[4];  // element offset of the row's pixel (CONV: pixel of tap (0, 0); TCONV: the row)
  int y[4], x[4];     // CONV: input coordinates of tap (0, 0); TCONV: y = frame; -1 marks a row past M
};

__device__ __forceinline__ void a_rows_init(const GemmP& p, int m0, int r0, ARows& ar) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + r0 + 32 * i;
    ar.y[i] = -1 << 20;
    ar.x[i] = 0;
    ar.base[i] = 0;
    if (m >= p.M) continue;
    if (p.mode == AV2V_A_CONV3X3) {
      const int ox = m % p.Wo, t = m / p.Wo, oy = t % p.Ho, n = t / p.Ho;
      const int y0 = p.up2 ? oy - 1 + p.py : oy * p.stride - 1;
      const int x0 = p.up2 ? ox - 1 + p.px : ox * p.stride - 1;
      ar.y[i] = y0;
      ar.x[i] = x0;
      ar.base[i] = (static_cast<long long>(n) * p.Hin + y0) * p.Win + x0;
    } else {  // TCONV3
      ar.base[i] = m;
      ar.y[i] = (m % (p.F * p.HW)) / p.HW;
    }
  }
}

__device__ __forceinline__ void load_stage(const GemmP& p, const ARows& ar, int kb, int n0, uint32_t sA, uint32_t sB) {
  const int tid = threadIdx.x;
  const int ch = tid & 7, r0 = tid >> 3;
  const int k0 = kb * BK;
  // ---- A
  if (p.mode == AV2V_A_CONV3X3) {
    const int tap = k0 / p.Cin, c = k0 - tap * p.Cin + ch * 8;
    const int ky = tap / p.taps_w, kx = tap - ky * p.taps_w;
    const bool cval = c < p.chan;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int y = ar.y[i] + ky, x = ar.x[i] + kx;
      const bool v = cval && y >= 0 && y < p.Hin && x >= 0 && x < p.Win;
      const __half* src = p.a + (ar.base[i] + static_cast<long long>(ky) * p.Win + kx) * p.chan + c;
      cp_async16(sA + sw128_offset(r0 + 32 * i, ch), v ? src : p.a, v);
    }
  } else {  // TCONV3: tap kt reads frame f + kt - 1 of the same clip and pixel
    const int kt = k0 / p.Cin, c = k0 - kt * p.Cin + ch * 8;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int f = ar.y[i] + kt - 1;
      const bool v = ar.y[i] >= 0 && f >= 0 && f < p.F;
      const __half* src = p.a + (ar.base[i] + static_cast<long long>(kt - 1) * p.HW) * p.Cin + c;
      cp_async16(sA + sw128_offset(r0 + 32 * i, ch), v ? src : p.a, v);
    }
  }
  // ---- B (weights [N][K])
  const bool kval = k0 + ch * 8 < p.K;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int n = n0 + r0 + 32 * i;
    const bool v = kval && n < p.N;
    cp_async16(sB + sw128_offset(r0 + 32 * i, ch), v ? p.w + static_cast<long long>(n) * p.K + k0 + ch * 8 : p.w, v);
  }
}

__global__ void __launch_bounds__(kThreads, 2) gemm_wgmma_kernel(const __grid_constant__ GemmP p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t s0 = smem_u32(smem);
  auto sA = [&](int s) { return s0 + static_cast<uint32_t>(s) * 2 * kTileBytes; };
  auto sB = [&](int s) { return s0 + static_cast<uint32_t>(s) * 2 * kTileBytes + kTileBytes; };

  const int n_t = blockIdx.x % p.n_tiles;
  const int m_t = blockIdx.x / p.n_tiles;
  const int m0 = m_t * BM, n0 = n_t * BN;
  const int wg = threadIdx.x >> 7;

  ARows ar;
  a_rows_init(p, m0, threadIdx.x >> 3, ar);

  float d[1][64];  // the warp's band: tile rows 16 * warp .. + 15
#pragma unroll
  for (int i = 0; i < 64; ++i) d[0][i] = 0.f;

  const int nk = p.num_kb;
#pragma unroll
  for (int s = 0; s < kStages - 2; ++s) {
    if (s < nk) load_stage(p, ar, s, n0, sA(s), sB(s));
    cp_async_commit();
  }
  for (int kb = 0; kb < nk; ++kb) {
    cp_async_wait<kStages - 3>();
    fence_proxy_async_smem();  // this thread's landed cp.async writes -> visible to wgmma (async proxy), then publish
    __syncthreads();
    {
      const int pf = kb + kStages - 2;
      if (pf < nk) load_stage(p, ar, pf, n0, sA(pf % kStages), sB(pf % kStages));
      cp_async_commit();
    }
    const int s = kb % kStages;
    const uint32_t a_base = sA(s) + wg * 64 * 128;
    const uint32_t b_base = sB(s);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k)
      wgmma_m64n128_ss(d[0], sw128_desc(a_base + k * 32), sw128_desc(b_base + k * 32), 1);
    wgmma_commit();
    wgmma_wait<1>();
    reg_fence(d[0]);
  }
  // the ring slot block nk - 3 left stays free: the residual tile of slot 0 is fetched there under the last wgmma
  const int r0 = 16 * (threadIdx.x >> 5);
  if (p.residual) fetch_residual_band<true>(p, 0, m0, n0, r0, sA(nk % kStages));
  wgmma_wait<0>();
  reg_fence(d[0]);

  // ---- epilogue: the staging tile of slot s is ring slot (nk + s) % kStages
  const int n_res = p.residual ? p.n_slots : 1;  // distinct tiles: without a residual every slot stores the same one
  if (n_res > 1) {
    __syncthreads();  // the other ring slots held the last operands: every warpgroup has retired its wgmma
    for (int s = 1; s < n_res; ++s) fetch_residual_band<true>(p, s, m0, n0, r0, sA((nk + s) % kStages));
  }
  cp_async_commit();
  cp_async_wait<0>();
  __syncwarp();  // the residual chunks this warp's lanes fetched for each other have landed
  for (int s = 0; s < n_res; ++s) epilogue_bands<1>(p, d, m0, n0, r0, sA((nk + s) % kStages));
  __syncwarp();
  for (int s = 0; s < p.n_slots; ++s) copy_out_band<true>(p, s, m0, n0, r0, sA((nk + (p.residual ? s : 0)) % kStages));
}

}  // namespace
}  // namespace av2v

using namespace av2v;

extern "C" int av2v_gemm_f16(const av2v_gemm_args* a, av2v_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  AV2V_REQUIRE(a != nullptr, AV2V_EINVAL, "gemm: null args");
  AV2V_REQUIRE(a->a && a->w && a->out, AV2V_EINVAL, "gemm: null a/w/out pointer");
  AV2V_REQUIRE(a->M > 0 && a->N > 0 && a->K > 0, AV2V_EINVAL, "gemm: M,N,K must be positive (%d,%d,%d)", a->M, a->N,
               a->K);
  AV2V_REQUIRE(a->N % 8 == 0 && a->K % 8 == 0, AV2V_EINVAL, "gemm: N and K must be multiples of 8 (%d,%d)", a->N,
               a->K);
  AV2V_REQUIRE((a->geglu || a->ldo >= a->N) && a->ldo % 8 == 0, AV2V_EINVAL,
               "gemm: ldo must be >= N and a multiple of 8");
  AV2V_REQUIRE(a->n_slots >= 1, AV2V_EINVAL, "gemm: n_slots must be >= 1");
  AV2V_REQUIRE(!a->residual || a->n_slots <= kStages, AV2V_ENOSUP, "gemm: at most %d slots with a residual (one staging tile each)", kStages);
  AV2V_REQUIRE(a->n_slots == 1 || a->slot_stride % 8 == 0, AV2V_EALIGN, "gemm: slot_stride must be a multiple of 8");
  AV2V_REQUIRE(aligned16(a->a) && aligned16(a->w) && aligned16(a->out), AV2V_EALIGN,
               "gemm: a/w/out must be 16-byte aligned");
  AV2V_REQUIRE(!a->bias || aligned16(a->bias), AV2V_EALIGN, "gemm: bias must be 16-byte aligned");
  AV2V_REQUIRE(!a->rowbias || (aligned16(a->rowbias) && a->rows_per_rowbias > 0), AV2V_EALIGN,
               "gemm: rowbias must be 16-byte aligned with rows_per_rowbias > 0");
  AV2V_REQUIRE(!a->residual || aligned16(a->residual), AV2V_EALIGN, "gemm: residual must be 16-byte aligned");

  GemmP p{};
  p.mode = a->mode;
  p.a = static_cast<const __half*>(a->a);
  p.w = static_cast<const __half*>(a->w);
  p.M = a->M;
  p.N = a->N;
  p.K = a->K;
  p.bias = static_cast<const __half*>(a->bias);
  p.rowbias = static_cast<const __half*>(a->rowbias);
  p.rows_per_rowbias = a->rows_per_rowbias;
  p.residual = static_cast<const __half*>(a->residual);
  p.out = static_cast<__half*>(a->out);
  p.ldo = a->ldo;
  p.n_slots = a->n_slots;
  p.slot_stride = a->slot_stride;
  p.geglu = a->geglu ? 1 : 0;
  p.stride = 1;
  p.taps_w = 3;
  if (a->geglu) {
    AV2V_REQUIRE(a->mode == AV2V_A_LINEAR, AV2V_EINVAL, "gemm/geglu: LINEAR mode only");
    AV2V_REQUIRE(a->N % 64 == 0, AV2V_EINVAL, "gemm/geglu: N must be a multiple of 64 (got %d)", a->N);
    AV2V_REQUIRE(!a->residual && !a->rowbias && a->n_slots == 1, AV2V_EINVAL, "gemm/geglu: no residual / rowbias / slots");
    AV2V_REQUIRE(a->ldo >= a->N / 2, AV2V_EINVAL, "gemm/geglu: ldo must be >= N/2");
  }
  if (a->mode == AV2V_A_LINEAR) {
    AV2V_REQUIRE((a->a2 != nullptr || a->lda >= a->K) && a->lda % 8 == 0, AV2V_EINVAL, "gemm: lda must be >= K and a multiple of 8");
    p.lda = a->lda;
    p.k_split = a->K;
    if (a->a2 != nullptr) {  // two-source K loop: A = [a | a2]
      AV2V_REQUIRE(a->k_split > 0 && a->k_split < a->K && a->k_split % BK == 0, AV2V_EINVAL,
                   "gemm: k_split must be a multiple of 64 inside (0, K) (got %d, K = %d)", a->k_split, a->K);
      AV2V_REQUIRE(a->lda >= a->k_split && a->lda2 >= a->K - a->k_split && a->lda2 % 8 == 0 && aligned16(a->a2), AV2V_EINVAL,
                   "gemm: a / a2 row strides must cover their column ranges (multiples of 8), a2 16-byte aligned");
      p.a2 = static_cast<const __half*>(a->a2);
      p.lda2 = a->lda2;
      p.k_split = a->k_split;
    }
    AV2V_REQUIRE(a->n_slots == 1, AV2V_ENOSUP, "gemm/linear: one output slot only (got n_slots = %d)", a->n_slots);
  } else if (a->mode == AV2V_A_CONV3X3) {
    AV2V_REQUIRE(a->NF > 0 && a->H > 0 && a->W > 0 && a->Cin > 0, AV2V_EINVAL, "gemm/conv3x3: bad geometry");
    AV2V_REQUIRE(a->Cin % BK == 0, AV2V_ENOSUP, "gemm/conv3x3: Cin must be a multiple of 64 (got %d)", a->Cin);
    const int up = a->up2_phase;  // 0: plain conv; 1..4: phase (py, px) = ((up-1) >> 1, (up-1) & 1) of nearest-up x 2 + conv 3 x 3
    AV2V_REQUIRE(up >= 0 && up <= 4, AV2V_EINVAL, "gemm/conv3x3: up2_phase must be 0..4 (got %d)", up);
    AV2V_REQUIRE(a->K == (up ? 4 : 9) * a->Cin, AV2V_EINVAL, "gemm/conv3x3: K must equal 9*Cin (4*Cin for an up2 phase)");
    AV2V_REQUIRE(!up || (a->stride <= 1 && !a->rowbias && !a->residual && a->n_slots == 1), AV2V_EINVAL,
                 "gemm/conv3x3: an up2 phase takes bias only (no stride, rowbias, residual, slots)");
    const int stride = a->stride == 0 ? 1 : a->stride;
    AV2V_REQUIRE(stride == 1 || stride == 2, AV2V_ENOSUP, "gemm/conv3x3: stride must be 1 or 2 (got %d)", a->stride);
    AV2V_REQUIRE(a->H % stride == 0 && a->W % stride == 0, AV2V_ENOSUP, "gemm/conv3x3: H, W must be multiples of the stride");
    const int chan = a->a_channels == 0 ? a->Cin : a->a_channels;  // channels really present (the rest of the K block reads zeros)
    AV2V_REQUIRE(chan > 0 && chan <= a->Cin && chan % 8 == 0, AV2V_EINVAL, "gemm/conv3x3: a_channels must be a multiple of 8 in (0, Cin]");
    AV2V_REQUIRE(static_cast<long long>(a->NF) * (a->H / stride) * (a->W / stride) == a->M, AV2V_EINVAL,
                 "gemm/conv3x3: M != NF*(H/stride)*(W/stride)");
    p.Hin = a->H;
    p.Win = a->W;
    p.chan = chan;
    p.Ho = a->H / stride;
    p.Wo = a->W / stride;
    p.stride = stride;
    p.Cin = a->Cin;
    if (up) {
      p.up2 = 1;
      p.taps_w = 2;
      p.py = (up - 1) >> 1;
      p.px = (up - 1) & 1;
    }
  } else if (a->mode == AV2V_A_TCONV3) {
    AV2V_REQUIRE(a->B > 0 && a->rows_per_clip > 0 && a->HW > 0 && a->Cin > 0, AV2V_EINVAL, "gemm/tconv3: bad geometry");
    AV2V_REQUIRE(a->Cin % BK == 0, AV2V_ENOSUP, "gemm/tconv3: Cin must be a multiple of 64 (got %d)", a->Cin);
    AV2V_REQUIRE(a->K == 3 * a->Cin, AV2V_EINVAL, "gemm/tconv3: K must equal 3*Cin");
    AV2V_REQUIRE(a->rows_per_clip % a->HW == 0, AV2V_EINVAL, "gemm/tconv3: rows_per_clip must be F*HW");
    AV2V_REQUIRE(static_cast<long long>(a->B) * a->rows_per_clip == a->M, AV2V_EINVAL, "gemm/tconv3: M != B*F*HW");
    p.Cin = a->Cin;
    p.HW = a->HW;
    p.F = a->rows_per_clip / a->HW;
  } else {
    return fail(AV2V_EINVAL, "gemm: unknown A mode %d", a->mode);
  }
  p.num_kb = (a->K + BK - 1) / BK;
  unsigned box[3];
  const bool ws = p.mode == AV2V_A_LINEAR || conv_ws_box(p, box);
  const int bn = ws ? ws_tile_n(p) : BN;
  p.n_tiles = (a->N + bn - 1) / bn;
  const long long tiles = static_cast<long long>((a->M + BM - 1) / BM) * p.n_tiles;
  AV2V_REQUIRE(tiles < (1ll << 31), AV2V_ENOSUP, "gemm: too many tiles");
  if (p.mode == AV2V_A_LINEAR) return gemm_linear_ws(p, static_cast<int>(tiles), stream);
  if (ws) return gemm_conv_ws(p, box, static_cast<int>(tiles), stream);
  static bool attr_set = false;
  if (!attr_set) {
    AV2V_CHECK_CUDA(cudaFuncSetAttribute(gemm_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    attr_set = true;
  }
  gemm_wgmma_kernel<<<static_cast<unsigned>(tiles), kThreads, kSmemBytes, stream>>>(p);
  AV2V_CHECK_CUDA(cudaGetLastError());
  return AV2V_OK;
}
