// Persistent, warp-specialized GEMM (sm_90a): every nn.Linear / 1 x 1 conv of the UNet (LINEAR), and the 3 x 3 / up2-phase /
// temporal convolutions whose 128-row tiles are each one TMA box of the input (conv_ws_box; the rest run on gemm_wgmma.cu).
//
//   out[slot][m, n] = sum_k A[m, k] * W[n, k] + bias[n] + rowbias[m / rows_per_rowbias, n] + residual[slot][m, n]   (or GEGLU)
//
// These GEMMs have short K loops (K = C: 5 blocks of 64 at C = 320), so a CTA that runs one tile through load, K loop and
// epilogue leaves the tensor cores idle for a large share of its life.  Here one CTA per SM walks a static tile schedule
// (tile blockIdx.x + i * gridDim.x, column tiles fastest, so the CTAs running at one time share A row blocks in L2) with
// three warpgroups:
//   producer (warpgroup 0, registers lowered): one thread issues the TMA loads of every K block g = i * num_kb + kb of the
//     CTA into a kStages ring (ring.cuh) of 32 / 36 KB stages (A 128 x 64 and W BN x 64 boxes, 128-byte swizzle = the
//     sw128 layout the wgmma descriptors read; TMA zero-fills ragged M / N, the K tail and the columns past k_split of a
//     two-source A).  It runs ahead across tile boundaries, so the next tile's first blocks land under this tile's last MMAs
//     and epilogue (tools/kernel_models.py models this schedule).
//   consumers (warpgroups 1, 2, registers raised): warpgroup w takes the CTA's tiles i = w, w + 2, ... whole: 128 rows x
//     BN columns as two wgmma.m64nBNk16 per k16 step (rows 0-63, 64-127) into BN fp32 accumulators per thread.  Their
//     K loops take turns (math order 0, 1, 0, 1, ...): a warpgroup hands the tensor cores over once it has issued its last
//     MMA of a tile and runs its epilogue under the other's K loop.
//
// The A source is a template parameter; only the producer's box coordinates and the epilogue's row mapping and slots differ.
//   LINEAR: A is [M][lda] (two sources split at k_split), box (k0, m0).
//   conv (kConv): K block kb lies inside one tap (Cin % 64 == 0), so it is a 64-channel slab of the channels-last input
//     shifted by the tap: the input is a 4-D tensor (CONV3X3 [NF][H][W][chan], TCONV3 [B][F][HW][C]) whose box
//     {64, bx, by, bn} holds exactly the 128 output rows of a tile, in row order (conv_ws_box picks it and refuses the
//     geometries where no box does; a 3 x 3 conv's last tile may be ragged, its box running past the last frame).  Tile row m0 starts the box at (m0 % ax + x_off, m0 / ax % ay + y_off, m0 / (ax ay)),
//     moved by the tap (kx, ky) = (tap % taps_w, tap / taps_w) of K block kb (tap = kb * 64 / Cin): the -1 offsets of a 3 x 3 conv, the phase offsets px - 1,
//     py - 1 of an up2 phase, the frame offset kt - 1 of the temporal conv.  TMA zero-fill outside the tensor is the
//     padding (out-of-image taps, the frames past either end of a clip, the channels past a_channels).  The smem image of a
//     box with 128-byte rows is the same sw128 tile whatever its shape, and every block holds the values gemm_wgmma.cu's
//     cp.async gather puts there, so K order, sum order and results are those of gemm_wgmma_kernel.
//
// The column tile BN is 128, or 160 where N is a multiple of 160 and the wider tiles shorten the schedule (ws_tile_n): the
// 64 x 64 level's N = 320 and 960 then run as whole tiles, and each A block feeds 160 columns.  At 160 the ring
// (4 x 36 KB) and the two staging tiles (2 x 40 KB) take 225 KB of shared memory.
//
// Epilogue: gemm_common.cuh's staged epilogue, shared with gemm_wgmma_kernel; GEGLU (BN = 128 only) pairs the h and gate
// columns that geglu_pack interleaves, output tile 128 x 64.  Each consumer warpgroup has its own 32 / 40 KB staging
// tile; each warp owns two bands (rows 16 w .. 16 w + 15 and 64 + 16 w .., one per accumulator) and fetches their
// residual chunks by cp.async before its K loop, so a warp needs only __syncwarp: all of a warp's residual reads complete
// before its first store (a residual that aliases out stays safe), and its copy-out reads complete before the next tile's residual fetch or stores
// refill the tile.  Conv with a residual in several slots (PnP conv injection) runs the slots one after another through
// the one staging tile: fetch residual s (slot 0's before the K loop), epilogue, copy out to slot s, __syncwarp; without a
// residual the one tile is copied to every slot.  An up2 phase writes its rows to the phase's pixels of the 2x output.
#include "gemm_common.cuh"
#include "ring.cuh"

namespace av2v {
namespace {

constexpr int BM = 128, BK = 64;
constexpr int kStages = 4;
constexpr int kThreads = 384;
constexpr int kTileBytes = BM * BK * 2;                       // 16 KB: the A box
template <int kBN> constexpr int kStageBytes = kTileBytes + kBN * BK * 2;  // + the W box: 32 / 36 KB
template <int kBN> constexpr int kStagingBytes = BM * kBN * 2;             // 32 / 40 KB per consumer warpgroup
template <int kBN> constexpr int kSmemBytes = kStages * kStageBytes<kBN> + 2 * kStagingBytes<kBN> + 1024;
static_assert(kSmemBytes<160> <= 227 * 1024, "the 160-wide ring and staging tiles must fit an SM's shared memory");

struct WsP {
  CUtensorMap ta, ta2, tw;  // A (LINEAR: columns [0, k_split); conv: the input tensor), second source (columns [k_split, K)), W [N][K]
  GemmP g;
  int tiles;
  int ax, ay, x_off, y_off, taps_w;  // conv: the box origin of tile row m0 and the taps per kernel row (see the top)
};

// GEGLU: h * gelu(gate) of the accumulator column pairs jh = 8 g + jj and jg = jh + 4 (the pairs geglu_pack interleaves)
// -> chunk 4 g + jj of the 128 x 64 output tile, for the rows of both bands
__device__ __forceinline__ void geglu_epilogue(const GemmP& p, float (&d)[2][64], int n0, uint32_t tile) {
  const int cq = 2 * (threadIdx.x & 3);
#pragma unroll
  for (int g = 0; g < 2; ++g) {
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int jh = 8 * g + jj, jg = jh + 4;
      const int ch = n0 + 8 * jh + cq, cg = n0 + 8 * jg + cq;
      if (ch >= p.N) continue;
      float2 bh = make_float2(0.f, 0.f), bg = bh;
      if (p.bias) {
        bh = __half22float2(*reinterpret_cast<const __half2*>(p.bias + ch));
        bg = __half22float2(*reinterpret_cast<const __half2*>(p.bias + cg));
      }
#pragma unroll
      for (int half = 0; half < 2; ++half)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float h0 = d[half][4 * jh + 2 * h], h1 = d[half][4 * jh + 2 * h + 1];
          float g0 = d[half][4 * jg + 2 * h], g1 = d[half][4 * jg + 2 * h + 1];
          if (p.bias) {
            h0 += bh.x; h1 += bh.y; g0 += bg.x; g1 += bg.y;
          }
          st_shared_u32(tile + stage_offset(64 * half + acc_row(0) + 8 * h, 4 * g + jj) + 2 * cq,
                        pack_half2(h0 * gelu_erf_fast(g0), h1 * gelu_erf_fast(g1)));
        }
    }
  }
}

template <bool kConv, int kBN>
__global__ void __launch_bounds__(kThreads, 1) gemm_ws_kernel(const __grid_constant__ WsP P) {
  constexpr int kStage = kStageBytes<kBN>, kStaging = kStagingBytes<kBN>;
  const GemmP& p = P.g;
  extern __shared__ uint8_t smem_raw[];
  __shared__ StageRing<kStages> ring;
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t s0 = smem_u32(smem);
  auto sA = [&](int s) { return s0 + static_cast<uint32_t>(s) * kStage; };
  auto sB = [&](int s) { return sA(s) + kTileBytes; };
  const int nk = p.num_kb;
  if (threadIdx.x == 0) {
    ring.init(4);  // the warps of the consuming warpgroup
    fence_mbar_init();
  }
  __syncthreads();

  const int role = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 7), 0);  // warp-uniform for ptxas
  if (role == 0) {  // ---- producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int g = 0;
      for (int t = blockIdx.x; t < P.tiles; t += gridDim.x) {
        const int m0 = t / p.n_tiles * BM, n0 = t % p.n_tiles * kBN;
        int bx = 0, by = 0, bn = 0, c0 = 0, kx = 0;  // conv: the tile's box origin, block kb's channel and tap column
        if constexpr (kConv) {
          bx = m0 % P.ax + P.x_off;
          by = m0 / P.ax % P.ay + P.y_off;
          bn = m0 / (P.ax * P.ay);
        }
        for (int kb = 0; kb < nk; ++kb, ++g) {
          const int s = ring.stage(g), k0 = kb * BK;
          uint64_t* bar = ring.produce(g, kStage);
          if constexpr (kConv) {  // block kb = tap (ky, kx), channels c0 .. c0 + 63; walked without divisions
            tma_load_4d(sA(s), &P.ta, bar, c0, bx + kx, by, bn);
            if ((c0 += BK) == p.Cin) {
              c0 = 0;
              if (++kx == P.taps_w) kx = 0, ++by;
            }
          } else if (k0 < p.k_split) tma_load_4d(sA(s), &P.ta, bar, k0, m0, 0, 0);
          else tma_load_4d(sA(s), &P.ta2, bar, k0 - p.k_split, m0, 0, 0);
          tma_load_4d(sB(s), &P.tw, bar, k0, n0, 0, 0);
        }
      }
    }
    return;
  }

  // ---- consumers
  setmaxnreg_inc<232>();
  const int wg = role - 1;
  const uint32_t staging = s0 + kStages * kStage + wg * kStaging;
  turn_open(wg);  // a warpgroup hands over only when another tile follows: every sync has exactly one matching arrive

  const int r0 = 16 * ((threadIdx.x >> 5) & 3);  // the warp's bands: tile rows r0 .. r0 + 15 and r0 + 64 ..
  float d[2][kBN / 2];
  for (int i = wg, t = blockIdx.x + wg * gridDim.x; t < P.tiles; i += 2, t += 2 * gridDim.x) {
    const int m0 = t / p.n_tiles * BM, n0 = t % p.n_tiles * kBN;
    if (p.residual)
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        if constexpr (kConv) fetch_residual_band<true, kBN>(p, 0, m0, n0, r0 + 64 * b, staging);
        else fetch_residual_band<false, kBN>(p, 0, m0, n0, r0 + 64 * b, staging);
      }
    cp_async_commit();
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int e = 0; e < kBN / 2; ++e) d[h][e] = 0.f;
    const int g0 = i * nk;
    turn_take(wg);
    for (int kb = 0; kb < nk; ++kb) {
      const int g = g0 + kb, s = ring.stage(g);
      ring.wait(g);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        const uint64_t db = sw128_desc(sB(s) + k * 32);
        if constexpr (kBN == 128) {
          wgmma_m64n128_ss(d[0], sw128_desc(sA(s) + k * 32), db, 1);
          wgmma_m64n128_ss(d[1], sw128_desc(sA(s) + 64 * 128 + k * 32), db, 1);
        } else {
          wgmma_m64n160_ss(d[0], sw128_desc(sA(s) + k * 32), db, 1);
          wgmma_m64n160_ss(d[1], sw128_desc(sA(s) + 64 * 128 + k * 32), db, 1);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();
      reg_fence(d[0]);
      reg_fence(d[1]);
      if (kb > 0) ring.release(g - 1);
    }
    if (t + gridDim.x < P.tiles) turn_hand_over(wg);
    wgmma_wait<0>();
    reg_fence(d[0]);
    reg_fence(d[1]);
    ring.release(g0 + nk - 1);

    if constexpr (kConv) {
      // d stays live across the slots: the slot and copy-out loops stay rolled so that the copy-out's addresses fit beside it
      const int n_res = p.residual ? p.n_slots : 1;  // distinct tiles: without a residual every slot stores the same one
#pragma unroll 1
      for (int sl = 0; sl < n_res; ++sl) {
        if (sl > 0) {  // the copy-out of slot sl - 1 has read the warp's rows (__syncwarp below)
#pragma unroll
          for (int b = 0; b < 2; ++b) fetch_residual_band<true, kBN>(p, sl, m0, n0, r0 + 64 * b, staging);
          cp_async_commit();
        }
        cp_async_wait<0>();
        __syncwarp();  // the residual chunks this warp's lanes fetched for each other have landed
        epilogue_bands<2>(p, d, m0, n0, r0, staging);
        __syncwarp();
#pragma unroll 1
        for (int o = p.residual ? sl : 0; o < (p.residual ? sl + 1 : p.n_slots); ++o)
#pragma unroll 1
          for (int b = 0; b < 2; ++b) copy_out_band<true, kBN>(p, o, m0, n0, r0 + 64 * b, staging);
        __syncwarp();  // every lane's copy-out reads are done before the next slot or tile refills the warp's rows
      }
    } else {
      cp_async_wait<0>();
      __syncwarp();  // the residual chunks this warp's lanes fetched for each other have landed
      if constexpr (kBN == 128) {
        if (p.geglu) geglu_epilogue(p, d, n0, staging);
        else epilogue_bands<2>(p, d, m0, n0, r0, staging);
      } else {
        epilogue_bands<2>(p, d, m0, n0, r0, staging);  // GEGLU runs on 128-wide tiles (ws_tile_n)
      }
      __syncwarp();
#pragma unroll
      for (int b = 0; b < 2; ++b) copy_out_band<false, kBN>(p, 0, m0, n0, r0 + 64 * b, staging);
      __syncwarp();  // every lane's copy-out reads are done before the next tile refills the warp's rows
    }
  }
}

template <bool kConv, int kBN>
int launch_ws(WsP P, cudaStream_t stream) {
  const GemmP& g = P.g;
  if (int e = encode_rows_map(&P.tw, g.w, g.K, g.N, 1, 1, g.K, 0, kBN)) return e;
  static bool attr_set = false;  // one per instantiation
  if (!attr_set) {
    AV2V_CHECK_CUDA(cudaFuncSetAttribute(gemm_ws_kernel<kConv, kBN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         kSmemBytes<kBN>));
    attr_set = true;
  }
  const int tiles = P.tiles;
  const int grid = static_cast<int>(tiles < sm_count_cached() ? tiles : sm_count_cached());
  gemm_ws_kernel<kConv, kBN><<<grid, kThreads, kSmemBytes<kBN>, stream>>>(P);
  AV2V_CHECK_CUDA(cudaGetLastError());
  return AV2V_OK;
}

}  // namespace

// The column tile: 160 where it shortens the schedule.  Each CTA runs its tiles one after another, so a GEMM takes about
// ceil(tiles / SMs) tile times, and a tile's time grows with its width.  160 takes N = 320 and 960 (the 64 x 64 level) as
// whole tiles instead of 3 and 8 with the last half empty, and at N = 640 or 1280 it feeds each A block to more columns;
// 128 stays where its extra tiles fill SMs that 160 would leave idle (the 8 x 8 level's 24 row tiles at N = 1280).  GEGLU
// keeps 128: geglu_pack interleaves its h and gate columns per 128-column tile.
int ws_tile_n(const GemmP& p) {
  if (p.geglu || p.N % 160 != 0) return 128;
  const long long mt = (p.M + BM - 1) / BM, sms = sm_count_cached();
  const long long t128 = (mt * ((p.N + 127) / 128) + sms - 1) / sms * 128, t160 = (mt * (p.N / 160) + sms - 1) / sms * 160;
  return t160 <= t128 ? 160 : 128;
}

int gemm_linear_ws(const GemmP& g, int tiles, cudaStream_t stream) {
  WsP P{};
  P.g = g;
  if (int e = encode_rows_map(&P.ta, g.a, g.k_split, g.M, 1, 1, g.lda, 0, BM)) return e;
  P.ta2 = P.ta;
  if (g.a2 != nullptr)
    if (int e = encode_rows_map(&P.ta2, g.a2, g.K - g.k_split, g.M, 1, 1, g.lda2, 0, BM)) return e;
  P.tiles = tiles;
  return ws_tile_n(g) == 160 ? launch_ws<false, 160>(P, stream) : launch_ws<false, 128>(P, stream);
}

// A conv runs here iff the 128 output rows of every tile are one box of its input, in row order:
//   CONV3X3, stride 1 or an up2 phase (the GEMM rows are the NF x Ho x Wo pixels, Ho x Wo the input's extent): Wo divides
//     128 and either 128 divides Ho Wo (box Wo x 128 / Wo x 1) or Ho Wo divides 128 (whole frames, box Wo x Ho x
//     128 / (Ho Wo)).  The frame is the outermost dimension, so the box of a ragged last tile runs past frame NF - 1 into
//     zeros, on rows past M that are never stored;
//   TCONV3 (rows B x F x HW): 128 divides HW (box 128 x 1) or HW divides 128 and 128 / HW divides F (box HW x 128 / HW):
//     a box past the last frame of a clip would hold zeros where the tile's rows are the next clip's first frame.
// box = {bx, by, bn}, the box extents past the 64 channels.
bool conv_ws_box(const GemmP& p, unsigned (&box)[3]) {
  if (p.mode == AV2V_A_CONV3X3) {
    const int hw = p.Ho * p.Wo;
    if (p.stride != 1 || BM % p.Wo != 0) return false;
    if (hw >= BM) {
      if (hw % BM != 0) return false;
      box[0] = p.Wo, box[1] = BM / p.Wo, box[2] = 1;
    } else {
      if (BM % hw != 0) return false;
      box[0] = p.Wo, box[1] = p.Ho, box[2] = BM / hw;
    }
    return true;
  }
  if (p.mode == AV2V_A_TCONV3) {
    if (p.HW % BM == 0) box[0] = BM, box[1] = 1, box[2] = 1;
    else if (BM % p.HW == 0 && p.F % (BM / p.HW) == 0) box[0] = p.HW, box[1] = BM / p.HW, box[2] = 1;
    else return false;
    return true;
  }
  return false;
}

int gemm_conv_ws(const GemmP& g, const unsigned (&box)[3], int tiles, cudaStream_t stream) {
  WsP P{};
  P.g = g;
  using u64 = unsigned long long;
  const unsigned b4[4] = {64, box[0], box[1], box[2]};
  if (g.mode == AV2V_A_CONV3X3) {  // [NF][Hin][Win][chan]; stride 1, so Hin = Ho, Win = Wo
    const u64 row = static_cast<u64>(g.chan) * 2, plane = row * g.Win * g.Hin;
    const u64 dims[4] = {static_cast<u64>(g.chan), static_cast<u64>(g.Win), static_cast<u64>(g.Hin),
                         static_cast<u64>(g.M / (g.Ho * g.Wo))};
    const u64 strides[3] = {row, row * g.Win, plane};
    if (int e = encode_map_4d(&P.ta, g.a, dims, strides, b4)) return e;
    P.ax = g.Wo, P.ay = g.Ho, P.taps_w = g.taps_w;
    P.x_off = g.up2 ? g.px - 1 : -1;
    P.y_off = g.up2 ? g.py - 1 : -1;
  } else {  // TCONV3: [B][F][HW][Cin]
    const u64 row = static_cast<u64>(g.Cin) * 2;
    const u64 dims[4] = {static_cast<u64>(g.Cin), static_cast<u64>(g.HW), static_cast<u64>(g.F),
                         static_cast<u64>(g.M / (g.F * g.HW))};
    const u64 strides[3] = {row, row * g.HW, row * g.HW * g.F};
    if (int e = encode_map_4d(&P.ta, g.a, dims, strides, b4)) return e;
    P.ax = g.HW, P.ay = g.F, P.taps_w = 1;
    P.x_off = 0;
    P.y_off = -1;
  }
  P.ta2 = P.ta;
  P.tiles = tiles;
  return ws_tile_n(g) == 160 ? launch_ws<true, 160>(P, stream) : launch_ws<true, 128>(P, stream);
}

}  // namespace av2v
