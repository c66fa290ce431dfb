// Persistent, warp-specialized GEMM of the LINEAR A mode (sm_90a): every nn.Linear / 1 x 1 conv of the UNet.
//
//   out[m, n] = sum_k A[m, k] * W[n, k] + bias[n] + rowbias[m / rows_per_rowbias, n] + residual[m, n]   (or GEGLU)
//
// These GEMMs have short K loops (K = C: 5 blocks of 64 at C = 320), so a CTA that runs one tile through load, K loop and
// epilogue leaves the tensor cores idle for a large share of its life.  Here one CTA per SM walks a static tile schedule
// (tile blockIdx.x + i * gridDim.x, column tiles fastest, so the CTAs running at one time share A row blocks in L2) with
// three warpgroups:
//   producer (warpgroup 0, registers lowered): one thread issues the TMA loads of every K block of every tile of the CTA
//     into a kStages ring of 32 KB stages (A 128 x 64 and W 128 x 64 boxes, 128-byte swizzle = the sw128 layout the wgmma
//     descriptors read; TMA zero-fills ragged M / N, the K tail and the columns past k_split of a two-source A).  Stage s
//     has a full barrier (1 arrival + the transaction bytes) and an empty barrier (one arrival per consumer warp).  It runs
//     ahead across tile boundaries, so the next tile's first blocks land under this tile's last MMAs and epilogue.
//   consumers (warpgroups 1, 2, registers raised): warpgroup w takes the CTA's tiles i = w, w + 2, ... whole: 128 rows x
//     128 columns as two wgmma.m64n128k16 per k16 step (rows 0-63, 64-127) into 128 fp32 accumulators per thread.  Their
//     K loops take turns through two named barriers (math order 0, 1, 0, 1, ...): a warpgroup hands the tensor cores over
//     once it has issued its last MMA of a tile and runs its epilogue under the other's K loop.  A ring stage is released
//     after wgmma.wait_group has retired the MMAs that read it.
// Global block g = i * num_kb + kb of the CTA sits in stage g % kStages; its full phase is (g / kStages) & 1, and the
// producer refills the stage after the empty phase ((g / kStages) - 1) & 1 has completed (tools/kernel_models.py models
// this schedule).
//
// Epilogue (arithmetic as in gemm_wgmma.cu, so outputs are bit-identical to it): + bias / rowbias in fp32, + residual, one
// rounding; GEGLU pairs the h and gate columns that geglu_pack interleaves, output tile 128 x 64.  Each consumer warpgroup
// has its own 32 KB staging tile (128 rows x 256 bytes, 16-byte chunk c of row r at chunk c ^ (r & 7)); each warp owns the
// 32 rows its accumulators hold (16 of each 64-row half), fetches their residual chunks by cp.async before its K loop,
// writes the results in fragment order and copies its rows out with 16-byte stores, so a warp needs only __syncwarp: all
// of a warp's residual reads complete before its first store (a residual that aliases out stays safe), and its copy-out
// reads complete before the next tile's residual fetch or stores refill the tile.
#include "gemm_common.cuh"

namespace av2v {
namespace {

constexpr int BM = 128, BN = 128, BK = 64;
constexpr int kStages = 4;
constexpr int kThreads = 384;
constexpr int kTileBytes = BM * BK * 2;                // 16 KB: A and W boxes alike (BM == BN)
constexpr int kStageBytes = 2 * kTileBytes;
constexpr int kStagingBytes = BM * BN * 2;             // 32 KB per consumer warpgroup
constexpr int kSmemBytes = kStages * kStageBytes + 2 * kStagingBytes + 1024;

struct LinWsP {
  CUtensorMap ta, ta2, tw;  // A (columns [0, k_split)), second source (columns [k_split, K)), W [N][K]
  GemmP g;
  int tiles;
};

// byte offset of 16-byte chunk `chunk` of row `row` in a staging tile (256-byte rows), the layout of gemm_wgmma.cu's
__device__ __forceinline__ uint32_t stage_offset(int row, int chunk) {
  return static_cast<uint32_t>(row * 256 + ((chunk ^ (row & 7)) << 4));
}

// this warp's 32 rows (16 per 64-row half) of the residual tile -> staging tile, zero-filled past M / N
__device__ __forceinline__ void load_residual_rows(const GemmP& p, int m0, int n0, uint32_t tile) {
  const int lane = threadIdx.x & 31, ch = lane & 15, warp = (threadIdx.x >> 5) & 3;
  const int c = n0 + 8 * ch;
  const __half* src = p.residual + c;
#pragma unroll
  for (int half = 0; half < 2; ++half)
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int r = 64 * half + 16 * warp + 2 * i + (lane >> 4);
      const bool v = m0 + r < p.M && c < p.N;
      cp_async16(tile + stage_offset(r, ch), v ? src + static_cast<long long>(m0 + r) * p.ldo : p.residual, v);
    }
}

__device__ __forceinline__ void epilogue(const GemmP& p, float (&d)[2][64], int m0, int n0, uint32_t tile) {
  const int cq = 2 * (threadIdx.x & 3);
  if (p.geglu) {
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
    return;
  }
  const __half* rb[2][2];
#pragma unroll
  for (int half = 0; half < 2; ++half)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = m0 + 64 * half + acc_row(0) + 8 * h;
      rb[half][h] = p.rowbias && m < p.M ? p.rowbias + static_cast<long long>(m / p.rows_per_rowbias) * p.N : nullptr;
    }
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int c = n0 + 8 * j + cq;
    if (c >= p.N) continue;
    float2 b = make_float2(0.f, 0.f);
    if (p.bias) b = __half22float2(*reinterpret_cast<const __half2*>(p.bias + c));
#pragma unroll
    for (int half = 0; half < 2; ++half)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t at = tile + stage_offset(64 * half + acc_row(0) + 8 * h, j) + 2 * cq;
        float o0 = d[half][4 * j + 2 * h], o1 = d[half][4 * j + 2 * h + 1];
        if (p.bias) {
          o0 += b.x;
          o1 += b.y;
        }
        if (rb[half][h]) {
          const float2 t = __half22float2(*reinterpret_cast<const __half2*>(rb[half][h] + c));
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

// lane -> 16-byte chunk of a row, a warp instruction covers 2 rows x 256 bytes (GEGLU: 4 rows x 128 bytes)
__device__ __forceinline__ void copy_out(const GemmP& p, int m0, int n0, uint32_t tile) {
  const int lane = threadIdx.x & 31, warp = (threadIdx.x >> 5) & 3;
  const int lg = p.geglu ? 3 : 4;  // log2(chunks per output row of the tile)
  const int col0 = p.geglu ? n0 / 2 : n0, n_out = p.geglu ? p.N / 2 : p.N;
  __half* out = p.out + col0;
#pragma unroll
  for (int half = 0; half < 2; ++half)
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int idx = 32 * i + lane;
      const int r = 64 * half + 16 * warp + (idx >> lg), ch = idx & ((1 << lg) - 1);
      if ((idx >> lg) < 16 && m0 + r < p.M && col0 + 8 * ch < n_out)
        st_global_v4(out + static_cast<long long>(m0 + r) * p.ldo + 8 * ch, ld_shared_v4(tile + stage_offset(r, ch)));
    }
}

__global__ void __launch_bounds__(kThreads, 1) gemm_linear_ws_kernel(const __grid_constant__ LinWsP P) {
  const GemmP& p = P.g;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full[kStages], empty[kStages];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t s0 = smem_u32(smem);
  auto sA = [&](int s) { return s0 + static_cast<uint32_t>(s) * kStageBytes; };
  auto sB = [&](int s) { return sA(s) + kTileBytes; };
  const int nk = p.num_kb;
  if (threadIdx.x == 0) {
#pragma unroll
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 4);  // lane 0 of each warp of the consuming warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int role = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 7), 0);  // warp-uniform for ptxas
  if (role == 0) {  // ---- producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int g = 0;
      for (int t = blockIdx.x; t < P.tiles; t += gridDim.x) {
        const int m0 = t / p.n_tiles * BM, n0 = t % p.n_tiles * BN;
        for (int kb = 0; kb < nk; ++kb, ++g) {
          const int s = g % kStages, k0 = kb * BK;
          if (g >= kStages) mbar_wait<false>(&empty[s], ((g / kStages) - 1) & 1);  // the consumer released block g - kStages
          mbar_arrive_expect_tx(&full[s], kStageBytes);
          if (k0 < p.k_split) tma_load_4d(sA(s), &P.ta, &full[s], k0, m0, 0, 0);
          else tma_load_4d(sA(s), &P.ta2, &full[s], k0 - p.k_split, m0, 0, 0);
          tma_load_4d(sB(s), &P.tw, &full[s], k0, n0, 0, 0);
        }
      }
    }
    return;
  }

  // ---- consumers
  setmaxnreg_inc<232>();
  const int wg = role - 1;
  const uint32_t staging = s0 + kStages * kStageBytes + wg * kStagingBytes;
  // turn taking: warpgroup w waits on barrier 1 + w and, when another tile follows its own, hands over with an arrive on the
  // other's.  Warpgroup 1's arrive ahead of its first turn opens tile 0, so every sync has exactly one matching arrive.
  auto my_turn = [&] { if (wg == 0) named_bar_sync(1, 256); else named_bar_sync(2, 256); };
  auto hand_over = [&] { if (wg == 0) named_bar_arrive(2, 256); else named_bar_arrive(1, 256); };
  auto release = [&](int g) {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(&empty[g % kStages]);
  };
  if (wg == 1) named_bar_arrive(1, 256);

  float d[2][64];
  for (int i = wg, t = blockIdx.x + wg * gridDim.x; t < P.tiles; i += 2, t += 2 * gridDim.x) {
    const int m0 = t / p.n_tiles * BM, n0 = t % p.n_tiles * BN;
    if (p.residual) load_residual_rows(p, m0, n0, staging);
    cp_async_commit();
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int e = 0; e < 64; ++e) d[h][e] = 0.f;
    const int g0 = i * nk;
    my_turn();
    for (int kb = 0; kb < nk; ++kb) {
      const int g = g0 + kb, s = g % kStages;
      mbar_wait<false>(&full[s], (g / kStages) & 1);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        const uint64_t db = sw128_desc(sB(s) + k * 32);
        wgmma_m64n128_ss(d[0], sw128_desc(sA(s) + k * 32), db, 1);
        wgmma_m64n128_ss(d[1], sw128_desc(sA(s) + 64 * 128 + k * 32), db, 1);
      }
      wgmma_commit();
      wgmma_wait<1>();
      reg_fence(d[0]);
      reg_fence(d[1]);
      if (kb > 0) release(g - 1);
    }
    if (t + gridDim.x < P.tiles) hand_over();
    wgmma_wait<0>();
    reg_fence(d[0]);
    reg_fence(d[1]);
    release(g0 + nk - 1);

    cp_async_wait<0>();
    __syncwarp();  // the residual chunks this warp's lanes fetched for each other have landed
    epilogue(p, d, m0, n0, staging);
    __syncwarp();
    copy_out(p, m0, n0, staging);
    __syncwarp();  // every lane's copy-out reads are done before the next tile refills the warp's rows
  }
}

}  // namespace

int gemm_linear_ws(const GemmP& g, cudaStream_t stream) {
  AV2V_REQUIRE(g.n_slots == 1, AV2V_ENOSUP, "gemm/linear: one output slot only (got n_slots = %d)", g.n_slots);
  LinWsP P{};
  P.g = g;
  if (int e = encode_rows_map(&P.ta, g.a, g.k_split, g.M, 1, 1, g.lda, 0, BM)) return e;
  P.ta2 = P.ta;
  if (g.a2 != nullptr)
    if (int e = encode_rows_map(&P.ta2, g.a2, g.K - g.k_split, g.M, 1, 1, g.lda2, 0, BM)) return e;
  if (int e = encode_rows_map(&P.tw, g.w, g.K, g.N, 1, 1, g.K, 0, BN)) return e;
  const long long tiles = static_cast<long long>((g.M + BM - 1) / BM) * g.n_tiles;
  P.tiles = static_cast<int>(tiles);
  static bool attr_set = false;
  if (!attr_set) {
    AV2V_CHECK_CUDA(cudaFuncSetAttribute(gemm_linear_ws_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    attr_set = true;
  }
  const int grid = static_cast<int>(tiles < sm_count_cached() ? tiles : sm_count_cached());
  gemm_linear_ws_kernel<<<grid, kThreads, kSmemBytes, stream>>>(P);
  AV2V_CHECK_CUDA(cudaGetLastError());
  return AV2V_OK;
}

}  // namespace av2v
