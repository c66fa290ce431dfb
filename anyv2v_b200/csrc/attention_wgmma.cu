// PnP attention core on wgmma (sm_90a), head_dim 64: av2v_attn_pnp_f16 (spatial / cross / temporal attention, with the PnP
// Q/K injection folded in) and av2v_tattn_fused_f16 (temporal self-attention with the Q/K/V projection in the same kernel).
//
// A CTA holds 128 query slots, two warpgroups of 64.  Per 64-key tile a warpgroup computes S = Q K^T with wgmma.m64n64k16
// (Q and K as 128-byte-swizzled K-major tiles in shared memory), runs the online softmax on its accumulator registers
// (running max / sum per row, base-2 exponentials; a quarter of them on the FMA pipe, ex2_poly), converts P to fp16 in
// registers — the accumulator layout of S is the A-fragment layout of the next wgmma — and accumulates O += P V with V read
// MN-major ([keys][64], 64 contiguous) from shared memory.  With n_v = 3 (injected step) ONE P feeds the V of all three
// branches; n_v = 2 is the same step replayed from cached source Q / K, the two edit branches only.  K / V tiles are double-buffered with cp.async.  Rows-mode calls with 512 keys or more run attn_rows_kernel
// instead: the same per-row algorithm, warp-specialized (ring.cuh).  av2v_tattn_fused_f16 runs tattn_fused_kernel:
// persistent, its Q/K/V projection fed through the same ring, then the same attention per item (see its comment below).
//
// Query slots map to token rows by mode:
//   rows   : slot i of q tile qt -> token qt * 128 + i of sequence b; keys = the b / kv_batch_div-th key sequence.
//   frames : tokens are frame-major [clips][F][HW][*].  F <= 128: a CTA packs ppt = floor(128 / F) pixels of a clip, slot
//            i < ppt * F -> (pixel i / F, frame i % F), and the keys are the same 128 slots masked to the slot's own pixel.
//            Slots ppt * F .. 127 (the tail, empty when F | 128) hold no pixel: they load as zeros, and since slot / F >= ppt
//            for them they are never a key of a held slot, and they are never stored.  F > 128: one pixel per CTA, slot i ->
//            frame ft * 128 + i (f_tiles = ceil(F / 128) tiles), keys = all F frames of the pixel; frames >= F are neither
//            loaded as queries nor stored, and as keys they are zero-filled and masked.
#include "host_util.cuh"
#include "ptx.cuh"
#include "ring.cuh"

namespace av2v {
namespace {

constexpr int HD = 64;
constexpr int kThreads = 256;
constexpr int kTile = 64 * 128;  // bytes of a 64-row, 64-column fp16 tile

// 16-byte chunk loads of `rows` tile rows (64 fp16 each) into a swizzled tile, all 256 threads; row_ptr(r) -> source or null
// (a null row is zero-filled; `any` is a valid address handed to cp.async, which then reads nothing)
template <typename RowPtr>
__device__ __forceinline__ void load_tile(uint32_t dst, int rows, const __half* any, RowPtr row_ptr) {
  for (int c = threadIdx.x; c < rows * 8; c += kThreads) {
    const int r = c >> 3, ch = c & 7;
    const __half* src = row_ptr(r);
    cp_async16(dst + sw128_offset(r, ch), src ? src + ch * 8 : any, src != nullptr);
  }
}

// Online-softmax attention of one warpgroup's 64 query rows against one 64-key tile.  keep(row, key) masks scores;
// m / l: running max (base-2 scaled) and partial sum of the thread's rows r, r + 8.
template <int NV, typename Keep>
__device__ __forceinline__ void attn_tile(uint32_t q_wg, uint32_t k_tile, const uint32_t (&v_tile)[NV], float (&o)[NV][32],
                                          float (&m)[2], float (&l)[2], float scale_log2, Keep keep) {
  float s[32];
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < HD / 16; ++k) wgmma_m64n64_ss<0>(s, sw128_desc(q_wg + k * 32), sw128_desc(k_tile + k * 32), k > 0);
  wgmma_commit();
  wgmma_wait<0>();
  reg_fence(s);

  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const float v = keep(acc_row(i), acc_col(i)) ? s[i] * scale_log2 : -INFINITY;
    s[i] = v;
    mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], v);
  }
  float corr[2], ref[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
    mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
    const float mn = fmaxf(m[h], mx[h]);
    ref[h] = mn == -INFINITY ? 0.f : mn;  // a row with every key masked so far keeps p = 0
    corr[h] = ex2_approx(m[h] - ref[h]);
    m[h] = mn;
    l[h] *= corr[h];
  }
#pragma unroll
  for (int b = 0; b < NV; ++b)
#pragma unroll
    for (int i = 0; i < 32; ++i) o[b][i] *= corr[(i >> 1) & 1];
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const float x = s[i] - ref[(i >> 1) & 1];
    s[i] = ((i >> 2) & 3) == 3 ? ex2_poly(x) : ex2_approx(x);
    l[(i >> 1) & 1] += s[i];
  }
  uint32_t pa[4][4];
#pragma unroll
  for (int kk = 0; kk < 4; ++kk)
#pragma unroll
    for (int r = 0; r < 4; ++r) pa[kk][r] = pack_half2(s[8 * kk + 2 * r], s[8 * kk + 2 * r + 1]);
  wgmma_fence();
#pragma unroll
  for (int b = 0; b < NV; ++b)
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_m64n64_rs<1>(o[b], pa[kk], sw128_desc(v_tile[b] + kk * 2048), 1);
  wgmma_commit();
  wgmma_wait<0>();
#pragma unroll
  for (int b = 0; b < NV; ++b) reg_fence(o[b]);
}

// O / l -> fp16, rows mapped by out_row(slot) (negative: not stored)
template <int NV, typename OutRow>
__device__ __forceinline__ void store_o(float (&o)[NV][32], float (&l)[2], __half* const (&obase)[NV], int wg, OutRow out_row) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
    l[h] = l[h] > 0.f ? 1.f / l[h] : 0.f;
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const long long orow = out_row(wg * 64 + acc_row(2 * h));
    if (orow < 0) continue;
#pragma unroll
    for (int b = 0; b < NV; ++b)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int i = 4 * j + 2 * h;
        *reinterpret_cast<uint32_t*>(obase[b] + orow + acc_col(i)) = pack_half2(o[b][i] * l[h], o[b][i + 1] * l[h]);
      }
  }
}

// --------------------------------------------------------------------------------------------------- av2v_attn_pnp_f16
struct AttnP {
  int seq_mode;
  const __half *q, *k, *v;
  __half* o;
  int ldq, ldk, ldv, ldo;
  int heads;
  long long v_branch_stride, o_branch_stride;
  float scale_log2;
  int seq, seq_kv, kv_div, q_tiles;  // rows
  int F, HW, ppt, pix_tiles, f_tiles;  // frames
};

template <int NV>
__global__ void __launch_bounds__(kThreads) attn_kernel(const __grid_constant__ AttnP p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t sQ = smem_u32(smem);
  auto sK = [&](int buf) { return sQ + 2 * kTile + buf * (1 + NV) * kTile; };
  auto sV = [&](int buf, int b) { return sK(buf) + (1 + b) * kTile; };
  const int wg = threadIdx.x >> 7;

  // item -> (sequence / pixel group, head, query tile); qrow(slot) / krow(key) give token rows, -1 for none
  int item = blockIdx.x;
  const bool packed = p.seq_mode == AV2V_SEQ_FRAMES && p.F <= 128;
  int h, qt, b = 0, clip = 0, pix0 = 0, n_kv;
  if (p.seq_mode == AV2V_SEQ_ROWS) {
    qt = item % p.q_tiles;
    item /= p.q_tiles;
    h = item % p.heads;
    b = item / p.heads;
    n_kv = (p.seq_kv + 63) / 64;
  } else if (packed) {
    qt = item % p.pix_tiles;
    item /= p.pix_tiles;
    h = item % p.heads;
    clip = item / p.heads;
    pix0 = qt * p.ppt;
    n_kv = 2;
  } else {
    qt = item % p.f_tiles;
    item /= p.f_tiles;
    h = item % p.heads;
    item /= p.heads;
    pix0 = item % p.HW;
    clip = item / p.HW;
    n_kv = (p.F + 63) / 64;
  }
  // packed: slot i holds pixel pix0 + i / F when that is below pix_end; tail slots (i / F >= ppt) and pixels past HW hold none
  const int pix_end = min(pix0 + p.ppt, p.HW);
  const long long clip_row = static_cast<long long>(clip) * p.F * p.HW;
  auto qrow = [&](int i) -> long long {
    if (p.seq_mode == AV2V_SEQ_ROWS) {
      const int t = qt * 128 + i;
      return t < p.seq ? static_cast<long long>(b) * p.seq + t : -1;
    }
    if (packed) {
      const int pix = pix0 + i / p.F;
      return pix < pix_end ? clip_row + static_cast<long long>(i % p.F) * p.HW + pix : -1;
    }
    const int f = qt * 128 + i;
    return f < p.F ? clip_row + static_cast<long long>(f) * p.HW + pix0 : -1;
  };
  auto krow = [&](int u) -> long long {  // key u of the key sequence(s)
    if (p.seq_mode == AV2V_SEQ_ROWS)
      return u < p.seq_kv ? static_cast<long long>(b / p.kv_div) * p.seq_kv + u : -1;
    if (packed) {
      const int pix = pix0 + u / p.F;
      return pix < pix_end ? clip_row + static_cast<long long>(u % p.F) * p.HW + pix : -1;
    }
    return u < p.F ? clip_row + static_cast<long long>(u) * p.HW + pix0 : -1;
  };
  const int hc = h * HD;
  auto load_kv = [&](int kt, int buf) {
    load_tile(sK(buf), 64, p.k, [&](int r) -> const __half* {
      const long long row = krow(kt * 64 + r);
      return row < 0 ? nullptr : p.k + row * p.ldk + hc;
    });
#pragma unroll
    for (int vb = 0; vb < NV; ++vb)
      load_tile(sV(buf, vb), 64, p.v, [&](int r) -> const __half* {
        const long long row = krow(kt * 64 + r);
        return row < 0 ? nullptr : p.v + vb * p.v_branch_stride + row * p.ldv + hc;
      });
  };
  load_tile(sQ, 128, p.q, [&](int r) -> const __half* {
    const long long row = qrow(r);
    return row < 0 ? nullptr : p.q + row * p.ldq + hc;
  });
  load_kv(0, 0);
  cp_async_commit();

  float o[NV][32];
#pragma unroll
  for (int vb = 0; vb < NV; ++vb)
#pragma unroll
    for (int i = 0; i < 32; ++i) o[vb][i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  const int nk = p.seq_kv;  // rows: keys per key sequence; frames: F (keys past it are zero-filled, and masked here)
  for (int kt = 0; kt < n_kv; ++kt) {
    if (kt + 1 < n_kv) {
      load_kv(kt + 1, (kt + 1) & 1);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    fence_proxy_async_smem();
    __syncthreads();
    uint32_t vt[NV];
#pragma unroll
    for (int vb = 0; vb < NV; ++vb) vt[vb] = sV(kt & 1, vb);
    const int q0 = wg * 64, k0 = kt * 64;
    if (packed) {
      const int F = p.F;
      attn_tile<NV>(sQ + wg * kTile, sK(kt & 1), vt, o, m, l, p.scale_log2,
                    [&](int r, int c) { return (q0 + r) / F == (k0 + c) / F; });
    } else {
      attn_tile<NV>(sQ + wg * kTile, sK(kt & 1), vt, o, m, l, p.scale_log2, [&](int, int c) { return k0 + c < nk; });
    }
    __syncthreads();  // every warpgroup is done with this buffer before the next prefetch overwrites it
  }
  __half* ob[NV];
#pragma unroll
  for (int vb = 0; vb < NV; ++vb) ob[vb] = p.o + vb * p.o_branch_stride + hc;
  store_o<NV>(o, l, ob, wg, [&](int i) -> long long {
    const long long row = qrow(i);
    return row < 0 ? -1 : row * p.ldo;
  });
}

template <int NV>
constexpr int attn_smem() { return 2 * kTile + 2 * (1 + NV) * kTile + 1024; }

// --------------------------------------------------------------------------------------------------- rows mode, pipelined
// attn_rows_kernel: the rows-mode path of av2v_attn_pnp_f16, warp-specialized.  384 threads: warpgroup 0 is the producer (one
// thread issues TMA loads; registers lowered to 40), warpgroups 1 and 2 are the consumers (64 query rows each; raised to 232).
// Q (128 rows) is loaded once; K and the NV V tiles of key tile j are ring block j (ring.cuh); the tensor maps zero-fill
// keys past seq_kv and query rows past seq, so 0 * NaN never reaches PV.  Per turn a consumer issues PV(j) and S(j + 1)
// as one wgmma group, hands over, waits for it, releases stage j and runs softmax(j + 1) under the other's MMAs.
// Key tile: 128 keys at NV = 1 (S m64n128, half the rescale work of 64); 64 at NV = 3, where O alone holds 96 registers and
// S + P of 128 keys would not fit the 168 a thread of a 384-thread CTA is compiled for.  NV = 2 keeps the 64 keys of NV = 3:
// a branch's online softmax then rescales at the same tiles, so its output is bit-identical to the same branch at NV = 3.
// Per-row algorithm as attn_tile: running max over raw scores, x = s * scale_log2 - ref in one FMA, a quarter of the
// exponentials (key columns 24-31 of every 32) on the FMA pipe, fp16 P as the register A operand of PV, one division by l at
// the store.
template <int NV>
__host__ __device__ constexpr int rows_keys() { return NV == 1 ? 128 : 64; }
constexpr int kRowsStages = 6;  // 6 x (K + NV V tiles): 192 KB at either NV, 1 CTA per SM
template <int NV>
constexpr int rows_smem() { return 2 * kTile + kRowsStages * (1 + NV) * rows_keys<NV>() * 128 + 1024; }
constexpr int kRowsThreads = 384;
// Rows-mode calls with fewer keys stay on attn_kernel: with one CTA per SM, the prologue (Q and the first stage in flight) and
// the store are not hidden behind another CTA, and a key loop of 4 tiles or fewer does not pay for them (tools/attn_bench.py:
// 64- and 256-token self-attention and 145-key cross-attention are no faster, 1024- and 4096-token self-attention 2x faster).
constexpr int kRowsMinKeys = 512;

struct AttnRowsP {
  CUtensorMap tq, tk, tv;  // 4-D (column, token, sequence, V branch) fp16 maps, boxes 64 x 128 (Q) / 64 x key tile (K, V)
  __half* o;
  int ldo, heads, seq, seq_kv, kv_div, q_tiles;
  long long o_branch_stride;
  float scale_log2;
};

// softmax of one score tile (N = 2 * key tile / 4 registers) in place -> fp16 P fragments; rescales O and l by the raised
// running max.  kMask: keys at columns >= lim are past seq_kv.
template <int NV, int N, bool kMask>
__device__ __forceinline__ void rows_softmax(float (&s)[N], uint32_t (&pa)[N / 8][4], float (&o)[NV][32], float (&m)[2],
                                             float (&l)[2], float scale_log2, int lim) {
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int i = 0; i < N; ++i) {
    if (kMask && acc_col(i) >= lim) s[i] = -INFINITY;
    mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], s[i]);
  }
  float corr[2], nref[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
    mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
    const float mn = fmaxf(m[h], mx[h] * scale_log2);
    const float ref = mn == -INFINITY ? 0.f : mn;  // a row with every key masked so far keeps p = 0
    corr[h] = ex2_approx(m[h] - ref);
    nref[h] = -ref;
    m[h] = mn;
    l[h] *= corr[h];
  }
#pragma unroll
  for (int b = 0; b < NV; ++b)
#pragma unroll
    for (int i = 0; i < 32; ++i) o[b][i] *= corr[(i >> 1) & 1];
#pragma unroll
  for (int i = 0; i < N; ++i) {
    const float x = fmaf(s[i], scale_log2, nref[(i >> 1) & 1]);
    s[i] = ((i >> 2) & 3) == 3 ? ex2_poly(x) : ex2_approx(x);
    l[(i >> 1) & 1] += s[i];
  }
#pragma unroll
  for (int kk = 0; kk < N / 8; ++kk)
#pragma unroll
    for (int r = 0; r < 4; ++r) pa[kk][r] = pack_half2(s[8 * kk + 2 * r], s[8 * kk + 2 * r + 1]);
}

template <int NV>
__global__ void __launch_bounds__(kRowsThreads, 1) attn_rows_kernel(const __grid_constant__ AttnRowsP p) {
  constexpr int S = kRowsStages, KT = rows_keys<NV>(), N = KT / 2;
  constexpr uint32_t kKV = KT * 128;  // bytes of one K or V tile
  extern __shared__ uint8_t smem_raw[];
  __shared__ StageRing<S> ring;
  __shared__ __align__(8) uint64_t qbar;
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t sQ = smem_u32(smem);
  auto sK = [&](int s) { return sQ + 2 * kTile + s * (1 + NV) * kKV; };
  auto sV = [&](int s, int b) { return sK(s) + (1 + b) * kKV; };

  int item = blockIdx.x;
  const int qt = item % p.q_tiles;
  item /= p.q_tiles;
  const int h = item % p.heads;
  const int b = item / p.heads;
  const int n_kv = (p.seq_kv + KT - 1) / KT;
  if (threadIdx.x == 0) {
    ring.init(8);  // every consumer warp
    mbar_init(&qbar, 1);
    fence_mbar_init();
  }
  __syncthreads();

  const int role = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 7), 0);  // warp-uniform for ptxas
  if (role == 0) {  // ---- producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(&qbar, 2 * kTile);
      tma_load_4d(sQ, &p.tq, &qbar, h * HD, qt * 128, b, 0);
      const int kvb = b / p.kv_div;
      for (int j = 0; j < n_kv; ++j) {
        const int s = ring.stage(j);
        uint64_t* bar = ring.produce(j, (1 + NV) * kKV);
        tma_load_4d(sK(s), &p.tk, bar, h * HD, j * KT, kvb, 0);
#pragma unroll
        for (int vb = 0; vb < NV; ++vb) tma_load_4d(sV(s, vb), &p.tv, bar, h * HD, j * KT, kvb, vb);
      }
    }
    return;
  }

  // ---- consumers
  setmaxnreg_inc<232>();
  const int wg = role - 1;
  const uint32_t q_wg = sQ + wg * kTile;
  float o[NV][32];
#pragma unroll
  for (int vb = 0; vb < NV; ++vb)
#pragma unroll
    for (int i = 0; i < 32; ++i) o[vb][i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float s[N];
  uint32_t pa[N / 8][4];
  auto issue_s = [&](int j) {
#pragma unroll
    for (int k = 0; k < HD / 16; ++k) {
      if constexpr (KT == 128) wgmma_m64n128_ss(s, sw128_desc(q_wg + k * 32), sw128_desc(sK(ring.stage(j)) + k * 32), k > 0);
      else wgmma_m64n64_ss<0>(s, sw128_desc(q_wg + k * 32), sw128_desc(sK(ring.stage(j)) + k * 32), k > 0);
    }
  };
  auto issue_pv = [&](int j) {
#pragma unroll
    for (int vb = 0; vb < NV; ++vb)
#pragma unroll
      for (int kk = 0; kk < KT / 16; ++kk) wgmma_m64n64_rs<1>(o[vb], pa[kk], sw128_desc(sV(ring.stage(j), vb) + kk * 2048), 1);
  };
  auto softmax = [&](int j) {
    const int lim = p.seq_kv - j * KT;
    if (lim >= KT) rows_softmax<NV, N, false>(s, pa, o, m, l, p.scale_log2, lim);
    else rows_softmax<NV, N, true>(s, pa, o, m, l, p.scale_log2, lim);
  };
  turn_open(wg);  // both warpgroups take n_kv + 1 turns: this arrive stands in for warpgroup 1's hand-over after its last
  mbar_wait<false>(&qbar, 0);
  ring.wait(0);
  turn_take(wg);
  wgmma_fence();
  issue_s(0);
  wgmma_commit();
  turn_hand_over(wg);
  wgmma_wait<0>();
  reg_fence(s);
  softmax(0);
  for (int j = 0; j + 1 < n_kv; ++j) {
    ring.wait(j + 1);
    turn_take(wg);
    wgmma_fence();
    issue_pv(j);
    issue_s(j + 1);
    wgmma_commit();
    turn_hand_over(wg);
    wgmma_wait<0>();
#pragma unroll
    for (int vb = 0; vb < NV; ++vb) reg_fence(o[vb]);
    reg_fence(s);
    ring.release(j);
    softmax(j + 1);
  }
  turn_take(wg);
  wgmma_fence();
  issue_pv(n_kv - 1);
  wgmma_commit();
  if (wg == 0) turn_hand_over(wg);
  wgmma_wait<0>();
#pragma unroll
  for (int vb = 0; vb < NV; ++vb) reg_fence(o[vb]);
  ring.release(n_kv - 1);

  __half* ob[NV];
#pragma unroll
  for (int vb = 0; vb < NV; ++vb) ob[vb] = p.o + vb * p.o_branch_stride + h * HD;
  store_o<NV>(o, l, ob, wg, [&](int i) -> long long {
    const int t = qt * 128 + i;
    return t < p.seq ? (static_cast<long long>(b) * p.seq + t) * p.ldo : -1;
  });
}

// --------------------------------------------------------------------------------------------------- av2v_tattn_fused_f16
// tattn_fused_kernel: persistent and warp-specialized.  One CTA per SM walks the items blockIdx.x, + gridDim.x, ...; items are
// numbered heads fastest, then pixel tile, then clip, so the CTAs running at one time hold the heads of the same few pixel
// tiles and each x tile leaves HBM once (the other heads read it from L2; the weights, 3C x Cx, stay in L2 throughout).
// 384 threads: warpgroups 0 and 1 are the consumers (64 slots each; registers raised to 232), warpgroup 2 the producer
// (registers lowered to 40), whose thread 0 issues the TMA loads of every projection K block of every item of the CTA into a
// ring of tattn_stages stages (ring.cuh).  A stage holds the x block (the item's 128 slots x 64 channels, one box of x viewed
// as (channel, frame, pixel, clip): slot i = (pixel pix0 + i / F, frame i % F)) and the pass's weight boxes (64 x 64 rows of
// Q, K, V, or of V alone for the V-only passes of an n_v = 3 item).  The producer runs ahead across items, so the next item's
// first blocks land while this one runs its attention and stores (tools/kernel_models.py models this).
// Rows ppt * F .. 127 of a stage's x block (the tail, when F does not divide 128) are never written by a box of the launch,
// all boxes having one shape: they are zeroed once, before the first load, so the tail slots project to zero Q, K, V (a
// tail V row is multiplied by P = 0, and 0 x NaN would reach every row).  Pixels past HW are zero-filled by the TMA.
// Per item a consumer warpgroup runs the K loop of each pass with one MMA group in flight, writes the fp16 Q / K / V of its 64
// slots (after the other warpgroup has finished the previous item's attention: named barrier 1), and after a second barrier
// runs the attention of its 64 slots against the keys of the same pixel and stores O.  Each accumulator sums its K blocks in
// order, one wgmma group at a time, so results do not depend on the ring depth, the schedule or the grid size.
// QK = true (av2v_tattn_fused_qksrc_f16, NV = 2): pass 0 projects Q and K alone from the source tensor (map tqk, same box), and
// NV V-only passes follow, one per edit clip.  Every accumulator sums the same K blocks in the same order as at NV = 3.
struct TAttnP {
  CUtensorMap tx;   // x as (channel, frame, pixel, clip), box {64, F, ppt, 1}
  CUtensorMap tqk;  // QK only: the Q / K source, same view and box
  CUtensorMap tw;  // wqkv [3C][Cx], box 64 x 64
  __half* o;
  int ldo, F, HW, heads, Cx, ppt, pix_tiles, src_clips, items;
  int n_kt;  // key tiles per warpgroup: 1 (its own half) when F | 64, else 2
  float scale_log2;
};

template <int NV>
__host__ __device__ constexpr int tattn_stages() { return NV == 1 ? 4 : 3; }
constexpr int kTStageBytes = 2 * kTile + 3 * kTile;  // x block (128 x 64) + up to 3 weight boxes (64 x 64): 40 KB
constexpr int kTThreads = 384;
// smem: Q, K (128 x 64 each), V per branch (128 x 64), then the ring
template <int NV>
constexpr int tattn_smem() { return (2 + NV) * 2 * kTile + tattn_stages<NV>() * kTStageBytes + 1024; }

// accumulator (64 x 64 of warpgroup wg) -> fp16 into the swizzled 128 x 64 tile at `tile` (the projection GEMM's rounding)
__device__ __forceinline__ void acc_to_tile(const float (&acc)[32], uint32_t tile, int wg) {
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    const int r = wg * 64 + acc_row(i), c = acc_col(i);
    const uint32_t addr = tile + sw128_offset(r, c >> 3) + (c & 7) * 2;
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(pack_half2(acc[i], acc[i + 1])) : "memory");
  }
}

template <int NV, bool QK = false>
__global__ void __launch_bounds__(kTThreads, 1) tattn_fused_kernel(const __grid_constant__ TAttnP p) {
  constexpr int S = tattn_stages<NV>();
  constexpr int passes = QK ? NV + 1 : NV;
  extern __shared__ uint8_t smem_raw[];
  __shared__ StageRing<S> ring;
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t sQ = smem_u32(smem), sK = sQ + 2 * kTile;
  auto sV = [&](int b) { return sQ + (2 + b) * 2 * kTile; };
  auto sX = [&](int s) { return sQ + (2 + NV) * 2 * kTile + s * kTStageBytes; };  // the stages follow V
  auto sW = [&](int s, int q) { return sX(s) + (2 + q) * kTile; };
  const int F = p.F, C = p.heads * HD, nk = p.Cx / 64, slots = p.ppt * F;

  {  // the tail rows of every stage's x block
    uint8_t* ring_p = smem + (2 + NV) * 2 * kTile;
    const int tail_chunks = (128 - slots) * 8;
    for (int c = threadIdx.x; c < S * tail_chunks; c += kTThreads)
      *reinterpret_cast<uint4*>(ring_p + (c / tail_chunks) * kTStageBytes + slots * 128 + (c % tail_chunks) * 16) =
          make_uint4(0u, 0u, 0u, 0u);
    fence_proxy_async_smem();
  }
  if (threadIdx.x == 0) {
    ring.init(8);  // every consumer warp
    fence_mbar_init();
  }
  __syncthreads();

  // item -> (head h, pixel tile pt, clip): clip is the source clip at n_v = 3
  auto decode = [&](int item, int& h, int& pix0, int& clip) {
    h = item % p.heads;
    item /= p.heads;
    pix0 = item % p.pix_tiles * p.ppt;
    clip = item / p.pix_tiles;
  };

  const int role = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 7), 0);  // warp-uniform for ptxas
  if (role == 2) {  // ---- producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 256) {
      const uint32_t x_bytes = slots * 128;
      int g = 0;
      for (int item = blockIdx.x; item < p.items; item += gridDim.x) {
        int h, pix0, clip;
        decode(item, h, pix0, clip);
        // pass 0: Q, K, V of the (source) clip; pass b > 0: V of clip + b * src_clips.  QK: pass 0 is Q, K of source clip
        // `clip`, pass b > 0 the V of clip + (b - 1) * src_clips of x
        constexpr int w0 = QK ? 2 : 3;  // weight boxes of pass 0
        for (int b = 0; b < passes; ++b)
          for (int kb = 0; kb < nk; ++kb, ++g) {
            const int s = ring.stage(g);
            uint64_t* bar = ring.produce(g, x_bytes + (b == 0 ? w0 : 1) * kTile);
            if (!QK) tma_load_4d(sX(s), &p.tx, bar, kb * 64, 0, pix0, clip + b * p.src_clips);
            else if (b == 0) tma_load_4d(sX(s), &p.tqk, bar, kb * 64, 0, pix0, clip);
            else tma_load_4d(sX(s), &p.tx, bar, kb * 64, 0, pix0, clip + (b - 1) * p.src_clips);
            if (b == 0) {
#pragma unroll
              for (int q = 0; q < w0; ++q) tma_load_4d(sW(s, q), &p.tw, bar, kb * 64, q * C + h * HD, 0, 0);
            } else {
              tma_load_4d(sW(s, 0), &p.tw, bar, kb * 64, 2 * C + h * HD, 0, 0);
            }
          }
      }
    }
    return;
  }

  // ---- consumers
  setmaxnreg_inc<232>();
  const int wg = role;
  int g = 0;  // the CTA's global K block, in the producer's order
  // acc[q] (64 x 64 of this warpgroup's slots) = x block rows @ weight box q, over the nk K blocks of one pass
  auto project = [&](auto& acc) {
    constexpr int NP = sizeof(acc) / sizeof(acc[0]);
#pragma unroll
    for (int q = 0; q < NP; ++q)
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[q][i] = 0.f;
    for (int kb = 0; kb < nk; ++kb) {
      const int s = ring.stage(g + kb);
      ring.wait(g + kb);
      wgmma_fence();
#pragma unroll
      for (int q = 0; q < NP; ++q)
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_m64n64_ss<0>(acc[q], sw128_desc(sX(s) + wg * kTile + k * 32), sw128_desc(sW(s, q) + k * 32), 1);
      wgmma_commit();
      wgmma_wait<1>();
#pragma unroll
      for (int q = 0; q < NP; ++q) reg_fence(acc[q]);
      if (kb > 0) ring.release(g + kb - 1);
    }
    wgmma_wait<0>();
#pragma unroll
    for (int q = 0; q < NP; ++q) reg_fence(acc[q]);
    ring.release(g + nk - 1);
    g += nk;
  };

  const int q0 = wg * 64;
  for (int item = blockIdx.x; item < p.items; item += gridDim.x) {
    int h, pix0, clip;
    decode(item, h, pix0, clip);
    const int pix_end = min(pix0 + p.ppt, p.HW);
    {
      float acc[QK ? 2 : 3][32];
      project(acc);
      // the other warpgroup has finished the previous item's attention (its reads of Q / K / V)
      if (item != blockIdx.x) named_bar_sync(1, 256);
      acc_to_tile(acc[0], sQ, wg);
      acc_to_tile(acc[1], sK, wg);
      if constexpr (!QK) acc_to_tile(acc[2], sV(0), wg);
    }
#pragma unroll
    for (int b = QK ? 0 : 1; b < NV; ++b) {
      float acc[1][32];
      project(acc);
      acc_to_tile(acc[0], sV(b), wg);
    }
    fence_proxy_async_smem();
    named_bar_sync(1, 256);

    float o[NV][32];
#pragma unroll
    for (int b = 0; b < NV; ++b)
#pragma unroll
      for (int i = 0; i < 32; ++i) o[b][i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    // when F divides 64 no pixel crosses the 64-slot halves: each warpgroup then needs only its own key half.  For every
    // other F some pixel does (e.g. F = 24: slots 48..71), so both warpgroups visit both key tiles.  The tile count is the
    // same for both and the tile index is data, not control flow, so both issue the same wgmma sequence.
    const int n_kt = p.n_kt;
    for (int it = 0; it < n_kt; ++it) {
      const int kt = n_kt == 1 ? wg : it;
      const int k0 = kt * 64;
      uint32_t vt[NV];
#pragma unroll
      for (int b = 0; b < NV; ++b) vt[b] = sV(b) + kt * kTile;
      attn_tile<NV>(sQ + wg * kTile, sK + kt * kTile, vt, o, m, l, p.scale_log2,
                    [&](int r, int c) { return (q0 + r) / F == (k0 + c) / F; });
    }
    // branch b writes the rows of its own clip, clip + b * src_clips; slot i holds pixel pix0 + i / F below pix_end
#pragma unroll
    for (int b = 0; b < NV; ++b) {
      float (&ob)[1][32] = *reinterpret_cast<float(*)[1][32]>(&o[b]);
      float lb[2] = {l[0], l[1]};
      __half* const o1[1] = {p.o + h * HD};
      const long long clip_row = static_cast<long long>(clip + b * p.src_clips) * F;
      store_o<1>(ob, lb, o1, wg, [&](int i) -> long long {
        const int pix = pix0 + i / F;
        return pix < pix_end ? ((clip_row + i % F) * p.HW + pix) * p.ldo : -1;
      });
    }
  }
}

}  // namespace
}  // namespace av2v

using namespace av2v;

extern "C" int av2v_attn_pnp_f16(const av2v_attn_args* a, av2v_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  AV2V_REQUIRE(a != nullptr, AV2V_EINVAL, "attn: null args");
  AV2V_REQUIRE(a->q && a->k && a->v && a->o, AV2V_EINVAL, "attn: null q/k/v/o");
  AV2V_REQUIRE(a->batch > 0 && a->seq > 0 && a->heads > 0, AV2V_EINVAL, "attn: batch/seq/heads must be positive");
  AV2V_REQUIRE(a->n_v >= 1 && a->n_v <= 3, AV2V_EINVAL, "attn: n_v must be 1, 2 or 3 (got %d)", a->n_v);
  AV2V_REQUIRE(a->ldq % 8 == 0 && a->ldk % 8 == 0 && a->ldv % 8 == 0 && a->ldo % 8 == 0, AV2V_EALIGN,
               "attn: row strides must be multiples of 8 elements");
  AV2V_REQUIRE(a->ldq >= a->heads * HD && a->ldk >= a->heads * HD && a->ldv >= a->heads * HD &&
                   a->ldo >= a->heads * HD,
               AV2V_EINVAL, "attn: row strides must cover heads*64 columns");
  AV2V_REQUIRE(aligned16(a->q) && aligned16(a->k) && aligned16(a->v) && aligned16(a->o), AV2V_EALIGN,
               "attn: q/k/v/o must be 16-byte aligned");
  AV2V_REQUIRE(a->scale > 0.f, AV2V_EINVAL, "attn: scale must be positive");
  AV2V_REQUIRE(a->n_v == 1 || (a->v_branch_stride % 8 == 0 && a->o_branch_stride % 8 == 0), AV2V_EALIGN,
               "attn: branch strides must be multiples of 8 elements");

  AttnP p{};
  p.seq_mode = a->seq_mode;
  p.q = static_cast<const __half*>(a->q);
  p.k = static_cast<const __half*>(a->k);
  p.v = static_cast<const __half*>(a->v);
  p.o = static_cast<__half*>(a->o);
  p.ldq = a->ldq;
  p.ldk = a->ldk;
  p.ldv = a->ldv;
  p.ldo = a->ldo;
  p.heads = a->heads;
  p.v_branch_stride = a->n_v > 1 ? a->v_branch_stride : 0;
  p.o_branch_stride = a->n_v > 1 ? a->o_branch_stride : 0;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  p.seq = a->seq;
  p.seq_kv = a->seq_kv > 0 ? a->seq_kv : a->seq;
  p.kv_div = a->kv_batch_div > 0 ? a->kv_batch_div : 1;
  long long items;
  if (a->seq_mode == AV2V_SEQ_ROWS) {
    AV2V_REQUIRE(a->batch % p.kv_div == 0, AV2V_EINVAL, "attn: batch must be a multiple of kv_batch_div");
    p.q_tiles = (a->seq + 127) / 128;
    items = static_cast<long long>(a->batch) * a->heads * p.q_tiles;
  } else if (a->seq_mode == AV2V_SEQ_FRAMES) {
    const int F = a->seq, HW = a->HW;
    AV2V_REQUIRE(HW > 0 && a->batch % HW == 0, AV2V_EINVAL, "attn/frames: batch must be clips*HW");
    AV2V_REQUIRE((a->seq_kv <= 0 || a->seq_kv == a->seq) && p.kv_div == 1, AV2V_ENOSUP,
                 "attn/frames: self-attention only (seq_kv / kv_batch_div are rows-mode options)");
    const int clips = a->batch / HW;
    p.F = F;
    p.HW = HW;
    if (F <= 128) {
      p.ppt = 128 / F;
      p.pix_tiles = (HW + p.ppt - 1) / p.ppt;
      items = static_cast<long long>(clips) * a->heads * p.pix_tiles;
    } else {
      p.f_tiles = (F + 127) / 128;
      items = static_cast<long long>(clips) * HW * a->heads * p.f_tiles;
    }
  } else {
    return fail(AV2V_EINVAL, "attn: unknown seq_mode %d", a->seq_mode);
  }
  AV2V_REQUIRE(items < (1ll << 31), AV2V_ENOSUP, "attn: too many work items");
  static bool attr_set = false;
  if (!attr_set) {
    AV2V_CHECK_CUDA(cudaFuncSetAttribute(attn_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, attn_smem<1>()));
    AV2V_CHECK_CUDA(cudaFuncSetAttribute(attn_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, attn_smem<2>()));
    AV2V_CHECK_CUDA(cudaFuncSetAttribute(attn_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, attn_smem<3>()));
    AV2V_CHECK_CUDA(cudaFuncSetAttribute(attn_rows_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, rows_smem<1>()));
    AV2V_CHECK_CUDA(cudaFuncSetAttribute(attn_rows_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, rows_smem<2>()));
    AV2V_CHECK_CUDA(cudaFuncSetAttribute(attn_rows_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, rows_smem<3>()));
    attr_set = true;
  }
  if (a->seq_mode == AV2V_SEQ_ROWS && p.seq_kv >= kRowsMinKeys) {
    AttnRowsP r{};
    const int C = a->heads * HD, kv_seqs = a->batch / p.kv_div;
    const int kt = a->n_v == 1 ? rows_keys<1>() : a->n_v == 2 ? rows_keys<2>() : rows_keys<3>();
    if (int e = encode_rows_map(&r.tq, a->q, C, a->seq, a->batch, 1, a->ldq, 0, 128)) return e;
    if (int e = encode_rows_map(&r.tk, a->k, C, p.seq_kv, kv_seqs, 1, a->ldk, 0, kt)) return e;
    if (int e = encode_rows_map(&r.tv, a->v, C, p.seq_kv, kv_seqs, a->n_v, a->ldv, p.v_branch_stride, kt)) return e;
    r.o = p.o;
    r.ldo = a->ldo;
    r.heads = a->heads;
    r.seq = a->seq;
    r.seq_kv = p.seq_kv;
    r.kv_div = p.kv_div;
    r.q_tiles = p.q_tiles;
    r.o_branch_stride = p.o_branch_stride;
    r.scale_log2 = p.scale_log2;
    if (a->n_v == 3) attn_rows_kernel<3><<<static_cast<unsigned>(items), kRowsThreads, rows_smem<3>(), stream>>>(r);
    else if (a->n_v == 2) attn_rows_kernel<2><<<static_cast<unsigned>(items), kRowsThreads, rows_smem<2>(), stream>>>(r);
    else attn_rows_kernel<1><<<static_cast<unsigned>(items), kRowsThreads, rows_smem<1>(), stream>>>(r);
  } else if (a->n_v == 3) attn_kernel<3><<<static_cast<unsigned>(items), kThreads, attn_smem<3>(), stream>>>(p);
  else if (a->n_v == 2) attn_kernel<2><<<static_cast<unsigned>(items), kThreads, attn_smem<2>(), stream>>>(p);
  else attn_kernel<1><<<static_cast<unsigned>(items), kThreads, attn_smem<1>(), stream>>>(p);
  AV2V_CHECK_CUDA(cudaGetLastError());
  return AV2V_OK;
}

// the launch of tattn_fused_kernel for validated arguments: a->n_v = 1 | 3, or n_v = 2 with Q / K from qk_src (QK = true)
static int tattn_fused_launch(const av2v_tattn_fused_args* a, const void* qk_src, int ld_src, cudaStream_t stream) {
  TAttnP p{};
  p.o = static_cast<__half*>(a->o);
  p.ldo = a->ldo;
  p.F = a->F;
  p.HW = a->HW;
  p.heads = a->heads;
  p.Cx = a->Cx;
  p.ppt = 128 / a->F;
  p.pix_tiles = (a->HW + p.ppt - 1) / p.ppt;
  p.n_kt = 64 % a->F == 0 ? 1 : 2;
  p.src_clips = a->n_v > 1 ? a->clips / a->n_v : a->clips;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  const long long items = static_cast<long long>(p.src_clips) * a->heads * p.pix_tiles;
  AV2V_REQUIRE(items < (1ll << 31), AV2V_ENOSUP, "tattn_fused: too many work items");
  p.items = static_cast<int>(items);
  // x [clips][F][HW][ldx] as (channel, frame, pixel, clip): the box {64, F, ppt, 1} lands in slot order (pixel-major)
  auto x_map = [&](CUtensorMap* map, const void* base, int ld, int clips) {
    const unsigned long long row = static_cast<unsigned long long>(ld) * 2, frame = row * a->HW;
    const unsigned long long dims[4] = {static_cast<unsigned long long>(a->Cx), static_cast<unsigned long long>(a->F),
                                        static_cast<unsigned long long>(a->HW), static_cast<unsigned long long>(clips)};
    const unsigned long long strides[3] = {frame, row, frame * a->F};
    const unsigned box[4] = {64, static_cast<unsigned>(a->F), static_cast<unsigned>(p.ppt), 1};
    return encode_map_4d(map, base, dims, strides, box);
  };
  if (int e = x_map(&p.tx, a->x, a->ldx, a->clips)) return e;
  if (qk_src != nullptr)
    if (int e = x_map(&p.tqk, qk_src, ld_src, p.src_clips)) return e;
  if (int e = encode_rows_map(&p.tw, a->wqkv, a->Cx, 3 * a->heads * HD, 1, 1, a->Cx, 0, 64)) return e;
  static bool attr_set = false;
  if (!attr_set) {
    AV2V_CHECK_CUDA(cudaFuncSetAttribute(tattn_fused_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, tattn_smem<1>()));
    AV2V_CHECK_CUDA(cudaFuncSetAttribute(tattn_fused_kernel<2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, tattn_smem<2>()));
    AV2V_CHECK_CUDA(cudaFuncSetAttribute(tattn_fused_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, tattn_smem<3>()));
    attr_set = true;
  }
  const unsigned grid = static_cast<unsigned>(items < sm_count_cached() ? items : sm_count_cached());
  if (qk_src != nullptr) tattn_fused_kernel<2, true><<<grid, kTThreads, tattn_smem<2>(), stream>>>(p);
  else if (a->n_v == 3) tattn_fused_kernel<3><<<grid, kTThreads, tattn_smem<3>(), stream>>>(p);
  else tattn_fused_kernel<1><<<grid, kTThreads, tattn_smem<1>(), stream>>>(p);
  AV2V_CHECK_CUDA(cudaGetLastError());
  return AV2V_OK;
}

extern "C" int av2v_tattn_fused_f16(const av2v_tattn_fused_args* a, av2v_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  AV2V_REQUIRE(a != nullptr, AV2V_EINVAL, "tattn_fused: null args");
  AV2V_REQUIRE(a->x && a->wqkv && a->o, AV2V_EINVAL, "tattn_fused: null x / wqkv / o");
  AV2V_REQUIRE(a->clips > 0 && a->F > 0 && a->HW > 0 && a->heads > 0 && a->Cx > 0, AV2V_EINVAL, "tattn_fused: bad shape");
  AV2V_REQUIRE(a->F <= 128, AV2V_ENOSUP, "tattn_fused: F must be at most 128 (got %d)", a->F);
  AV2V_REQUIRE(a->Cx % 64 == 0, AV2V_ENOSUP, "tattn_fused: the input width must be a multiple of 64 (got %d)", a->Cx);
  AV2V_REQUIRE(a->ldx % 8 == 0 && a->ldx >= a->Cx && a->ldo % 8 == 0 && a->ldo >= a->heads * HD, AV2V_EINVAL,
               "tattn_fused: row strides must be multiples of 8 covering the rows");
  AV2V_REQUIRE(aligned16(a->x) && aligned16(a->wqkv) && aligned16(a->o), AV2V_EALIGN, "tattn_fused: pointers must be 16-byte aligned");
  AV2V_REQUIRE(a->scale > 0.f, AV2V_EINVAL, "tattn_fused: scale must be positive");
  AV2V_REQUIRE(a->n_v == 1 || a->n_v == 3, AV2V_EINVAL, "tattn_fused: n_v must be 1 or 3 (got %d)", a->n_v);
  AV2V_REQUIRE(a->n_v == 1 || a->clips % 3 == 0, AV2V_EINVAL, "tattn_fused: n_v = 3 needs clips = 3 x clips-per-branch (got %d)", a->clips);
  return tattn_fused_launch(a, nullptr, 0, stream);
}

extern "C" int av2v_tattn_fused_qksrc_f16(const av2v_tattn_fused_qksrc_args* a, av2v_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  AV2V_REQUIRE(a != nullptr, AV2V_EINVAL, "tattn_fused_qksrc: null args");
  AV2V_REQUIRE(a->x && a->qk_src && a->wqkv && a->o, AV2V_EINVAL, "tattn_fused_qksrc: null x / qk_src / wqkv / o");
  AV2V_REQUIRE(a->clips > 0 && a->clips % 2 == 0 && a->F > 0 && a->HW > 0 && a->heads > 0 && a->Cx > 0, AV2V_EINVAL,
               "tattn_fused_qksrc: bad shape (clips must be even)");
  AV2V_REQUIRE(a->F <= 128, AV2V_ENOSUP, "tattn_fused_qksrc: F must be at most 128 (got %d)", a->F);
  AV2V_REQUIRE(a->Cx % 64 == 0, AV2V_ENOSUP, "tattn_fused_qksrc: the input width must be a multiple of 64 (got %d)", a->Cx);
  AV2V_REQUIRE(a->ldx % 8 == 0 && a->ldx >= a->Cx && a->ld_src % 8 == 0 && a->ld_src >= a->Cx && a->ldo % 8 == 0 &&
                   a->ldo >= a->heads * HD,
               AV2V_EINVAL, "tattn_fused_qksrc: row strides must be multiples of 8 covering the rows");
  AV2V_REQUIRE(aligned16(a->x) && aligned16(a->qk_src) && aligned16(a->wqkv) && aligned16(a->o), AV2V_EALIGN,
               "tattn_fused_qksrc: pointers must be 16-byte aligned");
  AV2V_REQUIRE(a->scale > 0.f, AV2V_EINVAL, "tattn_fused_qksrc: scale must be positive");
  const av2v_tattn_fused_args b{a->x, a->wqkv, a->o, a->ldx, a->ldo, a->clips, a->F, a->HW, a->heads, a->Cx, a->scale, 2};
  return tattn_fused_launch(&b, a->qk_src, a->ld_src, stream);
}
