// Channels-last GroupNorm(+SiLU) (K6 of the hot path; reference ops: pnp_utils.py:48-49, 92, 104 and every other
// GroupNorm -> SiLU pair of the UNet / VAE).  HBM-bound: 4 B per element (read x once, write y once).
//
//   x, y : [n_samples][rows][C] fp16;  statistics per (sample, group) over rows x (C / groups) elements
//
// ONE persistent kernel, one CTA per SM, built around the 50 MB L2 (round 1 ran two kernels = three HBM passes, 6 B/element):
//   * the samples are cut into L2-sized CHUNKS (<= kChunkBytes of x).  For each chunk the whole grid first streams the chunk
//     once for the statistics (phase A: HBM -> L2 -> smem), meets at a grid-wide barrier, and then streams the SAME rows again
//     for the normalisation (phase B): that second read hits in L2, so x crosses HBM once.  A clip-level sample of the 64 x 64
//     level (65 536 rows x 320 channels = 42 MB) is one sample larger than a chunk; the per-frame norms (48 samples of 2.6 MB) go 7 frames at a time.
//     Samples larger than L2 (128-frame clips) still work — phase B then walks the chunk back to front, so its first reads
//     hit the part of x that phase A touched last.
//   * rows are contiguous in the channels-last layout, so a slice of rows is ONE byte range: a producer warp moves it with
//     1-D bulk TMA copies (cp.async.bulk, kStages x ~20 KB in flight per SM, completion on mbarriers); the consumer threads
//     only ever read shared memory.  No per-thread global loads, no address arithmetic in the inner loop.
//   * deterministic: per-(sample, slice, group) partial sums of x - k (k: one pivot element per sample and group, so the
//     variance does not cancel when |mean| >> sigma) in a fixed order, folded in double; no float atomics.
//     The grid barrier is one integer atomic per CTA and chunk.
#include "host_util.cuh"
#include "ptx.cuh"

namespace av2v {
namespace {

constexpr int kGnMaxSlices = 512;   // slices per sample (partial-sum slots)
constexpr int kGnMaxGroups = 64;
constexpr int kStages = 4;
constexpr int kStageBytes = 30 * 1024;                 // one stage = T consumer threads x U 16-byte vectors <= this
constexpr long long kChunkBytes = 20ll << 20;          // x + y of a chunk (2 x 20 MB) stay inside the 50 MB L2
// Two builds: <U = 3, T <= 640> and <U = 4, T <= 480> (T = consumer threads, a multiple of the vectors per row and of 32; U =
// vectors per thread and stage).  The SiLU pass is a chain of ~10 dependent instructions per element with two MUFU ops in it
// (~70 cycles); at the HBM rate an SM must retire ~1.5 elements per clock and sub-partition, which takes >= 100 independent
// element chains per sub-partition: 5 warps x 3 vectors x 8 elements (or 3.75 x 4 x 8), all U vectors of a thread batched
// through each step of the chain (measured: the first version, 480 threads x one vector at a time, ran at 0.25 of the roofline).

// grid barrier state: [0] arrivals of the running launch, [1] exits.  Zero at module load; the last CTA to exit resets both,
// so consecutive (stream-ordered) launches start from zero.  One process drives one GPU (SURVEY 8b), launches are stream-ordered.
__device__ unsigned int g_gn_sync[2];

struct GnParams {
  const __half* x;
  const __half* x2;    // second source (channels [C1, C) of the logical input) or nullptr: skip-concat without a torch.cat
  int C1, vpr1;        // channels / 16-byte vectors per row of the first source (= C, vpr when x2 == nullptr)
  __half* y;
  const __half* gamma;
  const __half* beta;
  float* partial;  // [n][slices][groups][2]
  int n, rows, C, groups, cpg, vpr;
  int rp;              // row lanes: consumer threads = vpr * rp
  int stage_rows;      // rp * U
  int slices;          // slices per sample
  int slots;           // partial-sum slots per sample = min(slices, gridDim.x)
  int rows_per_slice;
  int chunk_samples, n_chunks;
  float eps;
  int silu;
};

__device__ __forceinline__ void bulk_load_1d(uint32_t smem_dst, const void* gsrc, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_dst), "l"(gsrc), "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ unsigned int ld_acquire_gpu(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// mbarrier wait of the hot loops: bounded by an iteration count instead of clock64() (the consumers poll often; every clock read
// is an issue slot the SiLU pass does not have)
__device__ __forceinline__ void mbar_wait_hot(uint64_t* bar, uint32_t parity) {
  for (uint32_t spins = 0; !mbar_try_wait(bar, parity); ++spins) {
    if (spins > (1u << 28)) {
      printf("av2v: groupnorm pipeline wait timeout (block %d thread %d)\n", blockIdx.x, threadIdx.x);
      __trap();
    }
  }
}

// the statistics pivot of (sample s, group g): the group's first channel in row 0 of the sample, read from the source that holds
// it (so the two-source form and the concatenated input shift by the same value)
__device__ __forceinline__ __half gn_pivot(const GnParams& p, int s, int g) {
  const int c = g * p.cpg;
  const long long row0 = static_cast<long long>(s) * p.rows;
  return c < p.C1 ? p.x[row0 * p.C1 + c] : p.x2[row0 * (p.C - p.C1) + (c - p.C1)];
}

template <int U, int kMaxT>
__global__ void __launch_bounds__(kMaxT + 32, 1)
gn_persistent_kernel(const GnParams p) {
  extern __shared__ __align__(128) uint8_t gsm[];
  uint8_t* stage_buf = gsm;                                                      // [kStages][kStageBytes]
  float* red = reinterpret_cast<float*>(gsm + kStages * kStageBytes);            // [rp][C][2] fold scratch, then [groups][2]
  const int T = p.vpr * p.rp;                                                    // consumer threads (multiple of 32)
  uint64_t* bars = reinterpret_cast<uint64_t*>(red + static_cast<size_t>(p.rp) * p.C * 2 + 2 * kGnMaxGroups);
  uint64_t* full = bars;
  uint64_t* empty = bars + kStages;
  const int t = threadIdx.x;
  const int G = gridDim.x;
  const bool is_producer = t >= T;

  if (t == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], T / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();

  const long long row_bytes1 = static_cast<long long>(p.C1) * 2, row_bytes2 = static_cast<long long>(p.C - p.C1) * 2;
  const uint32_t region2 = static_cast<uint32_t>(p.stage_rows * row_bytes1);  // byte offset of the second source's rows in a stage
  // per item: rows [rbeg, rend) of sample s
  auto item_rows = [&](int slice, int& rbeg, int& rend) {
    rbeg = slice * p.rows_per_slice;
    rend = min(p.rows, rbeg + p.rows_per_slice);
  };

  if (is_producer) {
    // ================================================================== producer warp: the same stage sequence as the consumers
    if (t == T) {
      int stage = 0;
      uint32_t phase = 0;
      for (int ch = 0; ch < p.n_chunks; ++ch) {
        const int s0 = ch * p.chunk_samples;
        const int ns = min(p.chunk_samples, p.n - s0);
        const int items = ns * p.slices;
        for (int pass = 0; pass < 2; ++pass) {
          // phase A: items ascending; phase B: items descending (what phase A read last is what L2 still holds for sure)
          const int my = (items - static_cast<int>(blockIdx.x) + G - 1) / G;  // number of items of this CTA (may be <= 0)
          for (int ii = 0; ii < my; ++ii) {
            const int j = static_cast<int>(blockIdx.x) + (pass == 0 ? ii : my - 1 - ii) * G;
            const int s = s0 + j / p.slices, slice = j % p.slices;
            int rbeg, rend;
            item_rows(slice, rbeg, rend);
            const long long row0 = static_cast<long long>(s) * p.rows + rbeg;
            const uint8_t* src = reinterpret_cast<const uint8_t*>(p.x) + row0 * row_bytes1;
            const uint8_t* src2 = p.x2 ? reinterpret_cast<const uint8_t*>(p.x2) + row0 * row_bytes2 : nullptr;
            for (int r = rbeg; r < rend; r += p.stage_rows) {
              const int nr = min(p.stage_rows, rend - r);
              mbar_wait(&empty[stage], phase ^ 1u);
              const uint32_t bytes = static_cast<uint32_t>(nr * row_bytes1), bytes2 = static_cast<uint32_t>(nr * row_bytes2);
              mbar_arrive_expect_tx(&full[stage], bytes + bytes2);
              // the stage holds the two sources' row blocks one after the other: [stage_rows][C1] then [stage_rows][C - C1]
              bulk_load_1d(smem_u32(stage_buf + stage * kStageBytes), src, bytes, smem_u32(&full[stage]));
              if (src2) bulk_load_1d(smem_u32(stage_buf + stage * kStageBytes + region2), src2, bytes2, smem_u32(&full[stage]));
              src += bytes;
              src2 += bytes2;
              if (++stage == kStages) {
                stage = 0;
                phase ^= 1u;
              }
            }
          }
        }
      }
    }
    return;
  }

  // ==================================================================== consumers: thread = (8-channel vector v, row lane r0)
  const int v = t % p.vpr, r0 = t / p.vpr;
  const int lane = t & 31;
  // where this thread's 8-channel vector lives inside a stage: first or second source block, row pitch of that block
  const bool in2 = v >= p.vpr1;
  const int spitch = in2 ? p.vpr - p.vpr1 : p.vpr1;                                         // 16-byte vectors per row of the block
  const uint32_t sbase = in2 ? region2 + static_cast<uint32_t>(v - p.vpr1) * 16u : static_cast<uint32_t>(v) * 16u;
  int stage = 0;
  uint32_t phase = 0;
  unsigned int barrier_no = 0;
  auto consumer_sync = [&]() { asm volatile("bar.sync 1, %0;" ::"r"(T) : "memory"); };
  auto release_stage = [&]() {
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[stage]);
    if (++stage == kStages) {
      stage = 0;
      phase ^= 1u;
    }
  };

  for (int ch = 0; ch < p.n_chunks; ++ch) {
    const int s0 = ch * p.chunk_samples;
    const int ns = min(p.chunk_samples, p.n - s0);
    const int items = ns * p.slices;
    const int my = (items - static_cast<int>(blockIdx.x) + G - 1) / G;

    // ------------------------------------------------------------------ phase A: statistics
    // A CTA's items j = b, b + G, ... of a chunk are in ascending sample order, so its items of one sample are consecutive: the
    // per-thread sums run across them and are folded ONCE per (CTA, sample) into partial[sample][slot], slot = offset of the CTA's
    // first item inside the sample = a number in [0, min(slices, G)) that exactly one CTA owns (no zero-fill, no atomics).
    // The sums are SHIFTED: S1 = sum (x - k), S2 = sum (x - k)^2 with one pivot k per (sample, group), the group's first channel
    // in row 0 of the sample (gn_pivot).  Unshifted fp32 sums of x and x^2 lose the variance to cancellation in E[x^2] - mean^2
    // once |mean| / sigma is large (at 300, 43 % of the outputs of a 64 x 64 frame were > 1 fp16 ulp off); x - k is of the size of
    // sigma, so S2 / N - (S1 / N)^2 keeps the fp32 sums' relative precision.
    {
      float2 sm_[4], sq_[4];  // packed fp32x2 accumulators (two channels per issue slot; the same IEEE add / fma per lane)
      uint4 kh = make_uint4(0u, 0u, 0u, 0u);  // pivots of this thread's 8 channels (fp16), for the sample being summed
      int piv_sample = -1;
#pragma unroll
      for (int e = 0; e < 4; ++e) sm_[e] = sq_[e] = make_float2(0.f, 0.f);
      int soff[U];  // this thread's vectors inside a stage (constant)
#pragma unroll
      for (int u = 0; u < U; ++u) soff[u] = (r0 + u * p.rp) * spitch;
      for (int ii = 0; ii < my; ++ii) {
        const int j = static_cast<int>(blockIdx.x) + ii * G;
        const int sl_ = j / p.slices;  // sample index inside the chunk
        const int s = s0 + sl_, slice = j - sl_ * p.slices;
        if (s != piv_sample) {
          piv_sample = s;
          __half* khh = reinterpret_cast<__half*>(&kh);
#pragma unroll
          for (int e = 0; e < 8; ++e) khh[e] = gn_pivot(p, s, (v * 8 + e) / p.cpg);
        }
        int rbeg, rend;
        item_rows(slice, rbeg, rend);
        for (int r = rbeg; r < rend; r += p.stage_rows) {
          const int nr = min(p.stage_rows, rend - r);
          mbar_wait_hot(&full[stage], phase);
          const uint4* sb = reinterpret_cast<const uint4*>(stage_buf + stage * kStageBytes + sbase);
          uint4 a4[U];
#pragma unroll
          for (int u = 0; u < U; ++u) a4[u] = (r0 + u * p.rp < nr) ? sb[soff[u]] : kh;  // fill: x - k = 0 adds nothing
          float2 kv[4];  // fp32 pivots, converted per stage (kept live across the loop they spill the 672-thread build)
          const __half2* k2 = reinterpret_cast<const __half2*>(&kh);
#pragma unroll
          for (int e = 0; e < 4; ++e) kv[e] = __half22float2(k2[e]);
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const __half2* ah = reinterpret_cast<const __half2*>(&a4[u]);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float2 f = __half22float2(ah[e]);
              const float2 d = make_float2(__fsub_rn(f.x, kv[e].x), __fsub_rn(f.y, kv[e].y));
              sm_[e] = fadd2(sm_[e], d);
              sq_[e] = ffma2(d, d, sq_[e]);
            }
          }
          release_stage();
        }
        const bool last_of_sample = (ii + 1 == my) || ((j + G) / p.slices != sl_);
        if (!last_of_sample) continue;
        // fold: row lanes -> channel totals -> group totals (fixed order)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float* dst = red + (r0 * p.C + v * 8 + 2 * e) * 2;
          *reinterpret_cast<float4*>(dst) = make_float4(sm_[e].x, sq_[e].x, sm_[e].y, sq_[e].y);  // [channel][sum, sumsq]
          sm_[e] = sq_[e] = make_float2(0.f, 0.f);
        }
        consumer_sync();
        for (int c = t; c < p.C; c += T) {
          float ss = 0.f, qq = 0.f;
          for (int kk = 0; kk < p.rp; ++kk) {
            ss += red[(kk * p.C + c) * 2];
            qq += red[(kk * p.C + c) * 2 + 1];
          }
          red[c * 2] = ss;  // row-lane 0 now holds the channel totals (each thread only overwrites what it alone read at kk = 0)
          red[c * 2 + 1] = qq;
        }
        consumer_sync();
        if (t < p.groups) {
          float ss = 0.f, qq = 0.f;
          for (int c = t * p.cpg; c < (t + 1) * p.cpg; ++c) {
            ss += red[c * 2];
            qq += red[c * 2 + 1];
          }
          // first item of this CTA inside the sample: the smallest j' >= sl_ * slices with j' = blockIdx.x (mod G)
          const int base = sl_ * p.slices;
          const int first = base + ((static_cast<int>(blockIdx.x) - base) % G + G) % G;
          const int slot = first - base;
          float2* dst = reinterpret_cast<float2*>(p.partial) + (static_cast<long long>(s) * p.slots + slot) * p.groups + t;
          __stcg(dst, make_float2(ss, qq));
        }
        consumer_sync();  // `red` is reused
      }
    }

    // ------------------------------------------------------------------ grid barrier: every partial of the chunk is written
    ++barrier_no;
    consumer_sync();
    if (t == 0) {
      __threadfence();
      atomicAdd(&g_gn_sync[0], 1u);
      const unsigned int target = barrier_no * static_cast<unsigned int>(G);
      const long long t0 = clock64();
      while (ld_acquire_gpu(&g_gn_sync[0]) < target) {
        __nanosleep(64);
        if (clock64() - t0 > AV2V_WAIT_TIMEOUT_CYCLES) {
          printf("av2v: groupnorm grid barrier timeout (block %d, barrier %u)\n", blockIdx.x, barrier_no);
          __trap();
        }
      }
      __threadfence();
    }
    consumer_sync();

    // ------------------------------------------------------------------ phase B: normalise (+SiLU), items descending
    float* stat = red + static_cast<size_t>(p.rp) * p.C * 2;  // [groups][2] = mean, rstd of the current sample
    int cur_sample = -1;
    float2 a[4], b[4];
    int soff[U], doff[U];  // vector offsets inside a stage (source block pitch) / inside the output rows (full pitch)
#pragma unroll
    for (int u = 0; u < U; ++u) {
      soff[u] = (r0 + u * p.rp) * spitch;
      doff[u] = (r0 + u * p.rp) * p.vpr;
    }
    for (int ii = my - 1; ii >= 0; --ii) {
      const int j = static_cast<int>(blockIdx.x) + ii * G;
      const int s = s0 + j / p.slices, slice = j % p.slices;
      int rbeg, rend;
      item_rows(slice, rbeg, rend);
      if (s != cur_sample) {
        cur_sample = s;
        consumer_sync();  // everyone is done with the previous sample's `stat`
        // fold the sample's partials [slot][group]: thread = (group g, slot subset q); consecutive threads read consecutive
        // float2 (coalesced), eight independent loads in flight per thread; subsets summed per group in a fixed order, in double
        {
          double* dred = reinterpret_cast<double*>(red);  // [subsets][groups][2]
          const int subsets = T / p.groups;                // T is a multiple of 32 >= groups (groups <= 64 divides T for 32 / 64)
          const int g = t % p.groups, q = t / p.groups;
          const float2* src = reinterpret_cast<const float2*>(p.partial) + static_cast<long long>(s) * p.slots * p.groups + g;
          const __half pivot = t < p.groups ? gn_pivot(p, s, t) : __float2half(0.f);  // in flight with the partial loads
          double ss = 0.0, qq = 0.0;
          if (q < subsets) {
            for (int sl = q; sl < p.slots; sl += 8 * subsets) {
              float2 v8[8];
#pragma unroll
              for (int u = 0; u < 8; ++u) {
                const int idx = sl + u * subsets;
                v8[u] = idx < p.slots ? __ldcg(src + static_cast<long long>(idx) * p.groups) : make_float2(0.f, 0.f);
              }
#pragma unroll
              for (int u = 0; u < 8; ++u) {
                ss += static_cast<double>(v8[u].x);
                qq += static_cast<double>(v8[u].y);
              }
            }
            dred[(q * p.groups + g) * 2] = ss;
            dred[(q * p.groups + g) * 2 + 1] = qq;
          }
          consumer_sync();
          if (t < p.groups) {
            ss = 0.0;
            qq = 0.0;
            for (int k2 = 0; k2 < subsets; ++k2) {
              ss += dred[(k2 * p.groups + t) * 2];
              qq += dred[(k2 * p.groups + t) * 2 + 1];
            }
            const double cnt = static_cast<double>(p.rows) * p.cpg;
            const double d1 = ss / cnt;  // mean of x - k
            const double mean = static_cast<double>(__half2float(pivot)) + d1;
            double var = qq / cnt - d1 * d1;
            if (var < 0.0) var = 0.0;
            stat[2 * t] = static_cast<float>(mean);
            stat[2 * t + 1] = static_cast<float>(1.0 / sqrt(var + static_cast<double>(p.eps)));
          }
        }
        consumer_sync();
        const uint4 gv = __ldg(reinterpret_cast<const uint4*>(p.gamma) + v);
        const uint4 bv = __ldg(reinterpret_cast<const uint4*>(p.beta) + v);
        const __half* gh = reinterpret_cast<const __half*>(&gv);
        const __half* bh = reinterpret_cast<const __half*>(&bv);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const int g = (v * 8 + e) / p.cpg;
          const float mean = stat[2 * g], rstd = stat[2 * g + 1];
          const float ae = rstd * __half2float(gh[e]);
          const float be = __half2float(bh[e]) - mean * ae;
          if (e & 1) {
            a[e >> 1].y = ae;
            b[e >> 1].y = be;
          } else {
            a[e >> 1].x = ae;
            b[e >> 1].x = be;
          }
        }
      }
      // this thread's output vectors of the current stage; advances by one stage of rows per iteration
      uint4* dst = reinterpret_cast<uint4*>(p.y) + (static_cast<long long>(s) * p.rows + rbeg) * p.vpr + v;
      for (int r = rbeg; r < rend; r += p.stage_rows, dst += static_cast<long long>(p.stage_rows) * p.vpr) {
        const int nr = min(p.stage_rows, rend - r);
        mbar_wait_hot(&full[stage], phase);
        const uint4* sb = reinterpret_cast<const uint4*>(stage_buf + stage * kStageBytes + sbase);
        // all U vectors of the thread go through each step of the dependent chain together (U x 8 independent chains), in packed
        // fp32x2 arithmetic (two elements per issue slot; the same IEEE fma / mul / add per lane)
        uint4 xv[U];
        float2 f[U][4], w[U][4];
#pragma unroll
        for (int u = 0; u < U; ++u) xv[u] = sb[(r0 + u * p.rp < nr) ? soff[u] : 0];  // out-of-range lanes recompute row 0, store nothing
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const __half2* xh = reinterpret_cast<const __half2*>(&xv[u]);
#pragma unroll
          for (int e = 0; e < 4; ++e) f[u][e] = ffma2(__half22float2(xh[e]), a[e], b[e]);
        }
        if (p.silu) {
          // the reference rounds the GroupNorm output to fp16 before SiLU (two separate ops); silu(g) = g / (1 + 2^(-g log2 e))
          const float2 nl2e = make_float2(-1.4426950408889634f, -1.4426950408889634f), one = make_float2(1.0f, 1.0f);
#pragma unroll
          for (int u = 0; u < U; ++u)
#pragma unroll
            for (int e = 0; e < 4; ++e) f[u][e] = __half22float2(__floats2half2_rn(f[u][e].x, f[u][e].y));
#pragma unroll
          for (int u = 0; u < U; ++u)
#pragma unroll
            for (int e = 0; e < 4; ++e) w[u][e] = fmul2(f[u][e], nl2e);
#pragma unroll
          for (int u = 0; u < U; ++u)
#pragma unroll
            for (int e = 0; e < 4; ++e) w[u][e] = fadd2(make_float2(ex2_approx(w[u][e].x), ex2_approx(w[u][e].y)), one);
#pragma unroll
          for (int u = 0; u < U; ++u)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(w[u][e].x) : "f"(w[u][e].x));
              asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(w[u][e].y) : "f"(w[u][e].y));
            }
#pragma unroll
          for (int u = 0; u < U; ++u)
#pragma unroll
            for (int e = 0; e < 4; ++e) f[u][e] = fmul2(f[u][e], w[u][e]);
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          if (r0 + u * p.rp < nr) {
            uint4 ov;
            ov.x = pack_half2(f[u][0].x, f[u][0].y);
            ov.y = pack_half2(f[u][1].x, f[u][1].y);
            ov.z = pack_half2(f[u][2].x, f[u][2].y);
            ov.w = pack_half2(f[u][3].x, f[u][3].y);
            dst[doff[u]] = ov;
          }
        }
        release_stage();
      }
    }
  }

  // last CTA out resets the barrier state for the next launch
  consumer_sync();
  if (t == 0) {
    __threadfence();
    const unsigned int old = atomicAdd(&g_gn_sync[1], 1u);
    if (old == static_cast<unsigned int>(G) - 1u) {
      g_gn_sync[0] = 0u;
      g_gn_sync[1] = 0u;
      __threadfence();
    }
  }
}

int gcd_int(int a, int b) { return b == 0 ? a : gcd_int(b, a % b); }

}  // namespace
}  // namespace av2v

using namespace av2v;

extern "C" int av2v_groupnorm_workspace_floats(int n_samples, int C) {
  (void)C;  // partial sums are kept per (sample, slice, group): independent of the channel count
  return n_samples * kGnMaxSlices * kGnMaxGroups * 2;
}

// partition_samples > 0: cut the samples into chunks and slices as for a call of that many samples (the per-sample statistics
// depend only on the slices, so they are then those of that call)
static int groupnorm_launch(const av2v_groupnorm_args* a, int partition_samples, cudaStream_t stream) {
  AV2V_REQUIRE(a != nullptr, AV2V_EINVAL, "groupnorm: null args");
  AV2V_REQUIRE(a->x && a->y && a->gamma && a->beta && a->workspace, AV2V_EINVAL, "groupnorm: null pointer");
  AV2V_REQUIRE(a->n_samples > 0 && a->rows > 0 && a->C > 0 && a->groups > 0, AV2V_EINVAL, "groupnorm: bad shape");
  AV2V_REQUIRE(a->C % a->groups == 0, AV2V_EINVAL, "groupnorm: C %% groups != 0");
  AV2V_REQUIRE(a->C % 8 == 0 && a->C <= 8192, AV2V_ENOSUP, "groupnorm: C must be a multiple of 8 and <= 8192");
  AV2V_REQUIRE(a->groups <= kGnMaxGroups, AV2V_ENOSUP, "groupnorm: at most 64 groups");
  AV2V_REQUIRE(aligned16(a->x) && aligned16(a->y) && aligned16(a->gamma) && aligned16(a->beta), AV2V_EALIGN,
               "groupnorm: pointers must be 16-byte aligned");

  GnParams p{};
  p.x = static_cast<const __half*>(a->x);
  p.x2 = static_cast<const __half*>(a->x2);
  p.C1 = a->x2 ? a->C1 : a->C;
  AV2V_REQUIRE(!a->x2 || (a->C1 > 0 && a->C1 < a->C && a->C1 % 8 == 0 && aligned16(a->x2)), AV2V_EINVAL,
               "groupnorm: two-source input needs 0 < C1 < C, C1 %% 8 == 0 and a 16-byte aligned x2");
  p.y = static_cast<__half*>(a->y);
  p.gamma = static_cast<const __half*>(a->gamma);
  p.beta = static_cast<const __half*>(a->beta);
  p.partial = a->workspace;
  p.n = a->n_samples;
  p.rows = a->rows;
  p.C = a->C;
  p.groups = a->groups;
  p.cpg = a->C / a->groups;
  p.vpr = a->C / 8;
  p.vpr1 = p.C1 / 8;
  p.eps = a->eps;
  p.silu = a->silu;
  // consumer threads T = vpr * rp: a multiple of 32, as many as fit 640 (U = 3 build) — or 480 with U = 4 when 640 is not reachable
  // but 480 is (C = 960, 1920: 120 / 240 vectors per row)
  const int rp0 = 32 / gcd_int(p.vpr, 32);
  const int unit = p.vpr * rp0;
  AV2V_REQUIRE(unit <= 640, AV2V_ENOSUP, "groupnorm: C = %d needs %d threads per row-lane set (max 640)", a->C, unit);
  const int t640 = (640 / unit) * unit, t480 = (480 / unit) * unit;
  const bool use4 = t480 * 4 > t640 * 3;  // more bytes per stage with the U = 4 build
  const int T = use4 ? t480 : t640;
  const int U = use4 ? 4 : 3;
  const int rp = T / p.vpr;
  p.rp = rp;
  const long long row_bytes = static_cast<long long>(a->C) * 2;
  p.stage_rows = rp * U;
  AV2V_REQUIRE(static_cast<long long>(p.stage_rows) * row_bytes <= kStageBytes, AV2V_ENOSUP, "groupnorm: stage overflow (C = %d)", a->C);

  // chunks of whole samples with at most kChunkBytes of x
  const long long sample_bytes = static_cast<long long>(a->rows) * row_bytes;
  long long cs = kChunkBytes / sample_bytes;
  if (cs < 1) cs = 1;
  const int np = partition_samples > 0 ? partition_samples : a->n_samples;
  if (cs > np) cs = np;
  // spread the samples evenly over the chunks (48 frames of 2.6 MB: 3 x 16, not 18 + 18 + 12)
  const int n_chunks = static_cast<int>((np + cs - 1) / cs);
  p.chunk_samples = (np + n_chunks - 1) / n_chunks;
  p.n_chunks = (a->n_samples + p.chunk_samples - 1) / p.chunk_samples;

  // slices per sample: the chunk's items (chunk_samples x slices) should fill whole rounds of the grid (one CTA per SM) — 48
  // frames go 7 at a time, and 7 x 37 slices = 259 ~ 2 x 132 items — with at least two pipeline stages per slice when the
  // sample is that long.  Score = fill of the last round, minus a little per extra round (per-item fold / barrier overhead).
  const int sms = sm_count_cached();
  int max_s = a->rows / (2 * p.stage_rows);
  if (max_s < 1) max_s = (a->rows + p.stage_rows - 1) / p.stage_rows >= 1 ? 1 : 1;
  if (max_s > kGnMaxSlices) max_s = kGnMaxSlices;
  int slices = 1;
  double best = -1.0;
  for (int cand = 1; cand <= max_s; ++cand) {
    const long long it = static_cast<long long>(p.chunk_samples) * cand;
    const long long rounds = (it + sms - 1) / sms;
    if (rounds > 6) break;
    const double fill = static_cast<double>(it) / static_cast<double>(rounds * sms);
    const double score = fill - 0.015 * static_cast<double>(rounds);
    if (score > best + 1e-9) {
      best = score;
      slices = cand;
    }
  }
  p.rows_per_slice = (a->rows + slices - 1) / slices;
  p.slices = (a->rows + p.rows_per_slice - 1) / p.rows_per_slice;  // no empty slices

  const long long items = static_cast<long long>(p.chunk_samples) * p.slices;
  const int grid = static_cast<int>(items < sms ? items : sms);  // <= one CTA per SM: all CTAs are co-resident (grid barrier)
  p.slots = p.slices < grid ? p.slices : grid;
  const size_t smem = static_cast<size_t>(kStages) * kStageBytes + (static_cast<size_t>(rp) * a->C * 2 + 2 * kGnMaxGroups) * sizeof(float) +
                      2 * kStages * sizeof(uint64_t) + 128;
  AV2V_REQUIRE(smem <= 227 * 1024, AV2V_ENOSUP, "groupnorm: shared memory budget exceeded (%zu B)", smem);
  static bool attr_set = false;
  if (!attr_set) {
    AV2V_CHECK_CUDA(cudaFuncSetAttribute(gn_persistent_kernel<3, 640>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    AV2V_CHECK_CUDA(cudaFuncSetAttribute(gn_persistent_kernel<4, 480>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  if (use4) gn_persistent_kernel<4, 480><<<grid, T + 32, smem, stream>>>(p);
  else gn_persistent_kernel<3, 640><<<grid, T + 32, smem, stream>>>(p);
  AV2V_CHECK_CUDA(cudaGetLastError());
  return AV2V_OK;
}

extern "C" int av2v_groupnorm_silu_f16(const av2v_groupnorm_args* a, av2v_stream_t stream) {
  return groupnorm_launch(a, 0, static_cast<cudaStream_t>(stream));
}

extern "C" int av2v_groupnorm_silu_part_f16(const av2v_groupnorm_args* a, int32_t partition_samples,
                                            av2v_stream_t stream) {
  AV2V_REQUIRE(a != nullptr && partition_samples >= a->n_samples, AV2V_EINVAL,
               "groupnorm: partition_samples must be at least n_samples");
  return groupnorm_launch(a, partition_samples, static_cast<cudaStream_t>(stream));
}
