"""CPU models of the synchronisation and index bookkeeping of the sm_90a kernels (csrc/gemm_wgmma.cu, csrc/gemm_ws.cu,
csrc/gemm_common.cuh, csrc/attention_wgmma.cu, csrc/ring.cuh).

A data race or a wrong index in these kernels shows up on the GPU only as occasionally wrong numbers, so the schedules are
restated here as discrete-event models with randomised latencies and checked for their hazards, each with a negative control
(the same model with one rule broken must be caught).  The pipeline constants are read from the kernel sources, so a change
there that breaks a rule fails here.
"""
from __future__ import annotations

import os
import random
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "anyv2v_b200", "csrc")


def _src(name):
    return open(os.path.join(CSRC, name)).read()


def gemm_pipeline_constants():
    """(stages, wait_group depth, prefetch distance) of the GEMM's cp.async ring, as written in gemm_wgmma.cu"""
    s = _src("gemm_wgmma.cu")
    stages = int(re.search(r"constexpr int kStages = (\d+);", s).group(1))
    wait = eval(re.search(r"cp_async_wait<(kStages - \d+)>\(\);\n\s*fence_proxy_async_smem", s).group(1), {"kStages": stages})
    dist = eval(re.search(r"const int pf = kb \+ (kStages - \d+);", s).group(1), {"kStages": stages})
    return stages, wait, dist


# ---------------------------------------------------------------------------------------------------------- GEMM ring
def simulate_gemm_ring(rng: random.Random, nk: int, stages: int, wait_depth: int, dist: int, n_wg: int = 2,
                       epilogue_tile: bool = False, tile_shift: int = 0):
    """gemm_wgmma_kernel's K loop.  Per K block kb, every thread: cp.async.wait_group(wait_depth) -> fence -> __syncthreads ->
    issue the loads of block kb + dist into slot (kb + dist) % stages, commit -> wgmma kb on slot kb % stages, commit ->
    wgmma.wait_group(1) (wgmma kb - 1 retired).  Asserts: a block is landed before any wgmma reads it, and a slot is
    overwritten only after every warpgroup retired the wgmma that read it.  epilogue_tile: after its last wgmma issue a warp
    starts filling the epilogue's staging tile (cp.async of the residual, or its stores) in slot (nk + tile_shift) % stages
    without a block barrier: whatever block last held that slot must have been retired by every warpgroup."""
    land = {}
    groups = []  # one cp.async group per prologue stage / iteration, in commit order: the block it loads or None
    retire = [dict() for _ in range(n_wg)]
    t_wg = [0.0] * n_wg
    for s in range(dist):
        land[s] = rng.uniform(1, 50) if s < nk else 0.0
        groups.append(s if s < nk else None)
    for kb in range(nk):
        for w in range(n_wg):  # wait_group(wait_depth): all but the newest wait_depth groups have landed
            done = groups[:len(groups) - wait_depth] if wait_depth else groups
            t_wg[w] = max([t_wg[w]] + [land[g] for g in done if g is not None])
        T = max(t_wg)  # __syncthreads
        j = kb + dist
        if j < nk:
            prev = j - stages  # the block that last occupied slot j % stages
            if prev >= 0:
                for w in range(n_wg):
                    assert retire[w][prev] <= T, f"slot {j % stages} overwritten by block {j} while block {prev} is still read"
            land[j] = T + rng.uniform(1, 50)
            groups.append(j)
        else:
            groups.append(None)
        assert land[kb] <= T, f"wgmma reads block {kb} before its cp.async landed"
        for w in range(n_wg):
            issue = T + rng.uniform(0, 3)
            retire[w][kb] = issue + rng.uniform(1, 40)
            t_wg[w] = max(issue, retire[w].get(kb - 1, 0.0))  # wgmma.wait_group(1)
    if epilogue_tile:
        slot = (nk + tile_shift) % stages
        held = [b for b in range(nk) if b % stages == slot]
        for w in range(n_wg):
            for v in range(n_wg):
                assert not held or retire[v][held[-1]] <= t_wg[w], f"staging tile in slot {slot} while block {held[-1]} is still read"
    return True


# ---------------------------------------------------------------------------------------------------------- double buffer
def simulate_double_buffer(rng: random.Random, n: int, trailing_barrier: bool = True, n_wg: int = 2):
    """The K/V loop of attn_kernel: load 0; per step kt: issue the
    loads of kt + 1 into buffer (kt + 1) & 1, commit, wait_group(1) (wait_group(0) on the last step) -> fence ->
    __syncthreads -> every warpgroup computes on buffer kt & 1 -> __syncthreads.  Asserts the same two hazards as the GEMM
    ring; without the trailing barrier a fast warpgroup's prefetch overwrites the buffer a slow one still reads."""
    land = {0: rng.uniform(1, 50)}
    reads = {}  # step -> per-warpgroup end of compute
    t_wg = [0.0] * n_wg
    for kt in range(n):
        for w in range(n_wg):
            if kt + 1 < n:  # each thread issues its share of the next step's loads on arrival
                prev = kt - 1
                if prev >= 0:
                    for w2 in range(n_wg):
                        assert reads[prev][w2] <= t_wg[w], f"buffer {(kt + 1) & 1} overwritten while step {prev} reads it"
                land[kt + 1] = max(land.get(kt + 1, 0.0), t_wg[w] + rng.uniform(1, 50))
            t_wg[w] = max(t_wg[w], land[kt])  # wait_group(1): the group of step kt landed
        T = max(t_wg)  # __syncthreads
        assert land[kt] <= T
        reads[kt] = [T + rng.uniform(1, 60) for _ in range(n_wg)]
        t_wg = list(reads[kt])
        if trailing_barrier:
            t_wg = [max(t_wg)] * n_wg
    return True


def simulate_tile_handoff(rng: random.Random, barrier: bool = True, n_wg: int = 2):
    """tattn_fused_kernel between projection and attention: each warpgroup stores ITS 64 rows of the Q, K and V tiles
    (acc_to_tile), then fence + named barrier 1 (the two consumer warpgroups), then each warpgroup's attention reads key /
    value rows of BOTH halves (F = 128 sequences span them).  Asserts every row is written before it is read."""
    written = [rng.uniform(1, 80) for _ in range(n_wg)]  # end of each warpgroup's tile stores
    start = [w_end + rng.uniform(0, 5) for w_end in written]
    if barrier:
        start = [max(written)] * n_wg
    for w in range(n_wg):
        for owner in range(n_wg):
            assert written[owner] <= start[w], f"warpgroup {w} reads rows of warpgroup {owner} before they are stored"
    return True


# ---------------------------------------------------------------------------------------------------------- fused key tiles
def fused_key_tiles(F: int, wg: int, wrong: bool = False, old_rule: bool = False):
    """key tiles (64 slots each) the warpgroup wg visits in tattn_fused_kernel, as in the kernel: kt = wg when F divides 64 (no
    pixel crosses the 64-slot halves), else both.  old_rule: kt = wg for every F <= 64, right only when F divides 128"""
    if (F <= 64) if old_rule else (64 % F == 0):
        return [1 - wg if wrong else wg]
    return [0, 1]


def check_fused_key_tiles(F: int, wrong: bool = False, old_rule: bool = False):
    """every key of a query slot's own pixel (slot // F equal) lies in a visited tile, and the kept keys per row are exactly F;
    tail slots (slot >= floor(128 / F) * F, never stored) are not checked"""
    used = 128 // F * F
    for wg in range(2):
        tiles = fused_key_tiles(F, wg, wrong, old_rule)
        for r in range(64):
            q = wg * 64 + r
            if q >= used:
                continue
            kept = [64 * kt + c for kt in tiles for c in range(64) if q // F == (64 * kt + c) // F]
            assert len(kept) == F and all(k // F == q // F for k in kept), (F, wg, r, len(kept))
    return True


# ---------------------------------------------------------------------------------------------------------- frame slots
def frame_slot_rules():
    """checks that attention_wgmma.cu still launches and maps frames-mode work as frame_slot_items restates it"""
    s = _src("attention_wgmma.cu")
    for rule in ("p.ppt = 128 / F;", "p.pix_tiles = (HW + p.ppt - 1) / p.ppt;", "p.f_tiles = (F + 127) / 128;",
                 "n_kv = (p.F + 63) / 64;", "const int pix_end = min(pix0 + p.ppt, p.HW);", "return pix < pix_end ?",
                 "return f < p.F ?", "return u < p.F ?", "const int nk = p.seq_kv;", "p.n_kt = 64 % a->F == 0 ? 1 : 2;",
                 "const int kt = n_kt == 1 ? wg : it;", "pix0 = item % p.pix_tiles * p.ppt;",
                 "return pix < pix_end ? ((clip_row + i % F) * p.HW + pix) * p.ldo : -1;"):
        assert rule in s, f"attention_wgmma.cu no longer contains {rule!r}"
    return True


def frame_slot_items(kernel: str, F: int, HW: int, clips: int = 2, tail_masked: bool = True, old_rule: bool = False):
    """the work items of frames-mode attn_kernel ("attn") or tattn_fused_kernel ("fused", n_v = 1) for `clips` clips of F
    frames x HW pixels, as the host launches them and the kernel addresses them.  Yields (qrow, krow, keep): qrow[i] the token
    row query slot i loads and stores (-1: none), krow[u] the row key slot u loads (-1: zero-filled), keep[i, u] the score
    mask, with the key tiles a query's warpgroup does not visit masked out.  tail_masked=False: slots past floor(128 / F) * F
    take the next pixel, as when the tail is not masked; old_rule: the fused kernel's kt = wg for every F <= 64."""
    import numpy as np
    if kernel == "attn" and F > 128:  # unpacked: one pixel, ceil(F / 128) query tiles, ceil(F / 64) key tiles
        n_kv = (F + 63) // 64
        u = np.arange(n_kv * 64)
        keep_k = u < F
        for clip in range(clips):
            for pix in range(HW):
                for qt in range((F + 127) // 128):
                    f = qt * 128 + np.arange(128)
                    qrow = np.where(f < F, (clip * F + f) * HW + pix, -1)
                    krow = np.where(u < F, (clip * F + u) * HW + pix, -1)
                    yield qrow, krow, np.broadcast_to(keep_k, (128, n_kv * 64))
        return
    assert F <= 128
    ppt = 128 // F
    slot = np.arange(128)
    group = slot // F
    keep = group[:, None] == group[None, :]
    if kernel == "fused":
        n_kt = 1 if ((F <= 64) if old_rule else (64 % F == 0)) else 2
        for wg in range(2):
            visited = np.zeros(128, bool)
            for it in range(n_kt):
                kt = wg if n_kt == 1 else it
                visited[kt * 64:(kt + 1) * 64] = True
            keep[wg * 64:(wg + 1) * 64] &= visited[None, :]
    for clip in range(clips):
        for pt in range((HW + ppt - 1) // ppt):
            pix0 = pt * ppt
            pix_end = min(pix0 + ppt, HW) if tail_masked else HW
            pix = pix0 + group
            rows = np.where(pix < pix_end, (clip * F + slot % F) * HW + pix, -1)
            yield rows, rows, keep


def check_frame_slot_ownership(kernel: str, F: int, HW: int, clips: int = 2, **kw):
    """every (clip, pixel, frame) row is stored by exactly one work item, and every stored row keeps exactly the F key rows of
    its own (clip, pixel): none zero-filled, none of another pixel"""
    import numpy as np
    stored = np.zeros(clips * F * HW, np.int64)
    for qrow, krow, keep in frame_slot_items(kernel, F, HW, clips, **kw):
        q = np.nonzero(qrow >= 0)[0]
        np.add.at(stored, qrow[q], 1)
        valid = krow[krow >= 0]
        assert len(np.unique(valid)) == len(valid)
        k = keep[q]                                               # [stored rows, key slots]
        r = qrow[q][:, None]
        own = (krow[None, :] >= 0) & (krow[None, :] % HW == r % HW) & (krow[None, :] // HW // F == r // HW // F)
        bad = k & ~own                                            # a kept key that is zero-filled or of another pixel
        assert not bad.any(), f"{kernel} F={F} HW={HW}: row {int(r[bad.any(1)][0, 0])} keeps a key outside its pixel"
        n = k.sum(1)
        assert (n == F).all(), f"{kernel} F={F} HW={HW}: row {int(r[n != F][0, 0])} keeps {int(n[n != F][0])} keys, not {F}"
    assert (stored == 1).all(), (f"{kernel} F={F} HW={HW}: rows stored {int(stored.min())}..{int(stored.max())} times "
                                 f"(first bad row {int(np.nonzero(stored != 1)[0][0])})")
    return True


# ---------------------------------------------------------------------------------------------------------- GEMM epilogue
def acc_row(t, i):
    """ptx.cuh acc_row for warpgroup thread t: accumulator element i of wgmma m64nN"""
    return 16 * (t >> 5) + ((t & 31) >> 2) + 8 * ((i >> 1) & 1)


def acc_col(t, i):
    return 8 * (i >> 2) + 2 * (t & 3) + (i & 1)


def stage_offset(row, chunk, swizzle=True, bn=128, tail_swizzle=True):
    """gemm_common.cuh stage_offset<bn>: byte offset of 16-byte chunk `chunk` of row `row` in the epilogue's staging tile
    (256-byte rows; a 160-wide tile's chunks 16 .. 19 in a second part of 64-byte rows behind the first)"""
    if bn == 128 or chunk < 16:
        return row * 256 + ((chunk ^ (row & 7 if swizzle else 0)) << 4)
    return 128 * 256 + row * 64 + (((chunk - 16) ^ ((row >> 1) & 3 if tail_swizzle else 0)) << 4)


def copy_out_passes(bn=128, geglu=False):
    """copy_out_band's (and, for a tile's full width, fetch_residual_band's) passes over a band: (first chunk, log2 chunks
    per row, warp instructions).  Lane l of instruction i takes chunk first + idx % 2^lg of band row idx >> lg, idx = 32 i + l,
    if that row is < 16"""
    if geglu:
        return [(0, 3, 8)]
    return [(0, 4, 8)] + ([(16, 2, 2)] if bn == 160 else [])


def band_lanes(r0, bn=128, geglu=False):
    """per warp instruction of copy_out_band: [(lane, row, chunk)]"""
    for c0, lg, n in copy_out_passes(bn, geglu):
        for i in range(n):
            yield [(lane, r0 + ((32 * i + lane) >> lg), c0 + ((32 * i + lane) & ((1 << lg) - 1))) for lane in range(32)
                   if ((32 * i + lane) >> lg) < 16], c0, lg


def epilogue_bands(kernel: str):
    """warp -> first tile rows of the bands it owns in one staging tile: the rows its accumulators hold (acc_row).
    conv (gemm_wgmma_kernel): 8 warps, warpgroup wg's one accumulator holds tile rows 64 wg .. 64 wg + 63.
    linear (gemm_ws_kernel, LINEAR and conv alike): a consumer warpgroup's own tile, 4 warps, accumulator b holds tile rows 64 b .. 64 b + 63."""
    if kernel == "conv":
        return {w: [64 * (w // 4) + acc_row(32 * (w % 4), 0)] for w in range(8)}
    assert kernel == "linear", kernel
    return {w: [64 * b + acc_row(32 * w, 0) for b in range(2)] for w in range(4)}


def check_epilogue_staging(kernel: str, geglu: bool = False, swizzle: bool = True, bn: int = 128, tail_swizzle: bool = True):
    """The staging tile of the GEMM epilogue (gemm_common.cuh), per warp and band (epilogue_bands: a band is the 16 rows a
    warp holds in one accumulator; conv: 8 warps x 1 band, linear: 4 warps x 2 bands, GEGLU in linear only; bn = 160:
    gemm_ws_kernel's 160-wide tiles, linear only).  (1) Fragment-order 4-byte writes (and the residual reads at the same
    addresses): one instruction is 8 rows x 4 lanes; its 32 lanes hit 32 different banks, and over all instructions every
    (row, column pair) of the tile is written exactly once.  (2) Copy-out 16-byte reads (copy_out_passes: lane -> chunk of
    the band's rows in row-major order, per part of the tile): each quarter warp (one shared-memory wavefront of a 128-bit
    access) covers the 8 bank groups once, the lanes of a row read consecutive chunks (whole 128-byte lines of the output
    row, or a 160-wide tile's 64-byte tail), and every chunk is read exactly once BY THE WARP THAT WROTE IT — the kernels
    order the two with __syncwarp only.  (3) The residual cp.async pattern (2 rows x 16 chunks per instruction; the tail: the
    copy-out's) fetches every chunk once, again in the warp that consumes it.  swizzle=False / tail_swizzle=False are the
    negative controls."""
    assert not (geglu and kernel == "conv"), "GEGLU runs on gemm_ws_kernel<false> only"
    assert bn == 128 or (kernel == "linear" and not geglu), "160-wide tiles are gemm_ws_kernel's, without GEGLU"
    src = _src("gemm_common.cuh")
    assert "if (kBN == 128 || chunk < 16) return static_cast<uint32_t>(row * 256 + ((chunk ^ (row & 7)) << 4));" in src, \
        "stage_offset changed: update the model"
    assert "return static_cast<uint32_t>(128 * 256 + row * 64 + (((chunk - 16) ^ ((row >> 1) & 3)) << 4));" in src, \
        "stage_offset changed: update the model"
    for rule in ("const int r = r0 + 8 * i + (lane >> 2);", "const int ct = 16 + (lane & 3)", "for (int i = 0; i < 2; ++i) {"):
        assert src.count(rule) == 2, f"the tail passes of fetch_residual_band / copy_out_band changed ({rule!r}): update the model"
    for f, rule in (("gemm_wgmma.cu", "const int r0 = 16 * (threadIdx.x >> 5);"),
                    ("gemm_ws.cu", "const int r0 = 16 * ((threadIdx.x >> 5) & 3);"),
                    ("gemm_ws.cu", "fetch_residual_band<false, kBN>(p, 0, m0, n0, r0 + 64 * b, staging);"),
                    ("gemm_ws.cu", "copy_out_band<false, kBN>(p, 0, m0, n0, r0 + 64 * b, staging);")):
        assert rule in _src(f), f"{f} no longer contains {rule!r}: update the model"

    def so(r, c):
        return stage_offset(r, c, swizzle, bn, tail_swizzle)

    bands = epilogue_bands(kernel)
    cpr = 8 if geglu else bn // 8  # chunks per tile row: the GEGLU output tile is 128 x 64
    tile_bytes = 128 * 2 * bn
    writer = {}  # byte address of a 4-byte word -> warp
    for warp, rows in bands.items():
        chunks = [4 * g + jj for g in range(2) for jj in range(4)] if geglu else list(range(cpr))
        for r0 in rows:
            for chunk in chunks:
                for h in range(2):
                    addrs = [so(r0 + acc_row(lane, 2 * h), chunk) + 4 * (lane & 3) for lane in range(32)]
                    assert len({(a // 4) % 32 for a in addrs}) == 32, f"fragment store of chunk {chunk}: bank conflict"
                    for a in addrs:
                        assert 0 <= a < tile_bytes and a not in writer, "staging word written twice"
                        writer[a] = warp
    want = {so(r, c) + 4 * q for r in range(128) for c in range(cpr) for q in range(4)}
    assert set(writer) == want, "the fragment stores do not cover the tile"
    read = set()
    for warp, rows in bands.items():
        for r0 in rows:
            for lanes, c0, lg in band_lanes(r0, bn, geglu):
                for q in range(0, len(lanes), 8):
                    groups = {(so(r, c) // 16) % 8 for _, r, c in lanes[q:q + 8]}
                    assert len(groups) == 8, "copy-out read: bank conflict inside a quarter warp"
                for (l0, ra, ca), (l1, rb, cb) in zip(lanes, lanes[1:]):
                    assert (rb, cb) == ((ra, ca + 1) if ca + 1 < c0 + (1 << lg) else (ra + 1, c0)), \
                        "copy-out lanes are not consecutive chunks"
                for _, r, c in lanes:
                    a = so(r, c)
                    assert a not in read and all(writer[a + 4 * q] == warp for q in range(4)), "chunk read twice or by another warp"
                    read.add(a)
    assert len(read) == 128 * cpr
    if not geglu:
        fetched = {}
        for warp, rows in bands.items():
            for r0 in rows:
                lanes = [(r0 + 2 * i + (lane >> 4), lane & 15) for i in range(8) for lane in range(32)]
                if bn == 160:
                    lanes += [(r, c) for ls, c0, _ in band_lanes(r0, bn) if c0 == 16 for _, r, c in ls]
                for r, c in lanes:
                    a = so(r, c)
                    assert a not in fetched and writer[a] == warp, "residual chunk fetched twice or by another warp"
                    fetched[a] = warp
        assert len(fetched) == 128 * cpr
    return True


def check_ragged_copy_out(M: int, N: int, m0: int, n0: int, bn: int = 128, passes=None):
    """The output chunks the copy-out of one tile (m0, n0) stores, over every band of both kernels' band ownership alike
    (gemm_ws_kernel: 4 warps x 2 bands): every 16-byte chunk of the tile's rows < M and columns < N exactly once, nothing
    past them.  passes: copy_out_passes(bn) unless given (negative control: drop the tail pass)"""
    passes = copy_out_passes(bn) if passes is None else passes
    stored = {}
    for rows in epilogue_bands("linear").values():
        for r0 in rows:
            for c0, lg, n in passes:
                for i in range(n):
                    for lane in range(32):
                        idx = 32 * i + lane
                        r, c = r0 + (idx >> lg), c0 + (idx & ((1 << lg) - 1))
                        if (idx >> lg) < 16 and m0 + r < M and n0 + 8 * c < N:
                            stored[(m0 + r, n0 + 8 * c)] = stored.get((m0 + r, n0 + 8 * c), 0) + 1
    want = {(m, c) for m in range(m0, min(m0 + 128, M)) for c in range(n0, min(n0 + bn, N), 8)}
    assert set(stored) == want, f"copy-out of tile ({m0}, {n0}) misses or adds chunks"
    assert all(v == 1 for v in stored.values()), "an output chunk is stored twice"
    return True


def check_epilogue(geglu_pack, N_geglu=(128, 256, 2560)):
    """The GEMM epilogues' index arithmetic: (1) the accumulator layout maps the 128 threads x 64 registers of a warpgroup
    one-to-one onto its 64 x 128 block; (2) GEGLU (gemm_ws_kernel<false>): the (h, gate) columns the kernel pairs (jh,
    jg = jh + 4 inside each 64-column group; staged at chunk 4 g + jj, element cq of the tile row, i.e. output column
    n0 / 2 + 32 g + 8 jj + cq) are the pairs geglu_pack interleaved, every output column written once; (3) out_row_offset
    of an up2 phase (gemm_wgmma_kernel) maps the low-resolution pixels one-to-one onto the phase's pixels of the output;
    (4) the staging tile of each kernel's band ownership (check_epilogue_staging)."""
    import torch
    seen = {(acc_row(t, i), acc_col(t, i)) for t in range(128) for i in range(64)}
    assert len(seen) == 64 * 128 and all(0 <= r < 64 and 0 <= c < 128 for r, c in seen)
    for N in N_geglu:
        inner = N // 2
        w = torch.arange(N, dtype=torch.float64)[:, None]  # row n of W holds the value n: the packed order is visible
        wp, _ = geglu_pack(w, torch.zeros(N, dtype=torch.float64))
        packed = wp[:, 0].long().tolist()
        out_cols = {}
        for n0 in range(0, N, 128):
            for t in range(128):
                cq = 2 * (t & 3)
                for g in range(2):
                    for jj in range(4):
                        jh, jg = 8 * g + jj, 8 * g + jj + 4
                        ch, cg = n0 + 8 * jh + cq, n0 + 8 * jg + cq
                        if ch >= N:
                            continue
                        oc = n0 // 2 + 32 * g + 8 * jj + cq
                        for e in range(2):
                            h_src, g_src = packed[ch + e], packed[cg + e]
                            assert h_src < inner and g_src == h_src + inner, (N, ch, cg)
                            assert out_cols.setdefault(oc + e, h_src) == h_src
                            assert oc + e == h_src, (N, oc + e, h_src)  # output column j = h_j * gelu(gate_j)
        assert sorted(out_cols) == list(range(inner))
    for NF, H, W in ((2, 3, 5), (1, 8, 8), (3, 4, 16)):
        for ph in range(4):
            py, px = ph >> 1, ph & 1
            rows = set()
            for m in range(NF * H * W):
                j, t = m % W, m // W
                i, n = t % H, t // H
                rows.add((n * 2 * H + 2 * i + py) * (2 * W) + 2 * j + px)
            want = {(n * 2 * H + y) * (2 * W) + x for n in range(NF) for y in range(py, 2 * H, 2) for x in range(px, 2 * W, 2)}
            assert rows == want
    for kernel, geglu in (("conv", False), ("linear", False), ("linear", True)):
        check_epilogue_staging(kernel, geglu)
    check_epilogue_staging("linear", bn=160)
    return True


# ---------------------------------------------------------------------------------------------------------- stage ring
def kernel_body(name, kernel):
    """the source text of __global__ `kernel` in csrc/`name`, from its name to its closing brace"""
    s = _src(name)
    i = s.index(f" {kernel}(const __grid_constant__")
    return s[i:s.index("\n}\n", i)]


def ring_constants():
    """StageRing's rules as ring.cuh writes them, each a function of (g, S): the stage of block g, the full parity its consumer
    waits on, whether producing it waits on empty (refill) and on which parity; also checks the arrival counts RingModel
    assumes (full: 1, empty: one per consumer warp, released by lane 0 after __syncwarp)"""
    s = _src("ring.cuh")
    for rule in ("mbar_init(&full[s], 1);", "mbar_init(&empty[s], consumer_warps);",
                 "__syncwarp();\n    if ((threadIdx.x & 31) == 0) mbar_arrive(&empty[stage(g)]);"):
        assert rule in s, f"ring.cuh no longer contains {rule!r}: update the model"

    def rule(pattern):
        return eval("lambda g, S: " + re.search(pattern, s).group(1).replace("/", "//"))  # C division of g >= 0
    return dict(stage=rule(r"int stage\(int g\) \{ return (.+?); \}"),
                full=rule(r"mbar_wait<false>\(&full\[stage\(g\)\], (.+?)\);"),
                refill=rule(r"if \((.+?)\) mbar_wait<false>\(&empty"),
                empty=rule(r"mbar_wait<false>\(&empty\[stage\(g\)\], (.+?)\);"))


class _MBar:
    """an mbarrier as the list of its phase-completion times; a parity wait succeeds once the number of completed phases has
    the other parity (mbarrier.try_wait.parity P: the phase of parity P has completed)"""
    def __init__(self, count):
        self.count, self.pending, self.done = count, [], []

    def arrive(self, t, n=1):
        self.pending += [t] * n
        if len(self.pending) >= self.count:
            self.done.append(max(self.pending[:self.count]))
            self.pending = self.pending[self.count:]

    def wait(self, parity, t):
        for c in [t] + sorted(x for x in self.done if x > t):
            if sum(1 for x in self.done if x <= c) & 1 != parity:
                return c
        raise AssertionError(f"wait on parity {parity} never succeeds (deadlock)")


class RingModel:
    """StageRing<stages> (ring.cuh) under randomised TMA latencies, with the rules ring_constants() reads.  The producer thread
    is replayed on demand and in block order (wait(g) first produces every block up to g); its times depend only on its own
    empty waits and issue, so it runs ahead as the kernel's does.  Each block is read and released by `readers` consumer
    warpgroups of arrivals / readers warps (2 in the attention kernels; 1 in the GEMM, where a tile belongs to one).
    Asserts: no block is read before it landed, no stage is refilled before every reader released the block it held.
    Faults (negative controls): wrong_parity="producer" / "consumer" flips that side's wait parity, release=False (one warp
    of warpgroup 1 never arrives on empty), overrun (the producer skips its empty wait)."""
    def __init__(self, rng, stages, arrivals, readers, wrong_parity="", release=True, overrun=False):
        self.rng, self.S, self.readers, self.warps = rng, stages, readers, arrivals // readers
        self.rules = ring_constants()
        self.full = [_MBar(1) for _ in range(stages)]
        self.empty = [_MBar(arrivals) for _ in range(stages)]
        self.flip = {side: int(wrong_parity == side) for side in ("producer", "consumer")}
        self.release_ok, self.overrun = release, overrun
        self.land, self.released = {}, {}  # block -> landing time; block -> release times of its readers
        self.t_prod = 0.0

    def _produce(self, g):
        r, S = self.rules, self.S
        s = r["stage"](g, S)
        if r["refill"](g, S):
            if not self.overrun:
                self.t_prod = self.empty[s].wait(r["empty"](g, S) ^ self.flip["producer"], self.t_prod)
            done = self.released.get(g - S, [])
            assert len(done) == self.readers and max(done) <= self.t_prod, \
                f"stage {s} refilled with block {g} while block {g - S} is read"
        self.t_prod += self.rng.uniform(0.1, 2)
        self.land[g] = self.t_prod + self.rng.uniform(5, 60)
        self.full[s].arrive(self.land[g])

    def wait(self, g, w, t):
        """warpgroup w, at time t, waits for block g; returns when it may read it"""
        while len(self.land) <= g:
            self._produce(len(self.land))
        t = self.full[self.rules["stage"](g, self.S)].wait(self.rules["full"](g, self.S) ^ self.flip["consumer"], t)
        assert self.land[g] <= t, f"warpgroup {w} reads block {g} before it landed"
        return t

    def release(self, g, w, t):
        """every warp of warpgroup w releases block g at time t"""
        short = not self.release_ok and w == 1
        self.empty[self.rules["stage"](g, self.S)].arrive(t, self.warps - short)
        if not short:
            self.released.setdefault(g, []).append(t)


# ---------------------------------------------------------------------------------------------------------- rows attention ring
def rows_ring_constants():
    """(stages, empty-barrier arrivals) of attn_rows_kernel's K / V ring, as written in attention_wgmma.cu; also checks the
    tile order and turn closing the model restates"""
    k = kernel_body("attention_wgmma.cu", "attn_rows_kernel")
    stages = int(re.search(r"constexpr int kRowsStages = (\d+);", _src("attention_wgmma.cu")).group(1))
    arrivals = int(re.search(r"ring\.init\((\d+)\);", k).group(1))
    for rule in ("constexpr int S = kRowsStages,", "for (int j = 0; j < n_kv; ++j) {", "ring.produce(j, ", "ring.wait(0);",
                 "ring.wait(j + 1);", "ring.release(j);", "ring.release(n_kv - 1);", "if (wg == 0) turn_hand_over(wg);"):
        assert rule in k, f"attn_rows_kernel no longer contains {rule!r}: update the model"
    return stages, arrivals


def simulate_rows_ring(rng: random.Random, n: int, stages: int, arrivals: int = 8, pingpong: bool = True, **faults):
    """attn_rows_kernel's consumers w = 0, 1 on the ring (RingModel, tile j = block j): turn 0 issues S(0); turn k = 1 .. n
    issues PV(k - 1) and S(k) (k < n, after waiting for tile k); turns alternate through the named barriers (w = 0 first);
    once the wgmma group retired the warpgroup releases tile k - 1 and runs the softmax of tile k.  Asserts, beside the
    ring's: the MMA turns alternate 0, 1, 0, 1, ...  Negative controls: RingModel's faults, pingpong=False."""
    ring = RingModel(rng, stages, arrivals, 2, **faults)
    turns = []
    t_wg = [rng.uniform(0, 5), rng.uniform(0, 5)]
    handed = [0.0, None]  # handed[w]: when the other warpgroup last handed the turn to w (w = 0 starts with it)
    for k in range(n + 1):
        for w in range(2):
            t = ring.wait(k, w, t_wg[w]) if k < n else t_wg[w]
            if pingpong:
                assert handed[w] is not None
                t = max(t, handed[w])
            turns.append((t, w))
            handed[1 - w] = t + rng.uniform(0.1, 1)
            retire = t + rng.uniform(5, 40)
            if k > 0:
                ring.release(k - 1, w, retire)
            t_wg[w] = retire + rng.uniform(1, 30)  # softmax of tile k
    order = [w for _, w in sorted(turns, key=lambda x: x[0])]
    assert order == [0, 1] * (n + 1), "MMA turns of the two consumers do not alternate"
    return True


# ---------------------------------------------------------------------------------------------------------- persistent LINEAR GEMM
def linear_ws_constants():
    """(stages, empty-barrier arrivals) of gemm_ws_kernel's ring, as written in gemm_ws.cu; also checks that the tile
    schedule, the block numbering and the turn taking are the ones the models below restate"""
    k = kernel_body("gemm_ws.cu", "gemm_ws_kernel")
    stages = int(re.search(r"constexpr int kStages = (\d+);", _src("gemm_ws.cu")).group(1))
    arrivals = int(re.search(r"ring\.init\((\d+)\);", k).group(1))
    for rule in ("StageRing<kStages> ring;", "for (int t = blockIdx.x; t < P.tiles; t += gridDim.x)",
                 "for (int kb = 0; kb < nk; ++kb, ++g) {", "ring.produce(g, kStage);",
                 "for (int i = wg, t = blockIdx.x + wg * gridDim.x; t < P.tiles; i += 2, t += 2 * gridDim.x)",
                 "const int g0 = i * nk;", "const int g = g0 + kb, s = ring.stage(g);", "ring.wait(g);",
                 "if (kb > 0) ring.release(g - 1);", "ring.release(g0 + nk - 1);", "turn_open(wg);",
                 "if (t + gridDim.x < P.tiles) turn_hand_over(wg);"):
        assert rule in k, f"gemm_ws_kernel no longer contains {rule!r}: update the model"
    assert "tiles < sm_count_cached() ? tiles : sm_count_cached()" in _src("gemm_ws.cu")
    return stages, arrivals


def ws_tile_n(M: int, N: int, geglu: bool = False, sms: int = 132):
    """gemm_ws.cu ws_tile_n: the column tile of gemm_ws_kernel (av2v_gemm_f16 counts n_tiles in it): 160 when N is a
    multiple of 160 and ceil(tiles / SMs) tile widths, the schedule's length, are no longer than at 128"""
    src = _src("gemm_ws.cu")
    for r in ("if (p.geglu || p.N % 160 != 0) return 128;",
              "const long long mt = (p.M + BM - 1) / BM, sms = sm_count_cached();",
              "const long long t128 = (mt * ((p.N + 127) / 128) + sms - 1) / sms * 128, t160 = (mt * (p.N / 160) + sms - 1) / sms * 160;",
              "return t160 <= t128 ? 160 : 128;"):
        assert r in src, f"ws_tile_n no longer contains {r!r}: update the model"
    for r in ("const int bn = ws ? ws_tile_n(p) : BN;", "p.n_tiles = (a->N + bn - 1) / bn;"):
        assert r in _src("gemm_wgmma.cu"), f"gemm_wgmma.cu no longer contains {r!r}: update the model"
    if geglu or N % 160:
        return 128
    mt = -(-M // 128)
    return 160 if -(-mt * N // 160 // sms) * 160 <= -(-mt * -(-N // 128) // sms) * 128 else 128


def ws_smem_bytes(bn: int):
    """gemm_ws_kernel's dynamic shared memory at column tile bn, as gemm_ws.cu sizes it: the ring's stages (A 128 x 64 and
    W bn x 64 fp16 boxes), one 128 x bn fp16 staging tile per consumer warpgroup and 1 KB to align the ring to 1024 bytes"""
    src = _src("gemm_ws.cu")
    for rule in ("constexpr int kTileBytes = BM * BK * 2;",
                 "template <int kBN> constexpr int kStageBytes = kTileBytes + kBN * BK * 2;",
                 "template <int kBN> constexpr int kStagingBytes = BM * kBN * 2;",
                 "template <int kBN> constexpr int kSmemBytes = kStages * kStageBytes<kBN> + 2 * kStagingBytes<kBN> + 1024;"):
        assert rule in src, f"gemm_ws.cu no longer contains {rule!r}: update the model"
    stages = int(re.search(r"constexpr int kStages = (\d+);", src).group(1))
    stage = 128 * 64 * 2 + bn * 64 * 2
    assert stage % 1024 == 0, "a stage must keep the next one on the 1024-byte sw128 alignment"
    return stages * stage + 2 * 128 * bn * 2 + 1024


def linear_ws_schedule(tiles: int, sms: int, off_by_one: bool = False):
    """the persistent schedule as the kernel walks it: grid = min(tiles, sms) CTAs; per CTA the producer's tile list and
    each consumer warpgroup's (local index i, tile) list.  Asserts both sides agree, every tile is computed exactly once,
    and no CTA is idle.  off_by_one: the loops run to t <= tiles (negative control)."""
    grid = min(tiles, sms)
    end = tiles + 1 if off_by_one else tiles
    done = [0] * (tiles + 1)
    for b in range(grid):
        prod = list(range(b, end, grid))
        cons = {wg: list(zip(range(wg, 10 ** 9, 2), range(b + wg * grid, end, 2 * grid))) for wg in (0, 1)}
        assert prod, f"CTA {b} has no tile"
        merged = sorted(cons[0] + cons[1])
        assert [i for i, _ in merged] == list(range(len(prod))) and [t for _, t in merged] == prod, "consumers and producer disagree"
        for t in prod:
            assert t < tiles, f"CTA {b} computes tile {t} past the last ({tiles - 1})"
            done[t] += 1
    assert all(n == 1 for n in done[:tiles]), "a tile is computed twice or never"
    return True


def simulate_linear_ws(rng: random.Random, n_tiles: int, nk: int, stages: int, arrivals: int = 4, pingpong: bool = True,
                       early_refill: bool = False, **faults):
    """one CTA of gemm_ws_kernel with n_tiles tiles of nk K blocks on the ring (RingModel, block g = i * nk + kb, read by the
    tile's warpgroup alone).  Consumer w takes local tiles i = w, w + 2, ...: fetches the tile's residual into its staging
    tile (cp.async), waits for its turn (warpgroup 1 arrives on warpgroup 0's barrier first; a warpgroup hands over after
    issuing its last MMA when a tile follows), per block waits for it, issues, and releases block g - 1 once
    wgmma.wait_group(1) retired it (the last block after wait_group(0)); then the epilogue and the copy-out of the staging
    tile.  Asserts, beside the ring's: the K loops run one at a time in order 0, 1, 0, 1 ..., and a staging tile is refilled
    only after its copy-out read it.  Negative controls: RingModel's faults, pingpong=False, early_refill (the next residual
    fetch issued before the copy-out)."""
    ring = RingModel(rng, stages, arrivals, 1, **faults)
    loops = []
    t_wg = [rng.uniform(0, 5), rng.uniform(0, 5)]
    handed = [rng.uniform(0, 1), None]  # handed[w]: when the turn was handed to w (warpgroup 1's opening arrive: tile 0)
    copy_done = [None, None]      # end of the last copy-out of each staging tile
    next_fetch = [None, None]     # early_refill: when the next tile's fetch was issued
    for i in range(n_tiles):
        w = i % 2
        t = t_wg[w]
        fetch = next_fetch[w] if early_refill and next_fetch[w] is not None else t
        if copy_done[w] is not None:
            assert copy_done[w] <= fetch, f"staging tile {w} refilled by tile {i} before the copy-out of tile {i - 2} read it"
        res_land = fetch + rng.uniform(5, 50)
        if pingpong:
            assert handed[w] is not None, "a warpgroup waits for a turn nobody hands over (deadlock)"
            t = max(t, handed[w])
            handed[w] = None
        start = t
        prev_retire = 0.0
        for kb in range(nk):
            g = i * nk + kb
            t = ring.wait(g, w, t)
            t += rng.uniform(0.1, 2)                     # issue
            retire = t + rng.uniform(5, 30)
            if kb > 0:
                t = max(t, prev_retire)                  # wgmma.wait_group(1): block g - 1 retired
                ring.release(g - 1, w, t)
            prev_retire = retire
        loops.append((start, t, w))
        if i + 1 < n_tiles:
            handed[1 - w] = t + rng.uniform(0.1, 1)
        t = max(t, prev_retire)                          # wgmma.wait_group(0)
        ring.release(i * nk + nk - 1, w, t)
        t = max(t, res_land) + rng.uniform(5, 40)        # cp.async.wait_group(0), epilogue into the staging tile
        if early_refill:
            next_fetch[w] = t
        t += rng.uniform(5, 40)                          # copy-out
        copy_done[w] = t
        t_wg[w] = t
    loops.sort()
    assert [w for _, _, w in loops] == [i % 2 for i in range(n_tiles)], "the K loops do not take turns 0, 1, 0, 1, ..."
    for (s0, e0, _), (s1, _, _) in zip(loops, loops[1:]):
        assert e0 <= s1, "the K loops of the two consumers overlap"
    return True


# ---------------------------------------------------------------------------------------------------------- conv A tiles by TMA
def conv_ws_rules():
    """checks that gemm_ws.cu / gemm_wgmma.cu still dispatch the conv modes, place each box and walk the taps as
    conv_ws_box, conv_box_origin and tma_a_tile restate them"""
    s = _src("gemm_ws.cu")
    for rule in ("if (p.stride != 1 || BM % p.Wo != 0) return false;", "if (hw % BM != 0) return false;",
                 "box[0] = p.Wo, box[1] = BM / p.Wo, box[2] = 1;", "if (BM % hw != 0) return false;",
                 "box[0] = p.Wo, box[1] = p.Ho, box[2] = BM / hw;", "if (p.HW % BM == 0) box[0] = BM, box[1] = 1, box[2] = 1;",
                 "else if (BM % p.HW == 0 && p.F % (BM / p.HW) == 0) box[0] = p.HW, box[1] = BM / p.HW, box[2] = 1;",
                 "P.ax = g.Wo, P.ay = g.Ho, P.taps_w = g.taps_w;", "P.x_off = g.up2 ? g.px - 1 : -1;",
                 "P.y_off = g.up2 ? g.py - 1 : -1;", "P.ax = g.HW, P.ay = g.F, P.taps_w = 1;", "P.x_off = 0;", "P.y_off = -1;",
                 "const unsigned b4[4] = {64, box[0], box[1], box[2]};",
                 "bx = m0 % P.ax + P.x_off;", "by = m0 / P.ax % P.ay + P.y_off;", "bn = m0 / (P.ax * P.ay);",
                 "tma_load_4d(sA(s), &P.ta, bar, c0, bx + kx, by, bn);", "if ((c0 += BK) == p.Cin) {",
                 "if (++kx == P.taps_w) kx = 0, ++by;"):
        assert rule in s, f"gemm_ws.cu no longer contains {rule!r}: update the model"
    for rule in ("const bool ws = p.mode == AV2V_A_LINEAR || conv_ws_box(p, box);",
                 "if (ws) return gemm_conv_ws(p, box, static_cast<int>(tiles), stream);"):
        assert rule in _src("gemm_wgmma.cu"), f"gemm_wgmma.cu no longer contains {rule!r}: update the model"
    return True


def conv_geometry(mode: str, **g):
    """the GemmP fields av2v_gemm_f16 fills for a conv call.  mode "conv": NF, H, W, Cin, chan (a_channels, default Cin),
    stride (1), phase (0: plain; 1..4: up2 phase (py, px) = ((phase - 1) >> 1, (phase - 1) & 1)); mode "tconv": B, F, HW,
    Cin"""
    if mode == "conv":
        ph, st = g.get("phase", 0), g.get("stride", 1)
        d = dict(mode=mode, NF=g["NF"], Hin=g["H"], Win=g["W"], Ho=g["H"] // st, Wo=g["W"] // st, stride=st, Cin=g["Cin"],
                 chan=g.get("chan", g["Cin"]), up2=int(ph > 0), py=(ph - 1) >> 1 if ph else 0, px=(ph - 1) & 1 if ph else 0,
                 taps_w=2 if ph else 3)
        d.update(M=d["NF"] * d["Ho"] * d["Wo"], K=(4 if ph else 9) * d["Cin"])
    else:
        d = dict(mode=mode, B=g["B"], F=g["F"], HW=g["HW"], Cin=g["Cin"], M=g["B"] * g["F"] * g["HW"], K=3 * g["Cin"])
    return d


def conv_ws_box(p):
    """gemm_ws.cu conv_ws_box: (bx, by, bn), or None when the conv stays on gemm_wgmma_kernel"""
    if p["mode"] == "conv":
        hw = p["Ho"] * p["Wo"]
        if p["stride"] != 1 or 128 % p["Wo"]:
            return None
        if hw >= 128:
            return None if hw % 128 else (p["Wo"], 128 // p["Wo"], 1)
        return None if 128 % hw else (p["Wo"], p["Ho"], 128 // hw)
    if p["HW"] % 128 == 0:
        return (128, 1, 1)
    if 128 % p["HW"] == 0 and p["F"] % (128 // p["HW"]) == 0:
        return (p["HW"], 128 // p["HW"], 1)
    return None


def _conv_tensor(p):
    """the 4-D tensor gemm_conv_ws describes (dims innermost first) and its box origin terms ax, ay, x_off, y_off, taps_w"""
    if p["mode"] == "conv":
        return ((p["chan"], p["Win"], p["Hin"], p["NF"]), p["Wo"], p["Ho"], p["px"] - 1 if p["up2"] else -1,
                p["py"] - 1 if p["up2"] else -1, p["taps_w"])
    return (p["Cin"], p["HW"], p["F"], p["B"]), p["HW"], p["F"], 0, -1, 1


def tma_a_tile(p, x, m0, box, x_off=None, y_off=None, swap_phase=False):
    """the A tiles of every K block of the tile at row m0 as the producer loads them: the box origin of the tile, the tap
    walk (c0, kx, by) per block, and TMA's element placement (box element (i0, i1, i2, i3) -> tile row i1 + bx (i2 + by i3),
    column i0; zero outside the tensor).  x: the flat input, dense in the tensor's dims.  Returns [num_kb, 128, 64].
    x_off / y_off override the tap offsets; swap_phase exchanges the phase offsets (negative controls)."""
    import numpy as np
    dims, ax, ay, xo, yo, taps_w = _conv_tensor(p)
    if swap_phase:
        xo, yo = yo, xo
    xo = xo if x_off is None else x_off
    yo = yo if y_off is None else y_off
    bx_, by_, bn_ = box
    assert bx_ * by_ * bn_ == 128 and max(box) <= 256
    i0, i1, i2, i3 = np.meshgrid(np.arange(64), np.arange(bx_), np.arange(by_), np.arange(bn_), indexing="ij")
    row = (i1 + bx_ * (i2 + by_ * i3)).ravel()
    col = i0.ravel()
    bx, by, bn = m0 % ax + xo, m0 // ax % ay + yo, m0 // (ax * ay)
    c0 = kx = 0
    tiles = []
    for _ in range(p["K"] // 64):
        c = np.stack([(c0 + i0).ravel(), (bx + kx + i1).ravel(), (by + i2).ravel(), (bn + i3).ravel()])
        ok = np.all((c >= 0) & (c < np.array(dims)[:, None]), axis=0)
        flat = ((c[3] * dims[2] + c[2]) * dims[1] + c[1]) * dims[0] + c[0]
        t = np.zeros((128, 64), x.dtype)
        t[row, col] = np.where(ok, x[np.where(ok, flat, 0)], 0)
        tiles.append(t)
        c0 += 64
        if c0 == p["Cin"]:
            c0 = 0
            kx += 1
            if kx == taps_w:
                kx, by = 0, by + 1
    return np.stack(tiles)


def gather_a_tile(p, x, m0):
    """gemm_wgmma.cu a_rows_init + load_stage: the A tiles of every K block of the tile at row m0 as the cp.async gather
    fills them (16-byte chunks, zero-filled out of the image / clip, past a_channels and past M).  [num_kb, 128, 64]"""
    import numpy as np
    r = np.arange(128)
    m = m0 + r
    live = m < p["M"]
    ch = np.arange(64)
    tiles = []
    for kb in range(p["K"] // 64):
        k0 = kb * 64
        if p["mode"] == "conv":
            ox, t = m % p["Wo"], m // p["Wo"]
            oy, n = t % p["Ho"], t // p["Ho"]
            y0 = oy - 1 + p["py"] if p["up2"] else oy * p["stride"] - 1
            x0 = ox - 1 + p["px"] if p["up2"] else ox * p["stride"] - 1
            tap = k0 // p["Cin"]
            c = k0 - tap * p["Cin"] + ch
            ky, kx = tap // p["taps_w"], tap % p["taps_w"]
            y, xx = y0 + ky, x0 + kx
            v = live[:, None] & (c[None, :] // 8 * 8 < p["chan"]) & ((y >= 0) & (y < p["Hin"]) & (xx >= 0) & (xx < p["Win"]))[:, None]
            src = ((n * p["Hin"] + y) * p["Win"] + xx)[:, None] * p["chan"] + c[None, :]
        else:
            kt = k0 // p["Cin"]
            c = k0 - kt * p["Cin"] + ch
            fr = (m % (p["F"] * p["HW"])) // p["HW"]
            f = fr + kt - 1
            v = live[:, None] & ((f >= 0) & (f < p["F"]))[:, None] & np.ones(64, bool)[None, :]
            src = (m + (kt - 1) * p["HW"])[:, None] * p["Cin"] + c[None, :]
        tiles.append(np.where(v, x[np.where(v, src, 0)], 0))
    return np.stack(tiles)


def check_conv_tma_tiles(mode: str, box=None, **kw):
    """every A tile of every K block of every output tile: the producer's TMA boxes hold exactly what gemm_wgmma_kernel's
    gather loads.  box: force this box (default: conv_ws_box, which must accept the geometry); other keywords of
    tma_a_tile (x_off, y_off, swap_phase) break one rule for the negative controls."""
    import numpy as np
    geo = {k: v for k, v in kw.items() if k not in ("x_off", "y_off", "swap_phase")}
    bad = {k: v for k, v in kw.items() if k in ("x_off", "y_off", "swap_phase")}
    p = conv_geometry(mode, **geo)
    box = box or conv_ws_box(p)
    assert box is not None, f"{mode} {geo}: conv_ws_box refuses the geometry"
    dims = _conv_tensor(p)[0]
    n = dims[0] * dims[1] * dims[2] * dims[3]
    x = np.arange(1, n + 1, dtype=np.int64)  # every element distinct and nonzero: a zero is padding
    for m0 in range(0, p["M"], 128):
        want, got = gather_a_tile(p, x, m0), tma_a_tile(p, x, m0, box, **bad)
        if not np.array_equal(want, got):
            kb, r, c = (int(i[0]) for i in np.nonzero(want != got))
            raise AssertionError(f"{mode} {geo}: tile row {m0} K block {kb} row {r} col {c}: TMA box holds {got[kb, r, c]}, "
                                 f"the gather {want[kb, r, c]}")
    return True


# ---------------------------------------------------------------------------------------------------------- persistent fused temporal attention
def tattn_ws_constants():
    """(stages at n_v = 1, stages at n_v = 3, empty-barrier arrivals) of tattn_fused_kernel's projection ring, as written in
    attention_wgmma.cu; also checks the item order and block numbering the models below restate"""
    s = _src("attention_wgmma.cu")
    k = kernel_body("attention_wgmma.cu", "tattn_fused_kernel")
    m = re.search(r"tattn_stages\(\) \{ return NV == 1 \? (\d+) : (\d+); \}", s)
    arrivals = int(re.search(r"ring\.init\((\d+)\);", k).group(1))
    for rule in ("for (int item = blockIdx.x; item < p.items; item += gridDim.x)", "h = item % p.heads;",
                 "pix0 = item % p.pix_tiles * p.ppt;", "clip = item / p.pix_tiles;", "for (int kb = 0; kb < nk; ++kb, ++g) {",
                 "ring.wait(g + kb);", "if (kb > 0) ring.release(g + kb - 1);", "ring.release(g + nk - 1);", "g += nk;",
                 "tma_load_4d(sX(s), &p.tx, bar, kb * 64, 0, pix0, clip + b * p.src_clips);"):
        assert rule in k, f"tattn_fused_kernel no longer contains {rule!r}: update the model"
    for rule in ("const unsigned box[4] = {64, static_cast<unsigned>(a->F), static_cast<unsigned>(p.ppt), 1};",
                 "const unsigned long long strides[3] = {frame, row, frame * a->F};",
                 "items < sm_count_cached() ? items : sm_count_cached()"):
        assert rule in s, f"attention_wgmma.cu no longer contains {rule!r}: update the model"
    return int(m.group(1)), int(m.group(2)), arrivals


def tattn_ws_schedule(clips: int, pix_tiles: int, heads: int, sms: int):
    """the items of each CTA (grid = min(items, sms)), decoded heads fastest.  Asserts every (clip, pixel tile, head) is run
    once and that the items running at one time (item index // grid equal) cover whole pixel tiles: each x tile is wanted by
    all heads at once, so it leaves HBM once"""
    items = clips * pix_tiles * heads
    grid = min(items, sms)
    seen = {}
    for b in range(grid):
        for it in range(b, items, grid):
            h, rest = it % heads, it // heads
            key = (rest // pix_tiles, rest % pix_tiles, h)
            assert key not in seen, f"item {key} run twice"
            seen[key] = it
    assert len(seen) == items
    for (clip, pt, h), it in seen.items():
        first = seen[(clip, pt, 0)]
        assert it - first == h, f"the heads of (clip {clip}, tile {pt}) are not consecutive items"
    return True


def simulate_tattn_ring(rng: random.Random, n_items: int, passes: int, nk: int, stages: int, arrivals: int = 8, **faults):
    """tattn_fused_kernel's projection over the CTA's items on the ring (RingModel, block g = the CTA's g-th K block, item,
    pass and kb in order).  Consumers w = 0, 1: per block wait for it, issue, wait_group(1) -> release block g - 1; after a
    pass's last block wait_group(0) and release it; after an item's last pass an attention phase of random length.
    Negative controls: RingModel's faults."""
    ring = RingModel(rng, stages, arrivals, 2, **faults)
    t_wg = [rng.uniform(0, 5), rng.uniform(0, 5)]
    retire = {}
    for g in range(n_items * passes * nk):
        kb = g % nk
        for w in range(2):
            t = ring.wait(g, w, t_wg[w])
            retire[(g, w)] = t + rng.uniform(5, 40)
            if kb > 0:
                t = max(t, retire[(g - 1, w)])  # wait_group(1): block g - 1 retired
                ring.release(g - 1, w, t)
            if kb == nk - 1:
                t = max(t, retire[(g, w)])      # wait_group(0)
                ring.release(g, w, t)
                if (g // nk) % passes == passes - 1:
                    t += rng.uniform(10, 80)    # the item's attention and stores
            t_wg[w] = t
    return True


def tattn_box_slots(F: int, HW: int, clips: int, clip: int, pix0: int, wrong_order: bool = False):
    """the token row each of the 128 slots of a stage's x block holds after the kernel's TMA box {64, F, ppt, 1} of x viewed as
    (channel, frame, pixel, clip) at (0, 0, pix0, clip): box rows are written frame fastest, then pixel, so box row j is
    (pixel pix0 + j / F, frame j % F); pixels past HW are zero-filled (-1) and the rows past ppt * F are the zeroed tail (-1).
    wrong_order: the box walks (channel, pixel, frame), i.e. the frame and pixel strides swapped (negative control)."""
    import numpy as np
    ppt = 128 // F
    slots = np.full(128, -1)
    for j in range(ppt * F):
        p, f = (j % ppt, j // ppt) if wrong_order else (j // F, j % F)
        pix = pix0 + p
        slots[j] = (clip * F + f) * HW + pix if pix < HW else -1
    return slots


def check_tattn_box_slots(F: int, HW: int, clips: int = 2, **kw):
    """the box's slot contents equal frame_slot_items("fused")'s query rows for every item (tail and ragged pixels -1)"""
    ppt = 128 // F
    items = list(frame_slot_items("fused", F, HW, clips))
    pix_tiles = (HW + ppt - 1) // ppt
    for i, (qrow, _, _) in enumerate(items):
        clip, pt = divmod(i, pix_tiles)
        got = tattn_box_slots(F, HW, clips, clip, pt * ppt, **kw)
        assert (got == qrow).all(), f"F={F} HW={HW} clip {clip} tile {pt}: box slots differ from the slot map"
    return True


def tattn_qksrc_constants():
    """(stages, projection passes per item, empty-barrier arrivals) of tattn_fused_kernel<2, true> (av2v_tattn_fused_qksrc_f16),
    as written in attention_wgmma.cu; also checks the pass order tattn_pass_sources restates"""
    s = _src("attention_wgmma.cu")
    k = kernel_body("attention_wgmma.cu", "tattn_fused_kernel")
    m = re.search(r"tattn_stages\(\) \{ return NV == 1 \? (\d+) : (\d+); \}", s)
    passes = re.search(r"constexpr int passes = QK \? NV \+ (\d+) : NV;", k)
    arrivals = int(re.search(r"ring\.init\((\d+)\);", k).group(1))
    for rule in ("for (int b = 0; b < passes; ++b)", "constexpr int w0 = QK ? 2 : 3;",
                 "else if (b == 0) tma_load_4d(sX(s), &p.tqk, bar, kb * 64, 0, pix0, clip);",
                 "else tma_load_4d(sX(s), &p.tx, bar, kb * 64, 0, pix0, clip + (b - 1) * p.src_clips);",
                 "float acc[QK ? 2 : 3][32];", "for (int b = QK ? 0 : 1; b < NV; ++b) {"):
        assert rule in k, f"tattn_fused_kernel no longer contains {rule!r}: update the model"
    assert "tattn_fused_kernel<2, true><<<" in s, "av2v_tattn_fused_qksrc_f16 no longer launches tattn_fused_kernel<2, true>"
    return int(m.group(2)), 2 + int(passes.group(1)), arrivals


def tattn_pass_sources(nv: int, qk: bool, clip: int, src_clips: int, off_by_one: bool = False):
    """[(tensor, clip, what)] of each projection pass of one item, in the kernel's order: without qk, pass 0 projects Q, K, V
    of x's clip `clip` and pass b > 0 the V of clip + b * src_clips; with qk (n_v = 2), pass 0 projects Q, K of the source
    tensor's clip `clip` and pass b > 0 the V of x's clip + (b - 1) * src_clips.  off_by_one: the V passes of the qk variant
    read clip + b * src_clips (negative control)"""
    if not qk:
        return [("x", clip, "QKV")] + [("x", clip + b * src_clips, "V") for b in range(1, nv)]
    d = 0 if off_by_one else 1
    return [("src", clip, "QK")] + [("x", clip + (b - d) * src_clips, "V") for b in range(1, nv + 1)]


def check_tattn_qksrc_passes(src_clips: int, **kw):
    """every edit clip c + j * src_clips of x (j = 0, 1) has its V projected exactly once, by the item of source clip c, into
    V branch j; Q / K come from the source tensor; the branches are those the n_v = 3 call gives to clips 1, 2 of [source |
    uncond | cond]"""
    seen = {}
    for clip in range(src_clips):
        passes = tattn_pass_sources(2, True, clip, src_clips, **kw)
        assert passes[0] == ("src", clip, "QK")
        three = tattn_pass_sources(3, False, clip, src_clips)
        for j, (tensor, c, what) in enumerate(passes[1:]):
            assert tensor == "x" and what == "V" and 0 <= c < 2 * src_clips, f"source clip {clip}: V pass {j} reads clip {c}"
            assert c not in seen, f"edit clip {c} projected twice"
            seen[c] = (clip, j)
            assert three[1 + j][1] - src_clips == c, f"V branch {j} of source clip {clip} is not the n_v = 3 call's branch {j + 1}"
    assert sorted(seen) == list(range(2 * src_clips))
    return True
