"""TEST INFRASTRUCTURE — every kernel call of a model pass checked against its float64 contract, at the arguments the model
actually passes.

``CallAudit.install(monkeypatch)`` wraps the kernel entry points of ``anyv2v_b200.ops`` for one test; every model call site
goes through ``ops.<name>(...)``, so the package itself is untouched.  For each call the wrapper

1. snapshots every input that shares storage with what the call writes (``out``; ``freeu``'s ``hidden``, scaled in place;
   ``dpmpp2m_step``'s ``x0_prev``, read and then overwritten; ``ddim_step`` with ``out = x``; a residual that is also the
   output) — the contract must see the inputs the kernel saw;
2. runs the wrapped op (the sm_90a kernel, or under ``emulated_ops`` its contract) and synchronises;
3. evaluates the op's contract (tests/kernel_contracts.py ``*_exact``, tests/freeu_ref.py, tests/sampling_ref.py,
   tests/dpm_solver_ref.py, tests/source_cache_ref.py, tests/vae_tiling_ref.py) in
   float64 on the inputs' device, on a seeded subset of the call's independent units, each unit addressed exactly as the
   kernel addressed it (rowbias row m // rows_per_rowbias, the residual row, the output slot, the branch strides):

       linear, layernorm      rows: all if M <= 8192, else the first and last 128-row tiles and 2048 seeded rows
       conv3x3, upsample      frames: first, last and 2 seeded frames; every output slot
       tconv3                 clips: first and last
       attention (rows)       query sequences b (keys b // kv_batch_div): first, last and 2 seeded; all heads, rows, branches
       attention (frames),    pixels of a clip: first, last and 254 seeded per clip (edit clip c of a qksrc call: those of
       temporal_attention_    its source clip c mod clips / 2); all frames, heads and branches
       fused(_qksrc)
       groupnorm              samples: first, last and 2 seeded
       ddim_step(_eta)        every element, bit for bit
       dpmpp2m_step           every element of both stores (out and x0_prev), bit for bit
       freeu                  every element: backbone half bit-exact with torch's fp16 ``x * b``, the other half untouched,
                              the filtered skip within the FreeU bound;
       tile_stitch            images: first, last and 1 seeded; every element, bit for bit, from the call's own tiles

4. compares with the op's element-wise bound (tests/ulp_check.py) and records op, argument signature, worst error in fp16
   ulps and the smallest margin.  Failures are collected, not raised, so that one pass shows every bad call.  The same
   comparisons feed the sums of tests/bias_check.py, per op, so that ``assert_unbiased`` checks the mean error of each op
   over the whole pass: a store that rounds in one direction stays inside every call's bound but not inside that mean.

``perturb(op, index, args, out)`` runs after the op and before the check, so a test can corrupt one call's output (the
negative controls of tests/test_call_audit_cpu.py and tests/test_call_audit_passes_cpu.py); ``snapshot_after=True`` takes
the snapshots after the call instead of before, which must make the in-place ops fail.
"""
from __future__ import annotations

import inspect
import math
from dataclasses import dataclass, field

import torch

import dpm_solver_ref
import freeu_ref
import kernel_contracts as kc
import sampling_ref
import source_cache_ref
import vae_tiling_ref
from bias_check import Moments, moments
from ulp_check import (KAPPA_ATTN, KAPPA_FREEU, KAPPA_GEGLU, KAPPA_GEMM, KAPPA_NORM, cond_attention, cond_conv_abs, cond_freeu,
                       cond_geglu, cond_groupnorm, cond_layernorm, cond_linear, measure, ulp16)

AUDITED = ("linear", "conv3x3", "upsample2x_conv3x3", "tconv3", "attention", "temporal_attention_fused",
           "temporal_attention_fused_qksrc", "groupnorm", "layernorm", "ddim_step", "ddim_step_eta", "dpmpp2m_step", "freeu",
           "tile_stitch")
LAUNCHES = {"upsample2x_conv3x3": 4}  # kernel launches per call; 1 for the others
_WRITTEN_IN_PLACE = {"freeu": "hidden", "dpmpp2m_step": "x0_prev"}  # written arguments besides ``out``

ROWS_ALL = 8192      # linear / layernorm: every row up to this M
ROWS_TILE = 128      # ... else the first and last tile of this many rows
ROWS_SEEDED = 2048   # ... and this many seeded rows between them
ATTN_SCORES = 1 << 26  # float64 scores per piece of a rows-mode attention reference (queries are independent)


# ------------------------------------------------------------------------------------------------------------- subsets
def unit_subset(n: int, k: int, seed: int) -> torch.Tensor:
    """sorted indices of units 0 and n - 1 and k seeded units between them (all units if there are no more)"""
    if n <= k + 2:
        return torch.arange(n)
    g = torch.Generator().manual_seed(seed)
    mid = torch.randperm(n - 2, generator=g)[:k] + 1
    return torch.cat([torch.tensor([0, n - 1]), mid]).sort().values


def row_subset(M: int, seed: int) -> torch.Tensor:
    """every row if M <= ROWS_ALL, else the first and last ROWS_TILE rows and ROWS_SEEDED seeded rows between them"""
    if M <= ROWS_ALL:
        return torch.arange(M)
    g = torch.Generator().manual_seed(seed)
    mid = torch.randperm(M - 2 * ROWS_TILE, generator=g)[:ROWS_SEEDED] + ROWS_TILE
    return torch.cat([torch.arange(ROWS_TILE), mid, torch.arange(M - ROWS_TILE, M)]).sort().values


# ------------------------------------------------------------------------------------------------------------- records
@dataclass
class Record:
    index: int          # call number within the audit
    op: str
    sig: str            # argument signature, e.g. "attention rows n_v=3 batch=48 seq=4096 heads=5"
    attrs: dict         # the same as fields, for the tests' "this kind was reached" checks
    units: str          # what was checked
    n: int = 0          # elements compared
    worst_ulp: float = 0.0
    margin: float = 1.0  # min over the compared elements of (bound - err) / bound; < 0 fails
    ok: bool = True
    detail: str = ""
    bias: Moments = field(default_factory=Moments)  # the element-wise parts' sums of e (bit-exact parts have none)

    def line(self):
        return (f"#{self.index} {self.sig} [{self.units}]: worst {self.worst_ulp:.3g} ulp16, margin {self.margin:+.3g}"
                + ("" if self.ok else f" FAILED: {self.detail}"))


def _storage_key(t):
    return (t.device, t.untyped_storage().data_ptr())


def _snap(t, cache):
    """a copy of t's storage (one per storage: views keep their aliasing) with t's view of it"""
    key = _storage_key(t)
    if key not in cache:
        cache[key] = t.untyped_storage().clone()
    return torch.empty(0, dtype=t.dtype, device=t.device).set_(cache[key], t.storage_offset(), t.shape, t.stride())


def _sync(t):
    if t is not None and t.is_cuda:
        torch.cuda.synchronize(t.device)


def _idx(i, t):
    return i.to(t.device)


class CallAudit:
    def __init__(self, seed: int = 0, perturb=None, snapshot_after: bool = False):
        self.seed = seed
        self.perturb = perturb
        self.snapshot_after = snapshot_after
        self.records: list[Record] = []
        self.launches = 0

    # ---------------------------------------------------------------------------------------------------- install
    def install(self, monkeypatch):
        from anyv2v_b200 import ops
        for name in AUDITED:
            fn = getattr(ops, name)
            monkeypatch.setattr(ops, name, self._wrap(name, fn))
        return self

    def _wrap(self, name, fn):
        sig = _PRODUCT_SIGNATURES[name]  # bind as the product wrapper does (the contracts name a few parameters differently)

        def audited(*args, **kwargs):
            p = sig.bind(*args, **kwargs)
            p.apply_defaults()
            p = dict(p.arguments)
            written = [t for t in (p.get("out"), p.get(_WRITTEN_IN_PLACE.get(name))) if t is not None]
            keys = {_storage_key(t) for t in written}
            cache = {}

            def snapshot():
                return {k: (_snap(v, cache) if isinstance(v, torch.Tensor) and _storage_key(v) in keys else v)
                        for k, v in p.items()}

            snap = None if self.snapshot_after else snapshot()
            out = fn(*args, **kwargs)
            _sync(out if isinstance(out, torch.Tensor) else None)
            index = len(self.records)
            if self.perturb is not None:
                self.perturb(name, index, p, out)
            if self.snapshot_after:
                snap = snapshot()
            if name in _WRITTEN_IN_PLACE:  # the live tensor, for the check of what the call wrote into it
                snap["_after"] = p[_WRITTEN_IN_PLACE[name]]
            self.launches += LAUNCHES.get(name, 1)
            n0 = kc._launches  # the contracts count launches when they stand in for the kernels; the audit's own evaluations must not
            try:
                with torch.no_grad():
                    self.records.append(getattr(self, "_check_" + name)(index, snap, out))
            finally:
                kc._launches = n0
            return out

        return audited

    # ---------------------------------------------------------------------------------------------------- results
    def failures(self):
        return [r for r in self.records if not r.ok]

    def assert_clean(self):
        bad = self.failures()
        assert not bad, f"{len(bad)} of {len(self.records)} audited calls over their bound:\n" + "\n".join(r.line() for r in bad)

    def seen(self, op, **want):
        """records of `op` whose attrs hold every item of `want` (a value, or a predicate)"""
        def match(r):
            return r.op == op and all((v(r.attrs.get(k)) if callable(v) else r.attrs.get(k) == v) for k, v in want.items())
        return [r for r in self.records if match(r)]

    def table(self) -> str:
        rows = {}
        for r in self.records:
            c, u, m = rows.get(r.sig, (0, 0.0, math.inf))
            rows[r.sig] = (c + 1, max(u, r.worst_ulp), min(m, r.margin))
        w = max([len(s) for s in rows] + [9])
        lines = [f"{'signature':<{w}}  calls  worst ulp16  min margin"]
        lines += [f"{s:<{w}}  {c:5d}  {u:11.3g}  {m:+10.3g}" for s, (c, u, m) in rows.items()]
        return "\n".join(lines)

    def bias_by_op(self) -> dict:
        """op -> Moments pooled over every call of the op"""
        out = {}
        for r in self.records:
            out.setdefault(r.op, Moments())
            out[r.op] += r.bias
        return out

    def assert_unbiased(self):
        """every op with element-wise parts: mean error within the bias bound of tests/bias_check.py, with power"""
        bad = [f"{op}: {mo.line()}: {v}" for op, mo in self.bias_by_op().items() if mo.n_all and (v := mo.verdict())]
        assert not bad, "mean error of the pass over the bias bound:\n" + "\n".join(bad)

    def families(self) -> dict:
        """op -> (calls, worst ulp, smallest margin)"""
        out = {}
        for r in self.records:
            c, u, m = out.get(r.op, (0, 0.0, math.inf))
            out[r.op] = (c + 1, max(u, r.worst_ulp), min(m, r.margin))
        return out

    # ---------------------------------------------------------------------------------------------------- compare
    def _seed(self, index):
        return self.seed * 1000003 + index

    @staticmethod
    def _record(index, op, sig, attrs, units, parts):
        """parts: (what, got, ref, cond, kappa) element-wise bounds or (what, got, want) bit-exact comparisons"""
        rec = Record(index, op, sig, attrs, units)
        margin, worst, bad = math.inf, 0.0, []
        for part in parts:
            if len(part) == 3:
                what, got, want = part
                same = torch.equal(got.contiguous().view(torch.int16), want.contiguous().view(torch.int16))
                n = got.numel()
                if same:
                    m_ulp, m_margin = 0.0, 1.0
                else:
                    g, w = got.double().reshape(-1), want.double().reshape(-1)
                    diff = (g != w) & ~(torch.isnan(g) & torch.isnan(w))
                    i = int(torch.nonzero(diff)[0]) if bool(diff.any()) else 0
                    m_ulp = float(((g - w).abs() / ulp16(w)).nan_to_num(math.inf).max())
                    m_margin = -math.inf
                    bad.append(f"{what}: {int(diff.sum())} of {n} elements differ from the contract, first at flat index {i}: "
                               f"got {float(g[i])!r} want {float(w[i])!r}")
            else:
                what, got, ref, cond, kappa = part
                m = measure(got, ref, cond, kappa)
                rec.bias += moments(got, ref, cond, kappa)
                n = m["n"]
                m_ulp, m_margin = m["err_ulp"], -m["over_rel"]
                if m["n_bad"]:
                    idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(m["worst"]), tuple(got.shape)))
                    bad.append(f"{what}: {m['n_bad']} of {n} elements over the bound, worst at {idx}: got {m['got']!r} ref "
                               f"{m['ref']!r}, err {m['worst_ulp_err']:.3g} ulp16, bound {m['bound_ulp']:.3g} ulp16")
            rec.n += n
            worst, margin = max(worst, m_ulp), min(margin, m_margin)
        rec.worst_ulp, rec.margin = worst, (margin if parts else 1.0)
        rec.ok = not bad
        rec.detail = "; ".join(bad)
        return rec

    # ---------------------------------------------------------------------------------------------------- per op
    def _check_linear(self, index, p, out):
        a, w, a2, geglu = p["a"], p["w"], p["a2"], bool(p["geglu"])
        M, N = a.shape[0], w.shape[0]
        K = a.shape[1] + (0 if a2 is None else a2.shape[1])
        rpr = p["rows_per_rowbias"]
        rows = row_subset(M, self._seed(index))
        r = _idx(rows, a)
        a_s, a2_s = a[r], (None if a2 is None else a2[r])
        res_s = None if p["residual"] is None else p["residual"].reshape(M, N)[r]
        rb_s = None if p["rowbias"] is None else p["rowbias"][r // rpr]  # the row's own rowbias row, as the kernel reads it
        got = out.reshape(M, -1)[r]
        ref = kc.linear_exact(a_s, w, p["bias"], res_s, rb_s, 1, geglu, a2_s)
        if geglu:
            cond, kappa = cond_geglu(a_s if a2_s is None else torch.cat([a_s, a2_s], 1), w, p["bias"]), KAPPA_GEGLU
        else:
            cond, kappa = cond_linear(a_s, w, p["bias"], rb_s, 1, res_s, a2_s), KAPPA_GEMM
        flags = [f for f, on in (("bias", p["bias"] is not None), (f"rowbias/{rpr}", rb_s is not None),
                                 ("res", res_s is not None), ("geglu", geglu), (f"a2 K={a.shape[1]}+{K - a.shape[1]}", a2 is not None),
                                 (f"lda={a.stride(0)}", a.stride(0) != a.shape[1])) if on]
        sig = " ".join([f"linear M={M} N={N} K={K}"] + flags)
        attrs = dict(M=M, N=N, K=K, geglu=geglu, two_source=a2 is not None, residual=res_s is not None,
                     rowbias=rb_s is not None, lda=a.stride(0))
        return self._record(index, "linear", sig, attrs, f"{len(rows)} of {M} rows", [("linear", got, ref, cond, kappa)])

    def _check_conv3x3(self, index, p, out):
        x, w, stride, slots, sstride = p["x"], p["w_packed"], p["stride"], p["n_slots"], p["slot_stride"]
        NF, H, W, C = x.shape
        Ho, Wo, Cout = H // stride, W // stride, w.shape[0]
        M, rpf = NF * Ho * Wo, Ho * Wo
        rpr = p["rows_per_rowbias"]
        frames = unit_subset(NF, 2, self._seed(index))
        m = _idx((frames[:, None] * rpf + torch.arange(rpf)).reshape(-1), x)
        xs = x[_idx(frames, x)]
        rb_s = None if p["rowbias"] is None else p["rowbias"][m // rpr]
        acc = kc.conv3x3_exact(xs, w, p["bias"], rb_s, 1, stride)
        cacc = cond_conv_abs(kc.conv3x3_exact, xs, w, p["bias"], rb_s, 1, stride)
        ld = out.stride(-2)
        rows = lambda t, s: t.as_strided((M, Cout), (ld, 1), t.storage_offset() + s * sstride)  # slot s, row m (kernel layout)
        parts = []
        for s in range(slots):
            res = None if p["residual"] is None else rows(p["residual"], s)[m].double()
            ref, cond = (acc, cacc) if res is None else (acc + res, cacc + res.abs())
            parts.append((f"conv3x3 slot {s}", rows(out, s)[m], ref, cond, KAPPA_GEMM))
        flags = [f for f, on in ((f"stride={stride}", stride != 1), (f"slots={slots}", slots > 1), ("bias", p["bias"] is not None),
                                 (f"rowbias/{rpr}", rb_s is not None), ("res", p["residual"] is not None),
                                 (f"Cin={w.shape[1] // 9}", C != w.shape[1] // 9), (f"ldo={ld}", ld != Cout)) if on]
        sig = " ".join([f"conv3x3 NF={NF} {H}x{W} C={C} Cout={Cout}"] + flags)
        attrs = dict(NF=NF, H=H, W=W, C=C, Cout=Cout, stride=stride, slots=slots, residual=p["residual"] is not None)
        return self._record(index, "conv3x3", sig, attrs, f"frames {frames.tolist()} of {NF}", parts)

    def _check_upsample2x_conv3x3(self, index, p, out):
        x, w = p["x"], p["w_phases"]
        NF, H, W, Cin = x.shape
        frames = unit_subset(NF, 2, self._seed(index))
        f = _idx(frames, x)
        xs = x[f]
        ref = kc.upsample2x_conv3x3_exact(xs, w, p["bias"])
        cond = cond_conv_abs(kc.upsample2x_conv3x3_exact, xs, w, p["bias"])
        sig = f"upsample2x_conv3x3 NF={NF} {H}x{W} Cin={Cin} Cout={w.shape[1]}"
        return self._record(index, "upsample2x_conv3x3", sig, dict(NF=NF, H=H, W=W, Cin=Cin, Cout=w.shape[1]),
                            f"frames {frames.tolist()} of {NF}", [("upsample", out[f], ref, cond, KAPPA_GEMM)])

    def _check_tconv3(self, index, p, out):
        x, w, F_, HW = p["x"], p["w_packed"], p["F"], p["HW"]
        B, R, Cin = x.shape
        Cout = w.shape[0]
        clips = torch.tensor(sorted({0, B - 1}))
        c = _idx(clips, x)
        xs = x[c]
        res = None if p["residual"] is None else p["residual"].reshape(B, R, Cout)[c]
        ref = kc.tconv3_exact(xs, w, F_, HW, p["bias"], res).view(len(clips), R, Cout)
        cond = cond_conv_abs(kc.tconv3_exact, xs, w, F_, HW, p["bias"], res).view(len(clips), R, Cout)
        got = out.reshape(B, R, -1)[c]
        sig = f"tconv3 B={B} F={F_} HW={HW} Cin={Cin} Cout={Cout}" + (" res" if res is not None else "")
        return self._record(index, "tconv3", sig, dict(B=B, F=F_, HW=HW, Cin=Cin, residual=res is not None),
                            f"clips {clips.tolist()} of {B}", [("tconv3", got, ref, cond, KAPPA_GEMM)])

    def _check_groupnorm(self, index, p, out):
        x, x2 = p["x"], p["x2"]
        n, rows, C1 = x.shape
        C = C1 + (0 if x2 is None else x2.shape[2])
        samples = unit_subset(n, 2, self._seed(index))
        parts = []
        for s in samples.tolist():  # one sample at a time: the per-clip samples hold 10^8 elements
            xs, x2s = x[s:s + 1], (None if x2 is None else x2[s:s + 1])
            ref = kc.groupnorm_exact(xs, p["gamma"], p["beta"], p["groups"], p["eps"], p["silu"], x2=x2s)
            cond = cond_groupnorm(xs, p["gamma"], p["beta"], p["groups"], p["eps"], p["silu"], x2=x2s)
            parts.append((f"groupnorm sample {s}", out[s:s + 1], ref, cond, KAPPA_NORM))
            del ref, cond
        chans = f"C={C1}" if x2 is None else f"C={C1}+{C - C1}"
        part = p["partition_samples"]
        sig = (f"groupnorm n={n} rows={rows} {chans} groups={p['groups']} eps={p['eps']:g}" + (" silu" if p["silu"] else "")
               + (f" partition_samples={part}" if part else ""))
        attrs = dict(n=n, rows=rows, C=C, two_source=x2 is not None, silu=bool(p["silu"]), eps=p["eps"], groups=p["groups"],
                     partition_samples=part)
        return self._record(index, "groupnorm", sig, attrs, f"samples {samples.tolist()} of {n}", parts)

    def _check_layernorm(self, index, p, out):
        x = p["x"]
        C = x.shape[-1]
        M = x.numel() // C
        rows = row_subset(M, self._seed(index))
        r = _idx(rows, x)
        xs = x.reshape(M, C)[r]
        ref = kc.layernorm_exact(xs, p["gamma"], p["beta"], p["eps"])
        cond = cond_layernorm(xs, p["gamma"], p["beta"], p["eps"])
        return self._record(index, "layernorm", f"layernorm rows={M} C={C}", dict(rows=M, C=C), f"{len(rows)} of {M} rows",
                            [("layernorm", out.reshape(M, C)[r], ref, cond, KAPPA_NORM)])

    def _attn_frames_rows(self, index, clips, F_, HW, n_src):
        """frame-major row indices [clips, F, P] of P checked pixels per clip (first, last, 254 seeded); clip c uses the pixel
        set of source clip c % n_src, so that the branches of one clip are checked at the same pixels"""
        psets = [unit_subset(HW, 254, self._seed(index) * 7919 + c) for c in range(n_src)]
        P = len(psets[0])
        pix = torch.stack([psets[c % n_src] for c in range(clips)])  # [clips, P]
        return (torch.arange(clips)[:, None, None] * F_ * HW + torch.arange(F_)[None, :, None] * HW + pix[:, None, :]), P

    def _check_attention(self, index, p, out):
        q, k, v = p["q"], p["k"], p["v"]
        heads, seq, batch, n_v, scale = p["heads"], p["seq"], p["batch"], p["n_v"], p["scale"]
        C = heads * 64
        ldv, ldo = v.stride(0), out.stride(0)
        vrows = p["v_branch_stride"] // ldv if n_v > 1 else 0  # n_v = 3: [source, uncond, cond]; n_v = 2: [uncond, cond]
        orows = p["o_branch_stride"] // ldo if n_v > 1 else 0
        cond_fn = cond_attention(scale)
        parts = []
        if not p["frames_mode"]:
            div = p["kv_batch_div"] if p["kv_batch_div"] > 0 else 1
            nk = p["seq_kv"] if p["seq_kv"] > 0 else seq
            seqs = unit_subset(batch, 2, self._seed(index))
            chunk = max(64, min(seq, ATTN_SCORES // (heads * nk)))
            for b in seqs.tolist():
                kb = b // div
                kk = k[kb * nk:(kb + 1) * nk]
                vv = torch.cat([v[br * vrows + kb * nk:br * vrows + (kb + 1) * nk, :C] for br in range(n_v)])
                for q0 in range(0, seq, chunk):
                    L = min(chunk, seq - q0)
                    qq = q[b * seq + q0:b * seq + q0 + L]
                    dummy = torch.empty((n_v * L, C), dtype=torch.float16, device=q.device)
                    ref, cond = kc.attention_exact(qq, kk, vv, heads, L, 1, dummy, scale, n_v, nk * vv.stride(0), L * C,
                                                   seq_kv=nk, cond=cond_fn)
                    for br in range(n_v):
                        o = out[br * orows + b * seq + q0:br * orows + b * seq + q0 + L, :C]
                        parts.append((f"attention seq {b} branch {br} queries {q0}:{q0 + L}", o, ref[br * L:(br + 1) * L],
                                      cond[br * L:(br + 1) * L], KAPPA_ATTN))
            units = f"sequences {seqs.tolist()} of {batch}"
            sig = f"attention rows n_v={n_v} batch={batch} seq={seq} heads={heads}"
            if p["seq_kv"] > 0 or div > 1:
                sig += f" seq_kv={nk} kv_batch_div={div}"
            attrs = dict(mode="rows", n_v=n_v, batch=batch, seq=seq, heads=heads, seq_kv=nk, kv_batch_div=div,
                         ldk_in_C=k.stride(0) / C)
        else:
            HW = p["HW"]
            clips = batch // HW
            idx, P = self._attn_frames_rows(index, clips, seq, HW, clips)
            flat = idx.reshape(-1)
            f = _idx(flat, q)
            vv = torch.cat([v[_idx(flat + br * vrows, v), :C] for br in range(n_v)])
            dummy = torch.empty((n_v * flat.numel(), C), dtype=torch.float16, device=q.device)
            ref, cond = kc.attention_exact(q[f, :C], k[f, :C], vv, heads, seq, clips * P, dummy, scale, n_v,
                                           flat.numel() * vv.stride(0), flat.numel() * C, frames_mode=True, HW=P, cond=cond_fn)
            n = flat.numel()
            for br in range(n_v):
                parts.append((f"attention frames branch {br}", out[_idx(flat + br * orows, out), :C], ref[br * n:(br + 1) * n],
                              cond[br * n:(br + 1) * n], KAPPA_ATTN))
            units = f"{P} of {HW} pixels per clip, {clips} clips"
            sig = f"attention frames n_v={n_v} clips={clips} F={seq} HW={HW} heads={heads}"
            attrs = dict(mode="frames", n_v=n_v, clips=clips, F=seq, HW=HW, heads=heads)
        return self._record(index, "attention", sig, attrs, units, parts)

    def _check_temporal_attention_fused(self, index, p, out):
        x, wqkv, heads, F_, HW, clips, n_v, scale = p["x"], p["wqkv"], p["heads"], p["F"], p["HW"], p["clips"], p["n_v"], p["scale"]
        C = heads * 64
        idx, P = self._attn_frames_rows(index, clips, F_, HW, clips // n_v)
        flat = _idx(idx.reshape(-1), x)
        dummy = torch.empty((flat.numel(), C), dtype=torch.float16, device=x.device)
        ref, cond = kc.temporal_attention_fused_exact(x[flat], wqkv, heads, F_, P, clips, dummy, scale, n_v,
                                                      cond=cond_attention(scale, rounded_operands=True))
        sig = f"temporal_attention_fused n_v={n_v} clips={clips} F={F_} HW={HW} heads={heads} Cx={x.shape[1]}"
        return self._record(index, "temporal_attention_fused", sig, dict(n_v=n_v, clips=clips, F=F_, HW=HW, heads=heads),
                            f"{P} of {HW} pixels per clip, {clips} clips",
                            [("temporal attention fused", out[flat, :C], ref, cond, KAPPA_ATTN)])

    def _check_temporal_attention_fused_qksrc(self, index, p, out):
        x, qk_src, wqkv, heads, F_, HW, clips, scale = p["x"], p["qk_src"], p["wqkv"], p["heads"], p["F"], p["HW"], p["clips"], p["scale"]
        C = heads * 64
        idx, P = self._attn_frames_rows(index, clips, F_, HW, clips // 2)  # edit clip c at the pixels of source clip c % (clips/2)
        flat = _idx(idx.reshape(-1), x)
        src = _idx(idx[:clips // 2].reshape(-1), qk_src)  # the source clips' rows: source clip c is laid out as edit clip c
        dummy = torch.empty((flat.numel(), C), dtype=torch.float16, device=x.device)
        ref, cond = source_cache_ref.temporal_attention_fused_qksrc_exact(
            x[flat], qk_src[src], wqkv, heads, F_, P, clips, dummy, scale, cond=cond_attention(scale, rounded_operands=True))
        n = src.numel()
        got = out[flat, :C]
        parts = [(f"temporal attention fused qksrc branch {br}", got[br * n:(br + 1) * n], ref[br * n:(br + 1) * n],
                  cond[br * n:(br + 1) * n], KAPPA_ATTN) for br in range(2)]
        sig = f"temporal_attention_fused_qksrc clips={clips} F={F_} HW={HW} heads={heads} Cx={x.shape[1]}"
        return self._record(index, "temporal_attention_fused_qksrc", sig, dict(clips=clips, F=F_, HW=HW, heads=heads),
                            f"{P} of {HW} pixels per clip, {clips} clips", parts)

    def _check_ddim_step(self, index, p, out):
        want = kc.ddim_step(p["x"], p["v_neg"], p["v_edit"], p["guidance"], p["ca"], p["cb"], p["cc"], p["cd"],
                            inverse=p["inverse"], coef_dev=p["coef_dev"])
        sig = f"ddim_step n={p['x'].numel()}" + (" inverse" if p["inverse"] else "") + (" cfg" if p["v_edit"] is not None else "")
        sig += " in-place" if p["out"] is not None and _storage_key(p["out"]) == _storage_key(p["x"]) else ""
        return self._record(index, "ddim_step", sig, dict(n=p["x"].numel(), inverse=bool(p["inverse"])), "all",
                            [("ddim_step", out.reshape(-1), want.reshape(-1))])

    def _check_ddim_step_eta(self, index, p, out):
        want = sampling_ref.ddim_step_eta(p["x"], p["v_neg"], p["v_edit"], p["noise"], p["guidance"], p["ca"], p["cb"], p["cc"],
                                          p["cd"], p["cs"], coef_dev=p["coef_dev"])
        sig = f"ddim_step_eta n={p['x'].numel()}" + (" cfg" if p["v_edit"] is not None else "")
        return self._record(index, "ddim_step_eta", sig, dict(n=p["x"].numel()), "all",
                            [("ddim_step_eta", out.reshape(-1), want.reshape(-1))])

    def _check_dpmpp2m_step(self, index, p, out):
        x0_prev = p["x0_prev"].clone()  # the snapshot of the previous x0; the contract overwrites it with this step's
        want = dpm_solver_ref.dpmpp2m_step(p["x"], p["v_neg"], p["v_edit"], x0_prev, p["guidance"], p["alpha"], p["sigma"],
                                           p["a"], p["b"], p["c"], coef_dev=p["coef_dev"])
        c = float(p["c"] if p["coef_dev"] is None else p["coef_dev"][4])
        order = 1 if c == 0.0 else 2
        cfg = p["v_edit"] is not None
        in_place = p["out"] is not None and _storage_key(p["out"]) == _storage_key(p["x"])  # the snapshots share storage too
        sig = f"dpmpp2m_step n={p['x'].numel()} order={order}" + (" cfg" if cfg else "") + (" in-place" if in_place else "")
        return self._record(index, "dpmpp2m_step", sig, dict(n=p["x"].numel(), order=order, cfg=cfg, in_place=in_place), "all",
                            [("dpmpp2m_step out", out.reshape(-1), want.reshape(-1)),
                             ("dpmpp2m_step x0_prev", p["_after"].reshape(-1), x0_prev.reshape(-1))])

    def _check_freeu(self, index, p, out):
        h0, h1, skip, b, s = p["hidden"], p["_after"], p["skip"], p["b"], p["s"]
        half = h0.shape[-1] // 2
        s32 = float(torch.tensor(s, dtype=torch.float32))
        ref = freeu_ref.fourier_filter_closed_form(skip.double(), s32)
        parts = [("freeu hidden[..., :C/2]", h1[..., :half], h0[..., :half] * b),
                 ("freeu hidden[..., C/2:]", h1[..., half:], h0[..., half:]),
                 ("freeu filtered skip", out, ref, cond_freeu(skip, s), KAPPA_FREEU)]
        NF, H, W, Cs = skip.shape
        sig = f"freeu NF={NF} {H}x{W} Ch={h0.shape[-1]} Cs={Cs} b={b:g} s={s:g}"
        return self._record(index, "freeu", sig, dict(NF=NF, H=H, W=W, Ch=h0.shape[-1], Cs=Cs), "all", parts)

    def _check_tile_stitch(self, index, p, out):
        tiles = p["tiles"]
        geo = [p[k] for k in ("H", "W", "tile", "step", "blend", "row_limit")]
        N, rows, cols, C = len(tiles), len(tiles[0]), len(tiles[0][0]), tiles[0][0][0].shape[0]
        images = unit_subset(N, 1, self._seed(index))
        parts = [(f"tile_stitch image {n}", out[n], vae_tiling_ref.stitch_closed_form([tiles[n]], *geo)[0])
                 for n in images.tolist()]
        H, W, tile, step, blend, row_limit = geo
        sig = f"tile_stitch N={N} C={C} {H}x{W} tiles={rows}x{cols} tile={tile} step={step} blend={blend} row_limit={row_limit}"
        return self._record(index, "tile_stitch", sig, dict(N=N, C=C, H=H, W=W, rows=rows, cols=cols),
                            f"images {images.tolist()} of {N}", parts)


def _product_signatures():
    """the parameter lists of anyv2v_b200.ops, read before any test patches the module"""
    from anyv2v_b200 import ops
    return {name: inspect.signature(getattr(ops, name)) for name in AUDITED}


_PRODUCT_SIGNATURES = _product_signatures()
