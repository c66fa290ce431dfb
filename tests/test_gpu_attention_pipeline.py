"""GPU tests of the rows-mode attention kernel (attn_rows_kernel: producer warp, TMA stage ring, ping-pong consumers) against
the float64 contract, element by element within KAPPA_ATTN * cond (tests/ulp_check.py), inside guarded buffers.

Rows-mode calls with 512 keys or more run attn_rows_kernel, shorter ones attn_kernel.  The cases sit at the kernels' edges:
every rows-mode shape of the benchmark's inversion and edit steps (on seeded subsets of their sequences and heads), query lengths that are not multiples of the 128-row query tile, key lengths around the 64- and
128-key tiles (the tensor maps must zero-fill past the last key: the guards hold NaN there), NaN gaps between the V branches,
kv_batch_div > 1, distinct ldq / ldk / ldv / ldo, and grids of more CTAs than the GPU has SMs."""
import pytest
import torch

import kernel_contracts as kc
from guarded import check_output, guarded_input, guarded_output
from ulp_check import KAPPA_ATTN, assert_within_bound, cond_attention

pytestmark = pytest.mark.gpu
dev = "cuda"


def _branches(rows, C, nv, g, gap=64):
    """nv branches of V rows with `gap` NaN rows between them -> (values, branch stride in rows)"""
    v = [torch.randn(rows, C, generator=g).half() for _ in range(nv)]
    if nv == 1:
        return v[0], 0
    nan = torch.full((gap, C), float("nan"), dtype=torch.float16)
    return torch.cat([v[0], nan, v[1], nan, v[2]]), rows + gap


def _run(batch, heads, seq, seq_kv, div, nv, pad=(8, 16, 24, 40), scale=0.125, seed=0):
    from anyv2v_b200 import ops
    g = torch.Generator().manual_seed(seed)
    C = heads * 64
    ldq, ldk, ldv, ldo = (C + p for p in pad)
    nk = seq_kv if seq_kv else seq
    kv_rows = batch // max(div, 1) * nk
    q = torch.randn(batch * seq, C, generator=g).half()
    k = torch.randn(kv_rows, C, generator=g).half()
    vvals, vstride = _branches(kv_rows, C, nv, g)
    gq = guarded_input(q, ld=ldq, device=dev, guard=128 * ldq)
    gk = guarded_input(k, ld=ldk, device=dev, guard=128 * ldk)
    gv = guarded_input(vvals, ld=ldv, device=dev, guard=128 * ldv)
    out = guarded_output((nv * batch * seq, C), ld=ldo, device=dev)
    kw = dict(scale=scale, n_v=nv, v_branch_stride=vstride * ldv, o_branch_stride=batch * seq * ldo if nv == 3 else 0,
              seq_kv=seq_kv, kv_batch_div=div)
    ops.attention(gq.view, gk.view, gv.view, heads, seq, batch, out.view, **kw)
    torch.cuda.synchronize()
    what = f"attention rows b{batch} h{heads} s{seq} kv{seq_kv} div{div} nv{nv}"
    check_output(out, what)
    o = torch.empty(nv * batch * seq, ldo, dtype=torch.float16)[:, :C]  # the contract maps branches with out's row stride
    ref, cond = kc.attention_exact(gq.to("cpu").view, gk.to("cpu").view, gv.to("cpu").view, heads, seq, batch, o,
                                   cond=cond_attention(scale), **kw)
    got = out.view.cpu()
    assert_within_bound(got, ref, cond, KAPPA_ATTN, what, shape=tuple(got.shape))


# batch, heads, seq, seq_kv, kv_batch_div: the benchmark's rows-mode shapes (4096 x 5, 1024 x 10, 256 x 20, 64 x 20 self-
# attention; cross-attention to 145 keys with kv_batch_div 16) on a subset of sequences and heads
MODEL = [(1, 1, 4096, 0, 1), (1, 2, 1024, 0, 1), (2, 20, 256, 0, 1), (4, 20, 64, 0, 1),
         (16, 1, 1024, 145, 16), (16, 2, 256, 145, 16), (16, 2, 64, 145, 16)]


@pytest.mark.parametrize("nv", [1, 3])
@pytest.mark.parametrize("shape", MODEL, ids=lambda c: "b{}h{}s{}kv{}div{}".format(*c))
def test_rows_model_shapes(shape, nv):
    _run(*shape, nv=nv, seed=shape[2] + nv)


@pytest.mark.parametrize("nv", [1, 3])
@pytest.mark.parametrize("seq", [1, 100, 129, 200, 1000])
def test_rows_ragged_queries(seq, nv):
    """query lengths that are not multiples of the 128-row query tile (600 keys: attn_rows_kernel): the rows past seq load as
    zeros and are not stored"""
    _run(2, 2, seq, 600, 1, nv, seed=seq)


@pytest.mark.parametrize("nv", [1, 3])
@pytest.mark.parametrize("base", [0, 512])
@pytest.mark.parametrize("tail", [1, 63, 64, 65, 127, 128, 129, 145])
def test_rows_key_tails(tail, base, nv):
    """key lengths around the 64- and 128-key tiles, with NaN rows after the last key and between the V branches: below 512
    keys on attn_kernel, from 512 on attn_rows_kernel (whose last tile then holds tail % tile keys)"""
    _run(4, 2, 130, base + tail, 2, nv, seed=base + tail)


@pytest.mark.parametrize("nv", [1, 3])
def test_rows_more_ctas_than_sms(nv):
    """8 sequences x 4 heads x 8 query tiles = 256 CTAs (more than an H100's 132 SMs), 700 keys: the ring wraps several times"""
    _run(8, 4, 1000, 700, 1, nv, pad=(64, 0, 136, 8), scale=0.3, seed=nv)
