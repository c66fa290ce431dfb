"""Negative controls of the guarded-buffer checks (tests/guarded.py), on CPU: the float64 contract of the linear op
(tests/kernel_contracts.py) stands in for the kernel, untouched and tampered three ways.  Each tampering must make the
checks fail and the untouched contract must pass, which shows the guards catch each failure mode without a GPU."""
import pytest
import torch

import kernel_contracts as kc
from guarded import NAN_BITS, POISON_BITS, check_output, guarded_input, guarded_output
from parity_utils import assert_fp16_close

M, N, K = 37, 40, 24
LDA, LDO = K + 8, N + 8


def _operands():
    torch.manual_seed(0)
    a = guarded_input(torch.randn(M, K).half(), ld=LDA)
    w = guarded_input((torch.randn(N, K) / K ** 0.5).half())
    out = guarded_output((M, N), ld=LDO)
    return a, w, out


def _harness(kernel):
    """what the GPU contract tests do: run the 'kernel' on guarded views, check the guards, compare with float64"""
    a, w, out = _operands()
    kernel(a, w, out)
    check_output(out, "linear")
    assert_fp16_close(out.view, a.view.double() @ w.view.double().t(), "linear")


def _honest(a, w, out):
    kc.linear(a.view, w.view, out=out.view)


def _writes_past_the_view(a, w, out):
    _honest(a, w, out)
    out.buf[out.offset + (M - 1) * LDO + N] = 0.0  # the element after the last one


def _skips_a_row(a, w, out):
    kc.linear(a.view[1:], w.view, out=out.view[1:])


def _reads_the_ld_gap(a, w, out):
    wide = a.buf.as_strided((M, LDA), (LDA, 1), a.offset)  # the rows with their gap
    a_bad = a.view.clone()
    a_bad[M // 2, K - 1] = wide[M // 2, K]  # one column past the end of a row
    kc.linear(a_bad, w.view, out=out.view)


def test_guards_hold_their_patterns():
    a, _, out = _operands()
    bits_a, bits_o = a.buf.view(torch.int16), out.buf.view(torch.int16)
    assert bool((bits_a[~a.inside()] == NAN_BITS).all()) and torch.isnan(a.buf[~a.inside()]).all()
    assert bool((bits_o == POISON_BITS).all()) and torch.isnan(out.buf).all()
    assert a.offset * 2 % 16 == 0 and a.view.stride() == (LDA, 1) and out.view.stride() == (LDO, 1)


def test_untampered_contract_passes():
    _harness(_honest)


def test_stray_write_is_caught():
    a, w, out = _operands()
    _writes_past_the_view(a, w, out)
    with pytest.raises(AssertionError, match="outside the view"):
        check_output(out, "linear")
    with pytest.raises(AssertionError):
        _harness(_writes_past_the_view)


def test_skipped_row_is_caught():
    a, w, out = _operands()
    _skips_a_row(a, w, out)
    with pytest.raises(AssertionError, match="never written"):
        check_output(out, "linear")
    with pytest.raises(AssertionError):
        _harness(_skips_a_row)


def test_gap_read_is_caught():
    with pytest.raises(AssertionError, match="non-finite"):
        _harness(_reads_the_ld_gap)
