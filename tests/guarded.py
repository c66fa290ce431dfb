"""Guarded buffers for kernel tests: every tensor is a view inside a larger contiguous buffer.

The view has a guard band before its first element and after its last one, and where a row stride is allowed, a gap between
the width used and the row stride.
  - Inputs: the guards and gaps hold an fp16 NaN.  A kernel that reads one (a missing zero-fill, an off-by-one predicate, a
    row past the last key) produces a non-finite output, which ``assert_fp16_close`` rejects.
  - Outputs: the whole buffer, view included, is pre-filled with one distinctive NaN bit pattern (POISON).  ``check_output``
    then asserts that every element outside the view still holds it bit for bit (no stray writes) and that no element inside
    the view does (no unwritten elements).
Works on CPU tensors too, so the checks themselves can be tested without a GPU.
"""
from __future__ import annotations

import torch

NAN_BITS = 0x7E00     # fp16 quiet NaN: guards and gaps of inputs
POISON_BITS = 0x7E5A  # fp16 NaN with a payload no arithmetic produces: pre-fill of outputs
GUARD = 64            # default guard band in elements (128 bytes, keeps 16-byte alignment)


def nested_strides(shape, ld=None):
    """strides of a row-major tensor whose dim -2 steps by ``ld`` (default: shape[-1]); outer dims nest over it"""
    strides = [1] * len(shape)
    if len(shape) >= 2:
        strides[-2] = shape[-1] if ld is None else ld
        for i in range(len(shape) - 3, -1, -1):
            strides[i] = strides[i + 1] * shape[i + 1]
    return tuple(strides)


class Guarded:
    """``view``: a tensor of ``shape`` / ``strides`` at element ``offset`` of the 1-D fp16 buffer ``buf``"""

    def __init__(self, buf, shape, strides, offset, fill_bits):
        self.buf, self.shape, self.strides, self.offset, self.fill_bits = buf, tuple(shape), tuple(strides), offset, fill_bits
        self.view = buf.as_strided(self.shape, self.strides, offset)

    @classmethod
    def alloc(cls, shape, strides=None, *, fill_bits, device="cpu", guard=GUARD):
        strides = nested_strides(shape) if strides is None else tuple(strides)
        guard = -(-guard // 64) * 64
        span = 1 + sum((n - 1) * s for n, s in zip(shape, strides)) if all(n > 0 for n in shape) else 0
        bits = torch.full((guard + span + guard,), fill_bits, dtype=torch.int16, device=device)
        return cls(bits.view(torch.float16), shape, strides, guard, fill_bits)

    def inside(self) -> torch.Tensor:
        """bool mask over ``buf``: True at the elements of the view"""
        mask = torch.zeros(self.buf.numel(), dtype=torch.bool, device=self.buf.device)
        mask.as_strided(self.shape, self.strides, self.offset).fill_(True)
        return mask

    def to(self, device) -> "Guarded":
        """a copy of the whole buffer (guards included) on ``device``, with the same view geometry"""
        return Guarded(self.buf.to(device, copy=True), self.shape, self.strides, self.offset, self.fill_bits)


def guarded_input(values: torch.Tensor, *, ld=None, strides=None, device=None, guard=GUARD) -> Guarded:
    """``values`` (fp16) copied into a view whose guards and row gaps hold NaN"""
    shape = tuple(values.shape)
    g = Guarded.alloc(shape, strides if strides is not None else nested_strides(shape, ld), fill_bits=NAN_BITS,
                      device=values.device if device is None else device, guard=guard)
    g.view.copy_(values)
    return g


def guarded_output(shape, *, ld=None, strides=None, device="cpu", guard=GUARD) -> Guarded:
    """an output view whose whole buffer holds POISON"""
    return Guarded.alloc(tuple(shape), strides if strides is not None else nested_strides(tuple(shape), ld), fill_bits=POISON_BITS,
                         device=device, guard=guard)


def guarded_inout(values: torch.Tensor, *, device=None, guard=GUARD) -> Guarded:
    """an in-place operand: ``values`` in a contiguous view, POISON around it"""
    g = guarded_output(values.shape, device=values.device if device is None else device, guard=guard)
    g.view.copy_(values)
    return g


def check_output(g: Guarded, what: str) -> None:
    poison = g.buf.view(torch.int16) == POISON_BITS
    inside = g.inside()
    stray = (~inside & ~poison).nonzero()
    assert stray.numel() == 0, (f"{what}: {stray.numel()} element(s) written outside the view, first at buffer element "
                                f"{int(stray[0])} (view starts at {g.offset})")
    unwritten = (inside & poison).nonzero()
    assert unwritten.numel() == 0, (f"{what}: {unwritten.numel()} element(s) of the view never written, first at buffer element "
                                    f"{int(unwritten[0])} (view starts at {g.offset})")
