"""The layout and run-twice checks every GPU replay trusts (tests/kernel_check.py: layout, twice, determinism), run on CPU tensors against
fake kernels: each writes a [ROWS, C] output into a NaN-poisoned [ROWS + TAIL, PITCH] buffer, the way the replays call the real ones.  The
checks must reject a kernel that leaves an owned element unwritten, one that writes one element past its columns, one that writes into
the tail rows and one whose two runs differ in one bit, and accept an honest one."""
import pytest
import torch

from kernel_check import TAIL, determinism, layout, nan_buf, twice

ROWS, C, PITCH = 37, 24, 32


def _values():
    return torch.randn((ROWS, C), generator=torch.Generator().manual_seed(0)).bfloat16()


def honest(out, run):
    out[:ROWS, :C] = _values()


def unwritten(out, run):
    honest(out, run)
    out[ROWS - 1, C - 1] = float("nan")  # the last owned element never stored


def past_columns(out, run):
    honest(out, run)
    out[5, C] = 1.0  # one element past the call's columns


def into_tail(out, run):
    honest(out, run)
    out[ROWS, 0] = 1.0  # the first row after the output


def one_bit(out, run):
    honest(out, run)
    if run == 1:
        out[3, 7:8].view(torch.int16).bitwise_xor_(1)  # the second run differs in the last bit of one element


def check(kernel):
    calls = []

    def call(b):
        kernel(b["out"], len(calls))
        calls.append(1)
    runs = twice(call, lambda: dict(out=nan_buf((ROWS + TAIL, PITCH), torch.bfloat16, "cpu")))
    return layout(runs[0]["out"], 0, C, "output", rows=ROWS) + determinism(runs, ["out"])


@pytest.mark.parametrize("kernel", [unwritten, past_columns, into_tail, one_bit], ids=lambda k: k.__name__)
def test_check_rejects_fault(kernel):
    assert check(kernel)


def test_check_accepts_honest_kernel():
    assert check(honest) == []
