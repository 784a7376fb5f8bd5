"""Schedule of the encoder backward's weight-gradient GEMM (gene-GEMM mode 2), no GPU needed: the genes are cut into
64-gene blocks, each owned by exactly one CTA as part of one contiguous run, and the runs are as even as the SM budget
allows.  Each block's dW rows are one warpgroup's chain over all cells, so the schedule decides time only, not bits."""
import ctypes as C
import math

import numpy as np
import pytest


def schedule(G, sm):
    """first[ctas + 1]: CTA c owns the 64-gene blocks first[c] .. first[c + 1] - 1"""
    from dca_b200 import _lib
    lib = _lib.load()
    ctas = C.c_int32()
    _lib.check(lib.dca_enc_bwd_schedule(G, sm, None, 0, C.byref(ctas)), "dca_enc_bwd_schedule")
    first = np.full(ctas.value + 1, -1, np.int32)
    _lib.check(lib.dca_enc_bwd_schedule(G, sm, first.ctypes.data, first.size, C.byref(ctas)), "dca_enc_bwd_schedule")
    return first


@pytest.mark.parametrize("sm", [1, 7, 64, 128, 132, 400])
@pytest.mark.parametrize("G", [8, 64, 72, 2000, 19992, 20000, 20008])
def test_every_block_owned_once_and_runs_balanced(G, sm):
    blocks = -(-G // 64)
    first = schedule(G, sm)
    ctas = first.size - 1
    assert 1 <= ctas <= min(sm, blocks)
    # contiguous runs that tile [0, blocks): every block owned exactly once, every CTA owns at least one
    assert first[0] == 0 and first[-1] == blocks
    runs = np.diff(first)
    assert (runs >= 1).all()
    owner = np.repeat(np.arange(ctas), runs)
    assert owner.size == blocks and (np.bincount(owner, minlength=ctas) == runs).all()
    assert runs.max() <= math.ceil(blocks / ctas)
    assert runs.max() - runs.min() <= 1


def test_flagship_shape_makespan_is_three_blocks():
    """20000 genes = 313 blocks (the last one 32 genes) on 132 SMs: 49 CTAs of 3 blocks and 83 of 2."""
    runs = np.diff(schedule(20000, 132))
    assert runs.size == 132 and runs.max() == 3
    assert (runs == 3).sum() == 49 and (runs == 2).sum() == 83


def test_bad_arguments_are_refused():
    from dca_b200 import _lib
    lib = _lib.load()
    ctas = C.c_int32()
    assert lib.dca_enc_bwd_schedule(0, 132, None, 0, C.byref(ctas)) != 0
    assert lib.dca_enc_bwd_schedule(2000, 0, None, 0, C.byref(ctas)) != 0
