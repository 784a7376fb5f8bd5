"""The head backward as one band-ordered launch (tunable head_bwd_banded = 1, the default) computes the bits of the
two-launch path (head_bwd_banded = 0): the items and their summation orders are the same, only their order in time
differs.  Gene-GEMM mode 3 alone at the edges of the tiling, the benchmark shape and several SM budgets, outputs inside
guard bands; and whole training steps with updates."""
import numpy as np
import pytest
import torch

from oracle import dca_oracle as O
from tests.test_gpu_tc import _gg
from tests.util import synth_counts

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENTINEL = -7777.0


def _set_banded(v):
    from dca_b200 import _lib
    _lib.set_tunable("head_bwd_banded", v)


def _operands(B, G, nh, seed):
    g = torch.Generator(device=DEV); g.manual_seed(seed)
    Z = [(torch.randn(B, G, device=DEV, generator=g) * 1e-3).to(torch.bfloat16) for _ in range(nh)]
    H = torch.relu(torch.randn(B, 64, device=DEV, generator=g)).to(torch.bfloat16)
    W = (torch.randn(nh, 64, G, device=DEV, generator=g) * 0.2).to(torch.bfloat16).contiguous()
    return Z, H, W


def _run(ops, B, G, nh, banded, sm_count):
    """Mode 3 with every output inside a sentinel-filled buffer: dH with 3 guard rows, the Keras [64 x G] head
    gradients with ld = G + 8 and 2 guard rows, db with 8 guard elements."""
    Z, H, W = ops
    out = torch.full((B + 3, 64), SENTINEL, device=DEV); out[:B] = 0.0
    dWs, dbs = [], []
    for _ in range(nh):
        dW = torch.full((64 + 2, G + 8), SENTINEL, device=DEV); dW[:64, :G] = 0.0
        db = torch.full((G + 8,), SENTINEL, device=DEV); db[:G] = 0.0
        dWs.append(dW); dbs.append(db)
    _set_banded(banded)
    try:
        _gg(3, Z, H, W, B, G, nh, out_b=out, dW=dWs, dW_ld=G + 8, transposed=1, db=dbs, sm_count=sm_count)
    finally:
        _set_banded(1)
    return [out] + dWs + dbs


@pytest.mark.parametrize("sm_count", [1, 7, 100, 0])
@pytest.mark.parametrize("B,G,nh", [(4096, 20000, 3), (1100, 2000, 3), (4096, 20000, 1), (129, 72, 3), (1, 8, 3)])
def test_banded_launch_is_bit_identical_to_two_launches(B, G, nh, sm_count):
    if sm_count == 1 and B * G > 10 ** 7:
        pytest.skip("one CTA over the benchmark shape: covered by the smaller shapes")
    ops = _operands(B, G, nh, seed=B + G + nh)
    two = _run(ops, B, G, nh, 0, sm_count)
    band = _run(ops, B, G, nh, 1, sm_count)
    out = band[0]
    assert (out[B:] == SENTINEL).all(), "dH rows past B written"
    assert torch.isfinite(out[:B]).all()
    for i in range(nh):
        dW, db = band[1 + i], band[1 + nh + i]
        guard = torch.ones_like(dW, dtype=torch.bool); guard[:64, :G] = False
        assert (dW[guard] == SENTINEL).all(), "dW head %d written outside [64 x G]" % i
        assert (db[G:] == SENTINEL).all(), "db head %d written past G" % i
    for k, (a, b) in enumerate(zip(two, band)):
        assert torch.equal(a, b), ("output", k)


def test_training_steps_are_bit_identical_with_and_without_banding():
    """Two engines, one built with each head-backward path (a captured step keeps the path it was recorded with): five
    steps with updates give the same loss, gradients, parameters and BatchNorm state bit for bit."""
    from dca_b200.engine import DeviceEngine
    N, G, B = 1100, 2000, 1024
    Y = synth_counts(N, G, 7); X, sf = O.normalize_inputs(Y)
    rows = torch.as_tensor(np.random.default_rng(1).permutation(N)[:B].astype(np.int32)).to(DEV)
    Xd, Yd, sfd = (torch.as_tensor(a).to(DEV) for a in (X, Y, sf))
    engines = []
    try:
        for banded in (0, 1):
            _set_banded(banded)
            e = DeviceEngine(G, G, (64, 32, 64), "zinb-conddisp", max_batch=B, seed=3, gemm_path="tcgen05")
            for step in range(5):
                e.train_step(Xd, Yd, sfd, rows=rows)
                e.apply_update(1e-3, 5.0)
            torch.cuda.synchronize()
            engines.append(e)
    finally:
        _set_banded(1)
    a, b = engines
    assert a.read_loss() == b.read_loss()
    assert torch.equal(a.grads, b.grads)
    assert torch.equal(a.params, b.params)
    assert torch.equal(a.bn_state, b.bn_state)
