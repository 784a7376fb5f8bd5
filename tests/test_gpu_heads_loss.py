"""The heads + loss kernel of the zinb-conddisp tensor-core training step (dca_tc_heads_loss) against the two kernels it
replaces, dca_tc_heads_fwd -> dca_zinb_loss_fwd_bwd with bf16 gradients: dZ bit for bit, the loss to 1e-6."""
import ctypes as C
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
_SENTINEL = -7777.0            # every dZ element outside [B x G] must still hold this after the call


def _L():
    from dca_b200 import _lib
    return _lib


def _inputs(B, G, gather, use_sf, seed, hot_from=None):
    g = torch.Generator(device=DEV); g.manual_seed(seed)
    N = B + 37 if gather else B
    Hb = torch.relu(torch.randn(B, 64, device=DEV, generator=g)).to(torch.bfloat16).contiguous()
    Wk = torch.randn(3, 64, G, device=DEV, generator=g) * 0.25
    bias = torch.randn(3, G, device=DEV, generator=g) * 0.5
    if hot_from is not None:                  # genes past hot_from: activations at and beyond their clip bounds
        Wk[:, :, hot_from:] *= 8.0; bias[:, hot_from:] *= 12.0
    Wk = Wk.to(torch.bfloat16).contiguous(); bias = bias.reshape(-1).contiguous()
    lam = torch._standard_gamma(torch.full((N, G), 0.5, device=DEV), generator=g) * 2.0
    Y = torch.poisson(lam, generator=g)
    Y[torch.rand(N, G, device=DEV, generator=g) < 0.3] = 0
    Y[0, :min(G, 6)] = torch.tensor([0., 17., 40., 1000., 30000., 5.], device=DEV)[:min(G, 6)]
    rows = torch.randperm(N, device=DEV, generator=g)[:B].int().contiguous() if gather else None
    sf = torch.exp(torch.randn(N, device=DEV, generator=g) * 0.3).contiguous() if use_sf else None
    return Hb, Wk, bias, Y.contiguous(), rows, sf


def _ptr(t):
    return None if t is None else t.data_ptr()


def _workspace(lib, B, G):
    nb = C.c_size_t(); assert lib.dca_zinb_loss_workspace_bytes(B, G, C.byref(nb)) == 0
    return torch.zeros(nb.value, dtype=torch.uint8, device=DEV), nb.value


def _reference(lib, L, Hb, Wk, bias, Y, rows, sf, B, G, ridge, inv_n):
    """K2 then K3: the fp32 head outputs and the bf16 gradients and loss of the loss kernel."""
    outs = [torch.empty((B, G), device=DEV) for _ in range(3)]
    karr = (C.c_int32 * 3)(2, 3, 4)
    L.check(lib.dca_tc_heads_fwd(Hb.data_ptr(), B, Wk.data_ptr(), bias.data_ptr(), G, 3, C.byref(karr), None,
                                 outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(), G, None), "dca_tc_heads_fwd")
    dz = [torch.zeros((B, G), dtype=torch.bfloat16, device=DEV) for _ in range(3)]
    loss = torch.zeros(1, dtype=torch.float64, device=DEV)
    ws, nb = _workspace(lib, B, G)
    L.check(lib.dca_zinb_loss_fwd_bwd(Y.data_ptr(), Y.stride(0), _ptr(rows), _ptr(sf), outs[0].data_ptr(),
                                      outs[1].data_ptr(), outs[2].data_ptr(), G, B, G, L.AE_TYPE_IDS["zinb-conddisp"],
                                      ridge, inv_n, dz[0].data_ptr(), dz[1].data_ptr(), dz[2].data_ptr(), L.BF16, None,
                                      loss.data_ptr(), ws.data_ptr(), nb, None), "dca_zinb_loss_fwd_bwd")
    torch.cuda.synchronize()
    return outs, dz, float(loss.item())


class _Fused:
    """dca_tc_heads_loss into sentinel-filled gradients with ld = G + 8 and 3 guard rows."""

    def __init__(self, lib, L, Hb, Wk, bias, Y, rows, sf, B, G, ridge, inv_n):
        self.lib, self.L = lib, L
        self.inputs = (Hb, Wk, bias, Y, rows, sf)            # the kernel reads them through raw pointers
        self.dz = [torch.full((B + 3, G + 8), _SENTINEL, dtype=torch.bfloat16, device=DEV) for _ in range(3)]
        self.loss = torch.zeros(1, dtype=torch.float64, device=DEV)
        self.ws, self.nb = _workspace(lib, B, G)
        self.args = (Hb.data_ptr(), B, Wk.data_ptr(), bias.data_ptr(), G, Y.data_ptr(), Y.stride(0), _ptr(rows), _ptr(sf),
                     ridge, inv_n, self.dz[0].data_ptr(), self.dz[1].data_ptr(), self.dz[2].data_ptr(), G + 8,
                     self.loss.data_ptr(), self.ws.data_ptr(), self.nb)

    def __call__(self, stream=None):
        self.L.check(self.lib.dca_tc_heads_loss(*self.args, stream), "dca_tc_heads_loss")


def _check(B, G, gather, use_sf, ridge, seed, hot_from=None):
    L = _L(); lib = L.load()
    Hb, Wk, bias, Y, rows, sf = _inputs(B, G, gather, use_sf, seed, hot_from)
    inv_n = 1.0 / (B * G)
    outs, ref_dz, ref_loss = _reference(lib, L, Hb, Wk, bias, Y, rows, sf, B, G, ridge, inv_n)
    f = _Fused(lib, L, Hb, Wk, bias, Y, rows, sf, B, G, ridge, inv_n)
    f()
    torch.cuda.synchronize()
    for k, nm in enumerate(("dzm", "dzd", "dzp")):
        got = f.dz[k]
        assert torch.equal(got[:B, :G], ref_dz[k]), (nm, B, G)
        guard = torch.ones(got.shape, dtype=torch.bool, device=DEV); guard[:B, :G] = False
        assert torch.all(got[guard] == _SENTINEL), "%s written outside [B x G]" % nm
    loss = float(f.loss.item())
    assert np.isfinite(loss) and abs(loss - ref_loss) <= 1e-6 * abs(ref_loss), (loss, ref_loss)
    return outs, f, loss


@pytest.mark.parametrize("B,G,gather,use_sf", [
    (4096, 20000, True, True),     # the benchmark's batch shape
    (6001, 2000, True, True),      # a 1-row piece in the last cell block
    (129, 56, False, True),        # partial 128-gene group, 1-row last block
    (1, 8, False, False),
    (1, 72, True, False),
    (4096, 136, True, True),       # one full and one 8-gene group
])
def test_heads_loss_equals_heads_fwd_then_loss(B, G, gather, use_sf):
    _check(B, G, gather, use_sf, 0.0, seed=B + G)


def test_heads_loss_ridge():
    _check(300, 1000, True, True, 0.01, seed=11)


def test_heads_loss_plain_and_general_finishing():
    """Weights of the upper genes scaled so that activations reach the MeanAct / DispAct clip bounds and theta < 1/32:
    the rows x 128-gene groups then take both the plain and the general finishing path, which round differently."""
    B, G = 512, 1000
    outs, _, _ = _check(B, G, True, True, 0.0, seed=3, hot_from=512)
    m, d = outs[0], outs[1]
    assert bool((m <= 1e-5).any()) and bool((m >= 1e6).any()), "MeanAct clip bounds not reached"
    assert bool((d <= 1e-4).any()) and bool((d < 1.0 / 32).any()), "DispAct clip / small theta not reached"
    # the decision unit: one row x 128 aligned genes, plain when every activation is inside its range
    ok = (m > 1e-5) & (m < 1e6) & (d > 0.03125) & (d < 1e4)
    pad = torch.ones((B, 1024), dtype=torch.bool, device=DEV); pad[:, :G] = ok
    plain = pad.view(B, 8, 128).all(dim=2)
    assert bool(plain.any()) and bool((~plain).any()), "need groups on both finishing paths"


def test_heads_loss_direct_graph_replay_agree():
    """Direct call, stream capture, replay: the same loss and gradients bit for bit (fixed-order loss fold)."""
    B, G = 6001, 2000
    _, f, loss0 = _check(B, G, True, True, 0.0, seed=7)
    dz0 = [t.clone() for t in f.dz]
    s = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        f.loss.zero_()
        with torch.cuda.graph(graph, stream=s):
            f(s.cuda_stream)
    graph.replay()
    torch.cuda.synchronize()
    assert float(f.loss.item()) == loss0
    f.loss.zero_()
    for t in f.dz:
        t.fill_(_SENTINEL)
    graph.replay()
    torch.cuda.synchronize()
    assert float(f.loss.item()) == loss0
    for a, b in zip(f.dz, dz0):
        assert torch.equal(a, b)


def test_train_step_runs_heads_loss_kernel():
    """With 16-byte aligned counts the step runs the heads + loss kernel, one launch in place of the heads forward and
    the ring loss kernel.  Counts one float off alignment take the heads forward, the scalar loss kernel and its fold
    kernel: two launches more.  Both steps compute the same loss."""
    from oracle import dca_oracle as O
    from tests.util import synth_counts
    from dca_b200.engine import DeviceEngine, launch_count
    B, G = 256, 1000
    Y = synth_counts(B, G, 4); X, sf = O.normalize_inputs(Y)
    p0 = O.init_params(G, G, (64, 32, 64), "zinb-conddisp", True, seed=4, dtype=np.float32)
    Xd, sfd = torch.from_numpy(X).to(DEV), torch.from_numpy(sf).to(DEV)
    flat = torch.zeros(B * G + 4, device=DEV)
    runs = {}
    for name, off in (("aligned", 0), ("unaligned", 1)):
        Yd = flat[off:off + B * G].view(B, G)
        Yd.copy_(torch.from_numpy(Y))
        eng = DeviceEngine(G, G, (64, 32, 64), "zinb-conddisp", True, max_batch=B, device=torch.device(DEV),
                           gemm_path="tcgen05", seed=None)
        eng.set_weights(p0)
        torch.cuda.synchronize()
        n0 = launch_count()
        eng.train_step(Xd, Yd, sfd)
        torch.cuda.synchronize()
        runs[name] = (launch_count() - n0, eng.grads.clone(), eng.read_loss())
    assert runs["aligned"][0] == runs["unaligned"][0] - 2, (runs["aligned"][0], runs["unaligned"][0])
    assert abs(runs["aligned"][2] - runs["unaligned"][2]) <= 2e-5 * abs(runs["unaligned"][2])
