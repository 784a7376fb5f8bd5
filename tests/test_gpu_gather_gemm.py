"""The encoder GEMMs (K1: encoder forward, K5: encoder backward) reading the batch's rows of a larger bf16 X by index
(dca_tc_gene_gemm_rows) compute the same bits as on the gathered contiguous batch, and so does the whole training step,
which no longer copies the batch out of X."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HIDDEN = (64, 32, 64)
EXTRA_ROWS = 37          # the source X holds more rows than the batch
PAD = 8                  # ...and is stored with ld = G + 8, NaN in the padding columns


def _L():
    from dca_b200 import _lib
    return _lib


_SRC = {}


def _source(B, G):
    """[(B + EXTRA_ROWS) x (G + PAD)] bf16, NaN padding columns (one per shape, reused by the parameter sets)."""
    if (B, G) not in _SRC:
        _SRC.clear()
        g = torch.Generator(device=DEV); g.manual_seed(B * 7 + G)
        X = torch.randn((B + EXTRA_ROWS, G + PAD), generator=g, device=DEV).to(torch.bfloat16)
        X[:, G:] = float("nan")
        H = (torch.randn((B, 64), generator=g, device=DEV) * 1e-3).to(torch.bfloat16)     # dA1 of K5
        W = (torch.randn((G, 64), generator=g, device=DEV) * 0.05).to(torch.bfloat16)     # W1 of K1, Keras [G x 64]
        bias = torch.randn(64, generator=g, device=DEV) * 0.3
        _SRC[(B, G)] = (X, H, W, bias)
    return _SRC[(B, G)]


def _rows(kind, B, n_src, seed):
    rng = np.random.default_rng(seed)
    if kind == "permutation":
        r = rng.permutation(n_src)[:B]
    elif kind == "duplicates":
        r = rng.integers(0, n_src, B)
        r[B // 2:] = r[:B - B // 2]                    # every row of the first half appears again
    elif kind == "reversed":
        r = np.arange(n_src - 1, n_src - 1 - B, -1)
    else:                                               # "ends": the first and the last row of X
        r = rng.integers(0, n_src, B)
        r[0] = n_src - 1
        if B > 1:
            r[-1] = 0
    return torch.as_tensor(r.astype(np.int32)).to(DEV)


def _run(mode, Z, ldz, rows, B, G, H, W, bias, sms):
    """One K1 (mode 1) / K5 (mode 2) call; rows None: dca_tc_gene_gemm_sms on contiguous Z.  Returns the output."""
    L = _L(); lib = L.load()
    out = dW = None
    if mode == 1:
        out = bias.repeat(B, 1).contiguous()
    else:
        dW = torch.zeros((G, 64), device=DEV)
    common = dict(H=None if mode == 1 else H.data_ptr(), W=W.data_ptr() if mode == 1 else None,
                  out=None if out is None else out.data_ptr(), dW=None if dW is None else dW.data_ptr())
    tail = (common["H"], common["W"], common["out"], common["dW"], None, None, 64, 0, None, None, None, None, sms)
    if rows is None:
        st = lib.dca_tc_gene_gemm_sms(mode, Z.data_ptr(), None, None, ldz, B, G, 1, *tail)
    else:
        st = lib.dca_tc_gene_gemm_rows(mode, Z.data_ptr(), None, None, ldz, rows.data_ptr(), B, G, 1, *tail)
    L.check(st, "dca_tc_gene_gemm_rows" if rows is not None else "dca_tc_gene_gemm_sms")
    torch.cuda.synchronize()
    return out if mode == 1 else dW


SHAPES = [(B, G) for B in (1, 129, 4096, 6001) for G in (8, 56, 72, 2000)] + [(4096, 20000)]


@pytest.mark.parametrize("sms", [1, 7, 0], ids=["sm1", "sm7", "all_sms"])
@pytest.mark.parametrize("kind", ["permutation", "duplicates", "reversed", "ends"])
@pytest.mark.parametrize("B,G", SHAPES)
@pytest.mark.parametrize("mode", [1, 2])
def test_gene_gemm_rows_equals_gathered_batch(mode, B, G, kind, sms):
    """K1 (out_b) and K5 (dW1) with the batch named by row index into a padded, taller X against the same product on the
    pre-gathered contiguous X[rows]: bit-identical at every batch / gene remainder and SM budget.  The gathered tile
    rows are copied into shared memory by the threads, so this also pins that they land where the SWIZZLE_128B TMA box
    of the contiguous batch puts them, that genes past G are zeros rather than the NaN padding, and that the rows past
    the batch are zeros (K5 sums over them)."""
    X, H, W, bias = _source(B, G)
    rows = _rows(kind, B, X.shape[0], seed=B + G + mode)
    Xg = X[rows.long(), :G].contiguous()
    ref = _run(mode, Xg, G, None, B, G, H, W, bias, sms)
    got = _run(mode, X, G + PAD, rows, B, G, H, W, bias, sms)
    assert torch.isfinite(got).all()
    assert torch.equal(got, ref)


def test_gene_gemm_rows_rejects_head_backward():
    """Row indices are for the X operand of K1 / K5 only: the head backward (mode 3) refuses them."""
    L = _L(); lib = L.load()
    X, H, W, bias = _source(129, 72)
    rows = _rows("permutation", 129, X.shape[0], seed=3)
    st = lib.dca_tc_gene_gemm_rows(3, X.data_ptr(), None, None, 72 + PAD, rows.data_ptr(), 129, 72, 1, H.data_ptr(),
                                   W.data_ptr(), None, None, None, None, 72, 1, None, None, None, None, 0)
    assert st != 0


# ------------------------------------------------------------------------------------ the training step
def _problem(B, G, n_cells, seed):
    """Counts, size factors and a z-scored log1p X (bf16, stored with ld = G + 8) of n_cells cells; rows: a batch."""
    g = torch.Generator(device=DEV); g.manual_seed(seed)
    lam = torch.exp(torch.randn(G, generator=g, device=DEV) * 1.2 - 1.0)
    Y = torch.poisson(lam.expand(n_cells, G).contiguous(), generator=g)
    Y[torch.arange(n_cells, device=DEV), torch.randint(0, G, (n_cells,), generator=g, device=DEV)] += 1.0
    sf = (Y.sum(1) / Y.sum(1).median()).contiguous()
    lg = torch.log1p(Y / sf[:, None])
    Xf = (lg - lg.mean(0)) / lg.std(0).clamp_min(1e-6)
    Xs = torch.full((n_cells, G + PAD), float("nan"), device=DEV, dtype=torch.bfloat16)
    Xs[:, :G] = Xf.to(torch.bfloat16)
    X = Xs[:, :G]
    rows = torch.as_tensor(np.random.default_rng(seed).permutation(n_cells)[:B].astype(np.int32)).to(DEV)
    return X, Y, sf, rows


def _engine(G, B):
    from dca_b200.engine import DeviceEngine
    return DeviceEngine(G, G, HIDDEN, "zinb-conddisp", True, max_batch=B, x_dtype="bfloat16", device=DEV, seed=5)


def _state(eng):
    return {"loss": eng.read_loss(), "grads": eng.grads.clone(), "bn_state": eng.bn_state.clone()}


def _assert_same(a, b, what):
    assert a["loss"] == b["loss"], (what, a["loss"], b["loss"])
    for k in ("grads", "bn_state", "params"):
        if k in a:
            assert torch.equal(a[k], b[k]), (what, k)


@pytest.mark.parametrize("step", ["whole", "two_phase", "dp_one_rank"])
@pytest.mark.parametrize("B", [300, 4096])
def test_train_step_rows_equals_gathered_batch(B, step):
    """The training step with rows= (K1 / K5 read X in place) against the same engine state fed X[rows], Y[rows],
    sf[rows] with rows=None: loss, gradients, BatchNorm state and the parameters after apply_update bit-identical on the
    direct call, the graph capture and two graph replays (each on a new batch), for the whole step, its two phases and
    the data-parallel step on a one-rank communicator."""
    from dca_b200 import _lib
    G = 2000
    X, Y, sf, _ = _problem(B, G, B + 611, seed=B)
    a, b = _engine(G, B), _engine(G, B)
    if step == "dp_one_rank":
        try:
            a.comm_init(single_rank=True); b.comm_init(single_rank=True)
        except (_lib.DcaError, OSError) as e:
            pytest.skip("no NCCL for the one-rank communicator: %s" % e)
    side = torch.cuda.Stream(DEV)
    rng = np.random.default_rng(B + 1)
    # the gathered batches are fixed buffers, like the caller's X / Y / sf: the graph keys stay the same across steps
    Xg = torch.empty((B, G), dtype=torch.bfloat16, device=DEV); Yg = torch.empty((B, G), device=DEV)
    sfg = torch.empty(B, device=DEV); rows = torch.empty(B, dtype=torch.int32, device=DEV)

    def run(eng, *args, **kw):
        if step == "whole":
            eng.train_step(*args, **kw)
        elif step == "two_phase":
            eng.train_step(*args, phase=1, **kw); eng.train_step(*args, phase=2, **kw)
        else:
            eng.train_step_allreduce(*args, **kw)

    with torch.cuda.stream(side):
        for it in range(4):                         # direct call, graph capture, two replays
            rows.copy_(torch.as_tensor(rng.permutation(X.shape[0])[:B].astype(np.int32)))
            Xg.copy_(X[rows.long()]); Yg.copy_(Y[rows.long()]); sfg.copy_(sf[rows.long()])
            run(a, X, Y, sf, rows=rows)
            run(b, Xg, Yg, sfg)
            side.synchronize()
            sa, sb = _state(a), _state(b)
            _assert_same(sa, sb, "step %d" % it)
            a.apply_update(1e-3, 5.0); b.apply_update(1e-3, 5.0)
            side.synchronize()
            assert torch.equal(a.params, b.params), "parameters after step %d" % it
    assert a.info()["step_graphs"] >= 1 and b.info()["step_graphs"] >= 1
    a.close(); b.close()


def test_step_with_rows_launches_as_many_kernels_as_without():
    """Reading the batch's rows in place: a step with rows= launches no extra copy kernel."""
    from dca_b200.engine import launch_count
    G, B = 2000, 1000
    X, Y, sf, rows = _problem(B, G, B + 200, seed=11)
    Xg, Yg, sfg = X[rows.long()].contiguous(), Y[rows.long()].contiguous(), sf[rows.long()].contiguous()
    eng = _engine(G, B)
    counts = {}
    for name, args, kw in (("rows", (X, Y, sf), {"rows": rows}), ("gathered", (Xg, Yg, sfg), {})):
        eng.train_step(*args, **kw)                 # (first call: one-time initialisation)
        torch.cuda.synchronize()
        n0 = launch_count()
        eng.train_step(*args, **kw)
        torch.cuda.synchronize()
        counts[name] = launch_count() - n0
    eng.close()
    assert counts["rows"] == counts["gathered"], counts
