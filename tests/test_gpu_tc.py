"""wgmma kernels against same-rounding references (bf16-rounded operands, fp32/fp64 accumulate)."""
import ctypes as C
import numpy as np
import pytest
import torch

from oracle import dca_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _L():
    from dca_b200 import _lib
    return _lib


def _bf(a):
    return torch.as_tensor(np.ascontiguousarray(a)).to(DEV, torch.bfloat16).contiguous()


@pytest.mark.parametrize("a_mn,b_mn", [(0, 0), (1, 0), (0, 1), (1, 1)])
@pytest.mark.parametrize("N,K", [(64, 64), (256, 64), (64, 128), (128, 256)])
def test_tc_probe_operand_layouts(a_mn, b_mn, N, K):
    """D = A.B for every (K-major | MN-major) operand combination the Dense kernels rely on (wgmma descriptors)."""
    L = _L(); lib = L.load()
    M = 128
    rng = np.random.default_rng(N * 7 + K + a_mn * 2 + b_mn)
    A = rng.normal(0, 1, (M, K)).astype(np.float32)
    B = rng.normal(0, 1, (K, N)).astype(np.float32)
    Ab, Bb = _bf(A), _bf(B)
    ref = (Ab.double() @ Bb.double()).cpu().numpy()
    a_store = Ab.t().contiguous() if a_mn else Ab             # MN-major: stored [K x M]
    b_store = Bb.contiguous() if b_mn else Bb.t().contiguous()  # K-major B: stored [N x K]; MN-major: [K x N]
    D = torch.full((M, N), float("nan"), device=DEV)
    def run(al, asb, bl, bsb):
        D.fill_(float("nan"))
        st = lib.dca_tc_probe(a_store.data_ptr(), a_store.shape[0], a_store.shape[1], b_store.data_ptr(), b_store.shape[0],
                              b_store.shape[1], a_mn, b_mn, M, N, K, al, asb, bl, bsb, D.data_ptr(), None)
        L.check(st, "dca_tc_probe")
        torch.cuda.synchronize()
        got = D.cpu().numpy()
        return float(np.nanmax(np.abs(got - ref)) / np.max(np.abs(ref))) if np.isfinite(got).all() else float("inf")

    err = run(-1, -1, -1, -1)
    if not err < 1e-5:
        # diagnose: which (LBO, SBO) convention would have worked for the MN-major operands?
        notes = []
        for al, asb in ((-1, -1), (1024, K * 128), (K * 128, 1024), (0, 1024), (1024, 1024)):
            for bl, bsb in ((-1, -1), (1024, K * 128), (K * 128, 1024), (0, 1024), (1024, 1024)):
                e = run(al, asb, bl, bsb)
                if e < 1e-5:
                    notes.append("a(lbo,sbo)=(%d,%d) b(lbo,sbo)=(%d,%d)" % (al, asb, bl, bsb))
        pytest.fail("a_mn=%d b_mn=%d N=%d K=%d rel err %.3g; working overrides: %s" % (a_mn, b_mn, N, K, err, notes))


@pytest.mark.parametrize("B,G,nh", [(128, 256, 3), (4096, 2000, 3), (300, 1000, 2), (77, 200, 1)])
def test_tc_heads_fwd(B, G, nh):
    L = _L(); lib = L.load()
    rng = np.random.default_rng(B + G)
    H = np.maximum(rng.normal(0, 1, (B, 64)), 0).astype(np.float32)
    W = [rng.normal(0, 0.25, (64, G)).astype(np.float32) for _ in range(nh)]
    b = [rng.normal(0, 0.5, G).astype(np.float32) for _ in range(nh)]
    sf = np.exp(rng.normal(0, 0.3, B)).astype(np.float32)
    kinds = [2, 3, 4][:nh] if nh == 3 else ([2, 4] if nh == 2 else [2])
    Hb = _bf(H)
    Wk = torch.stack([_bf(w) for w in W], 0).contiguous()                      # [nh][64][G], Keras layout
    bias = torch.as_tensor(np.concatenate(b)).to(DEV)
    sfd = torch.as_tensor(sf).to(DEV)
    outs = [torch.full((B, G), float("nan"), device=DEV) for _ in range(3)]
    karr = (C.c_int32 * 3)(*(kinds + [0] * (3 - nh)))
    st = lib.dca_tc_heads_fwd(Hb.data_ptr(), B, Wk.data_ptr(), bias.data_ptr(), G, nh, C.byref(karr), sfd.data_ptr(),
                              outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(), G, None)
    L.check(st, "dca_tc_heads_fwd")
    torch.cuda.synchronize()
    Hd = Hb.double().cpu().numpy()
    for i, kind in enumerate(kinds):
        Wd = Wk[i].double().cpu().numpy()
        z = Hd @ Wd + b[i]
        ref = {2: lambda z: O.mean_act(z) * sf[:, None], 3: O.disp_act, 4: O.sigmoid}[kind](z)
        got = outs[i].cpu().numpy()
        assert np.all(np.isfinite(got)), "head %d has non-finite / unwritten outputs" % i
        np.testing.assert_allclose(got, ref, rtol=3e-5, atol=1e-7, err_msg="head kind %d" % kind)


def _gg(mode, Z, H, W, B, G, nh, out_b=None, dW=None, dW_ld=0, transposed=0, db=None, sm_count=None):
    """dca_tc_gene_gemm, or dca_tc_gene_gemm_sms when an SM budget is given (0: the device's SM count)."""
    L = _L(); lib = L.load()
    z = [Z[i].data_ptr() if i < nh else None for i in range(3)]
    dWp = [dW[i].data_ptr() if (dW is not None and i < nh) else None for i in range(3)]
    dbp = [db[i].data_ptr() if (db is not None and i < nh) else None for i in range(3)]
    args = (mode, z[0], z[1], z[2], Z[0].stride(0), B, G, nh, None if H is None else H.data_ptr(),
            None if W is None else W.data_ptr(), None if out_b is None else out_b.data_ptr(),
            dWp[0], dWp[1], dWp[2], dW_ld, transposed, dbp[0], dbp[1], dbp[2], None)
    st = lib.dca_tc_gene_gemm(*args) if sm_count is None else lib.dca_tc_gene_gemm_sms(*args, sm_count)
    L.check(st, "dca_tc_gene_gemm")
    torch.cuda.synchronize()


@pytest.mark.parametrize("B,G", [(128, 128), (4096, 2000), (300, 1000), (77, 264)])
def test_tc_encoder_forward_mode1(B, G):
    """K1: A1 += X . W1 (bf16 operands), output pre-filled with the bias."""
    rng = np.random.default_rng(B * 3 + G)
    X = _bf(rng.normal(0, 1, (B, G)))
    W1 = rng.normal(0, 0.05, (G, 64)).astype(np.float32)
    W1b = _bf(W1)                                         # [G x 64], Keras layout (MN-major B operand)
    bias = rng.normal(0, 0.3, 64).astype(np.float32)
    out = torch.as_tensor(np.tile(bias, (B, 1))).to(DEV).contiguous()
    _gg(1, [X], None, W1b, B, G, 1, out_b=out)
    ref = X.double().cpu().numpy() @ W1b.double().cpu().numpy() + bias
    np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=2e-5, atol=2e-5)


@pytest.mark.parametrize("B,G", [(128, 128), (4096, 2000), (300, 1000), (77, 264)])
def test_tc_encoder_backward_mode2(B, G):
    """K5: dW1[G x 64] += X^T . dA1."""
    rng = np.random.default_rng(B * 5 + G)
    X = _bf(rng.normal(0, 1, (B, G)))
    dA = _bf(rng.normal(0, 1e-3, (B, 64)))
    dW = torch.zeros((G, 64), device=DEV)
    _gg(2, [X], dA, None, B, G, 1, dW=[dW], dW_ld=64, transposed=0)
    ref = X.double().cpu().numpy().T @ dA.double().cpu().numpy()
    assert np.max(np.abs(dW.cpu().numpy() - ref)) < 2e-5 * np.max(np.abs(ref)) + 1e-12


@pytest.mark.parametrize("B,G,nh", [(128, 128, 1), (4096, 2000, 3), (300, 1000, 2), (77, 264, 3)])
def test_tc_head_backward_mode3(B, G, nh):
    """K4: dWh (Keras [64 x G]) += H^T . dZ, dH += dZ . Wh^T, db = colsum(dZ), one pass over dZ."""
    rng = np.random.default_rng(B * 7 + G + nh)
    dZ = [_bf(rng.normal(0, 1e-3, (B, G))) for _ in range(nh)]
    H = _bf(np.maximum(rng.normal(0, 1, (B, 64)), 0))
    Wk = [rng.normal(0, 0.2, (64, G)).astype(np.float32) for _ in range(nh)]
    Wp = torch.stack([_bf(w) for w in Wk], 0).contiguous()   # [nh][64][G]
    dH = torch.zeros((B, 64), device=DEV)
    dW = [torch.zeros((64, G), device=DEV) for _ in range(nh)]
    db = [torch.zeros(G, device=DEV) for _ in range(nh)]
    _gg(3, dZ, H, Wp, B, G, nh, out_b=dH, dW=dW, dW_ld=G, transposed=1, db=db)
    Hd = H.double().cpu().numpy(); Wd = np.concatenate([Wp[i].double().cpu().numpy() for i in range(nh)], 1)
    ref_dH = np.zeros((B, 64))
    for i in range(nh):
        z = dZ[i].double().cpu().numpy()
        ref_dH += z @ Wd[:, i * G:(i + 1) * G].T
        ref_dW = Hd.T @ z
        assert np.max(np.abs(dW[i].cpu().numpy() - ref_dW)) < 3e-5 * np.max(np.abs(ref_dW)) + 1e-12, "dW head %d" % i
        ref_db = z.sum(0)
        assert np.max(np.abs(db[i].cpu().numpy() - ref_db)) < 3e-5 * np.max(np.abs(ref_db)) + 1e-9, "db head %d" % i
    assert np.max(np.abs(dH.cpu().numpy() - ref_dH)) < 3e-5 * np.max(np.abs(ref_dH)) + 1e-12


# ---------------------------------------------------------------------------------------------------------------------
# Shapes at the edges of the tiling, outputs inside guard bands, padded inputs, and a grid smaller than the item count.
_SENTINEL = -7777.0           # every element outside the logical output must still hold this after the call


def _gg_operands(mode, B, G, nh, seed):
    """Seeded bf16 operands of one gene-GEMM mode and their float64 references."""
    rng = np.random.default_rng(seed)
    ops = {"mode": mode, "B": B, "G": G, "nh": nh}
    if mode == 1:
        ops["Z"] = [_bf(rng.normal(0, 1, (B, G)))]
        ops["W"] = _bf(rng.normal(0, 0.05, (G, 64)))
        ops["bias"] = rng.normal(0, 0.3, 64).astype(np.float32)
        ops["H"] = None
        ops["ref_out"] = ops["Z"][0].double().cpu().numpy() @ ops["W"].double().cpu().numpy() + ops["bias"]
    elif mode == 2:
        ops["Z"] = [_bf(rng.normal(0, 1, (B, G)))]
        ops["H"] = _bf(rng.normal(0, 1e-3, (B, 64)))
        ops["W"] = None
        ops["ref_dW"] = [ops["Z"][0].double().cpu().numpy().T @ ops["H"].double().cpu().numpy()]
    else:
        ops["Z"] = [_bf(rng.normal(0, 1e-3, (B, G))) for _ in range(nh)]
        ops["H"] = _bf(np.maximum(rng.normal(0, 1, (B, 64)), 0))
        ops["W"] = torch.stack([_bf(rng.normal(0, 0.2, (64, G))) for _ in range(nh)], 0).contiguous()   # [nh][64][G]
        Hd = ops["H"].double().cpu().numpy()
        zs = [z.double().cpu().numpy() for z in ops["Z"]]
        ops["ref_out"] = sum(z @ ops["W"][i].double().cpu().numpy().T for i, z in enumerate(zs))
        ops["ref_dW"] = [Hd.T @ z for z in zs]
        ops["ref_db"] = [z.sum(0) for z in zs]
    return ops


def _gg_run(ops, sm_count=None, pad_z=False):
    """One call with every output inside a larger sentinel-filled buffer: [B x 64] outputs get 3 guard rows, the
    [G x 64] encoder gradient 8 guard rows, the Keras [64 x G] head gradients ld = G + 8 and 2 guard rows, db 8 guard
    elements.  pad_z: Z is stored with ldz = G + 8 and NaN in the padding columns."""
    mode, B, G, nh = ops["mode"], ops["B"], ops["G"], ops["nh"]
    Z = ops["Z"]
    if pad_z:
        Zp = []
        for z in Z:
            buf = torch.full((B, G + 8), float("nan"), device=DEV, dtype=torch.bfloat16)
            buf[:, :G] = z
            Zp.append(buf)
        Z = Zp
    res = {"out": None, "dW": None, "db": None}
    kw = {}
    if mode in (1, 3):
        out = torch.full((B + 3, 64), _SENTINEL, device=DEV)
        out[:B] = torch.as_tensor(np.tile(ops["bias"], (B, 1))).to(DEV) if mode == 1 else 0.0
        res["out"] = out; kw["out_b"] = out
    if mode == 2:
        dW = torch.full((G + 8, 64), _SENTINEL, device=DEV); dW[:G] = 0.0
        res["dW"] = [dW]; kw.update(dW=[dW], dW_ld=64, transposed=0)
    if mode == 3:
        dWs, dbs = [], []
        for _ in range(nh):
            dW = torch.full((64 + 2, G + 8), _SENTINEL, device=DEV); dW[:64, :G] = 0.0
            db = torch.full((G + 8,), _SENTINEL, device=DEV); db[:G] = 0.0
            dWs.append(dW); dbs.append(db)
        res["dW"], res["db"] = dWs, dbs
        kw.update(dW=dWs, dW_ld=G + 8, transposed=1, db=dbs)
    _gg(mode, Z, ops["H"], ops["W"], B, G, nh, sm_count=sm_count, **kw)
    return res


def _gg_check(ops, res):
    """Logical outputs against the float64 references (the bounds of the tests above); guard bands untouched.
    Returns the worst relative error."""
    mode, B, G = ops["mode"], ops["B"], ops["G"]
    worst = 0.0

    def rel(got, ref):
        return float(np.max(np.abs(got - ref)) / (np.max(np.abs(ref)) + 1e-30))
    if res["out"] is not None:
        out = res["out"].cpu().numpy()
        assert np.all(out[B:] == _SENTINEL), "rows past B written"
        e = rel(out[:B], ops["ref_out"]); worst = max(worst, e)
        assert e < (2e-5 if mode == 1 else 3e-5), ("out", e)
    for i, dW in enumerate(res["dW"] or []):
        dW = dW.cpu().numpy()
        if mode == 2:
            assert np.all(dW[G:] == _SENTINEL), "dW rows past G written"
            e = rel(dW[:G], ops["ref_dW"][i])
        else:
            guard = np.ones(dW.shape, bool); guard[:64, :G] = False
            assert np.all(dW[guard] == _SENTINEL), "dW head %d written outside [64 x G]" % i
            e = rel(dW[:64, :G], ops["ref_dW"][i])
        worst = max(worst, e)
        assert e < (2e-5 if mode == 2 else 3e-5), ("dW", i, e)
    for i, db in enumerate(res["db"] or []):
        db = db.cpu().numpy()
        assert np.all(db[G:] == _SENTINEL), "db head %d written past G" % i
        e = rel(db[:G], ops["ref_db"][i]); worst = max(worst, e)
        assert e < 3e-5, ("db", i, e)
    return worst


def _gg_tensors(res):
    return [t for k in ("out", "dW", "db") for t in ([res[k]] if k == "out" else (res[k] or [])) if t is not None]


@pytest.mark.parametrize("B,G", [(1, 8), (1, 56), (1, 72), (129, 8), (129, 56), (129, 72)])
@pytest.mark.parametrize("mode", [1, 2, 3])
def test_gene_gemm_edge_shapes_guard_bands_and_padded_z(mode, B, G):
    """Fewer genes than one 64-wide TMA box (G = 8, 56), one full box plus a partial one (72), a single cell and one
    cell past a block (129): every mode against float64, nothing written outside the logical outputs, and Z stored
    with ldz = G + 8 and NaN padding gives the same bits as the contiguous Z (the padding is never read)."""
    ops = _gg_operands(mode, B, G, 3 if mode == 3 else 1, seed=B * 100 + G + mode)
    dense = _gg_run(ops)
    padded = _gg_run(ops, pad_z=True)
    _gg_check(ops, dense)
    _gg_check(ops, padded)
    for a, b in zip(_gg_tensors(dense), _gg_tensors(padded)):
        assert torch.isfinite(b).all()
        assert torch.equal(a, b)


@pytest.mark.parametrize("mode", [1, 2, 3])
def test_gene_gemm_sm_budget(mode):
    """A grid capped at 1 and 7 CTAs (each CTA then strides over many items, continuing its pipeline stage and mbarrier
    phase from one item to the next) against the full device: every output within the float64 bounds, and the weight /
    bias gradients -- each element owned by one item that spans all cells -- bit-identical whatever the grid.  The
    encoder-forward and dH3 products may round differently: the number of partial slots follows the grid."""
    B, G = 1100, 2000
    ops = _gg_operands(mode, B, G, 3 if mode == 3 else 1, seed=17 + mode)
    runs = {sm: _gg_run(ops, sm_count=sm) for sm in (1, 7, 0)}
    worst = {sm: _gg_check(ops, r) for sm, r in runs.items()}
    print("\n[gene gemm mode %d, B=%d G=%d] worst rel err by sm_count (0 = device): %s" % (mode, B, G, worst))
    for sm in (1, 7):
        for k in ("dW", "db"):
            for a, b in zip(runs[sm][k] or [], runs[0][k] or []):
                assert torch.equal(a, b), (sm, k)


@pytest.mark.parametrize("B,G", [(1, 8), (1, 56), (1, 72), (129, 8), (129, 56), (129, 72)])
def test_tc_heads_fwd_edge_shapes_and_guard_bands(B, G):
    """Heads forward at partial gene and cell tiles, outputs with ld_out = G + 8 and 3 guard rows: the logical
    [B x G] block against float64, every other element still the sentinel."""
    L = _L(); lib = L.load()
    rng = np.random.default_rng(B * 7 + G)
    Hb = _bf(np.maximum(rng.normal(0, 1, (B, 64)), 0))
    Wk = torch.stack([_bf(rng.normal(0, 0.25, (64, G))) for _ in range(3)], 0).contiguous()
    b = [rng.normal(0, 0.5, G).astype(np.float32) for _ in range(3)]
    sf = np.exp(rng.normal(0, 0.3, B)).astype(np.float32)
    bias = torch.as_tensor(np.concatenate(b)).to(DEV); sfd = torch.as_tensor(sf).to(DEV)
    outs = [torch.full((B + 3, G + 8), _SENTINEL, device=DEV) for _ in range(3)]
    karr = (C.c_int32 * 3)(2, 3, 4)
    L.check(lib.dca_tc_heads_fwd(Hb.data_ptr(), B, Wk.data_ptr(), bias.data_ptr(), G, 3, C.byref(karr), sfd.data_ptr(),
                                 outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(), G + 8, None), "dca_tc_heads_fwd")
    torch.cuda.synchronize()
    Hd = Hb.double().cpu().numpy()
    for i, act in enumerate((lambda z: O.mean_act(z) * sf[:, None], O.disp_act, O.sigmoid)):
        got = outs[i].cpu().numpy()
        guard = np.ones(got.shape, bool); guard[:B, :G] = False
        assert np.all(got[guard] == _SENTINEL), "head %d written outside [B x G]" % i
        ref = act(Hd @ Wk[i].double().cpu().numpy() + b[i])
        np.testing.assert_allclose(got[:B, :G], ref, rtol=3e-5, atol=1e-7, err_msg="head %d" % i)
