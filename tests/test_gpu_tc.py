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


def _gg(mode, Z, H, W, B, G, nh, out_b=None, dW=None, dW_ld=0, transposed=0, db=None):
    L = _L(); lib = L.load()
    z = [Z[i].data_ptr() if i < nh else None for i in range(3)]
    dWp = [dW[i].data_ptr() if (dW is not None and i < nh) else None for i in range(3)]
    dbp = [db[i].data_ptr() if (db is not None and i < nh) else None for i in range(3)]
    st = lib.dca_tc_gene_gemm(mode, z[0], z[1], z[2], Z[0].stride(0), B, G, nh, None if H is None else H.data_ptr(),
                              None if W is None else W.data_ptr(), None if out_b is None else out_b.data_ptr(),
                              dWp[0], dWp[1], dWp[2], dW_ld, transposed, dbp[0], dbp[1], dbp[2], None)
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
