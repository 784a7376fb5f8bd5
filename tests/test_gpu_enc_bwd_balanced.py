"""The encoder backward's weight gradient (K5, gene-GEMM mode 2: dW1 += X[rows]^T . dA1) in 64-gene blocks spread over
the SMs.  Each dW1 element is one warpgroup's wgmma chain over the cells in order, added to dW1 once, whatever the SM
budget, so the bits cannot depend on it; against float64 the result is within fp32 accumulation noise."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PAD = 8                                 # X stored with ld = G + 8, NaN in the padding columns
EXTRA_ROWS = 53                         # X holds more rows than the batch
SHAPES = [(B, G) for G in (72, 20000) for B in (1, 129, 4096, 8192)]


def _L():
    from dca_b200 import _lib
    return _lib


_SRC = {}


def _source(B, G):
    """X [(B + EXTRA_ROWS) x (G + PAD)] bf16 with NaN padding, dA1 [B x 64] bf16, batch rows (a permutation)."""
    if (B, G) not in _SRC:
        _SRC.clear()
        g = torch.Generator(device=DEV); g.manual_seed(B * 3 + G)
        n = B + EXTRA_ROWS
        X = torch.randn((n, G + PAD), generator=g, device=DEV).to(torch.bfloat16)
        X[:, G:] = float("nan")
        dA = (torch.randn((B, 64), generator=g, device=DEV) * 1e-3).to(torch.bfloat16)
        rows = torch.randperm(n, generator=g, device=DEV)[:B].to(torch.int32).contiguous()
        _SRC[(B, G)] = (X, dA, rows)
    return _SRC[(B, G)]


def _k5(Z, ldz, rows, B, G, dA, sms, dW0=None, transposed=False):
    """dW (+)= Z[rows]^T . dA by dca_tc_gene_gemm_rows mode 2 (rows None: Z's first B rows) on at most sms SMs."""
    L = _L(); lib = L.load()
    if transposed:
        dW = torch.zeros((64, G), device=DEV) if dW0 is None else dW0.t().contiguous()
    else:
        dW = torch.zeros((G, 64), device=DEV) if dW0 is None else dW0.clone()
    L.check(lib.dca_tc_gene_gemm_rows(2, Z.data_ptr(), None, None, ldz, None if rows is None else rows.data_ptr(), B, G,
                                      1, dA.data_ptr(), None, None, dW.data_ptr(), None, None, G if transposed else 64,
                                      int(transposed), None, None, None, None, sms), "dca_tc_gene_gemm_rows")
    torch.cuda.synchronize()
    return dW.t() if transposed else dW


@pytest.mark.parametrize("B,G", SHAPES)
def test_dw_bits_independent_of_sm_budget(B, G):
    """The same inputs on 1, 7, 64, 131 and 132 SMs (the CTAs then own runs of very different length): the same bits."""
    X, dA, rows = _source(B, G)
    dW0 = torch.randn((G, 64), generator=torch.Generator(device=DEV).manual_seed(G), device=DEV)
    ref = _k5(X, G + PAD, rows, B, G, dA, 132, dW0)
    assert torch.isfinite(ref).all()
    for sms in (1, 7, 64, 131):
        assert torch.equal(_k5(X, G + PAD, rows, B, G, dA, sms, dW0), ref), sms


@pytest.mark.parametrize("B,G", SHAPES)
def test_dw_rows_equal_contiguous_copy(B, G):
    """Rows read in place (cp.async) and the gathered contiguous batch (TMA boxes): bit-identical, on the full budget
    and on 7 SMs."""
    X, dA, rows = _source(B, G)
    Xg = X[rows.long(), :G].contiguous()
    for sms in (0, 7):
        assert torch.equal(_k5(X, G + PAD, rows, B, G, dA, sms), _k5(Xg, G, None, B, G, dA, sms)), sms


@pytest.mark.parametrize("B,G", SHAPES)
def test_dw_matches_float64(B, G):
    """Against X[rows]^T . dA1 in float64 of the same bf16 operands, added to a non-zero dW once: within fp32
    accumulation noise of the sum of |products| (bf16 rounding of the operands is not involved)."""
    X, dA, rows = _source(B, G)
    dW0 = torch.randn((G, 64), generator=torch.Generator(device=DEV).manual_seed(G + 1), device=DEV) * 1e-3
    got = _k5(X, G + PAD, rows, B, G, dA, 0, dW0).double()
    Xr = X[rows.long(), :G].double()
    ref = dW0.double() + Xr.t() @ dA.double()
    scale = Xr.abs().t() @ dA.double().abs() + dW0.double().abs()
    err = (got - ref).abs()
    assert torch.isfinite(got).all()
    assert (err <= 2e-6 * np.sqrt(max(B, 1)) * scale + 1e-30).all(), float((err / (scale + 1e-30)).max())


@pytest.mark.parametrize("G", [72, 20000])
def test_dw_transposed_layout_same_bits(G):
    """dW in Keras [64 x G] layout (staging tile transposed): the same bits as the [G x 64] layout."""
    B = 129
    X, dA, rows = _source(B, G)
    dW0 = torch.randn((G, 64), generator=torch.Generator(device=DEV).manual_seed(5), device=DEV)
    a = _k5(X, G + PAD, rows, B, G, dA, 0, dW0)
    b = _k5(X, G + PAD, rows, B, G, dA, 0, dW0, transposed=True)
    assert torch.equal(a, b)
