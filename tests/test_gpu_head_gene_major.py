"""The gene-major head products of the heads + loss kernel (wgmma m64n16: A = the head weights MN-major in their Keras
[64 k][genes] layout, B = 16 rows of H3 K-major) against a float64 product, and bit for bit against the cell-major
m64n128 products of the heads forward (A = H3 K-major, B = the weights MN-major).  dZ of the heads + loss kernel is
bit-identical to the heads forward followed by the loss kernel only if the two orientations give the same fp32."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _L():
    from dca_b200 import _lib
    return _lib


def _probe(a_store, b_store, a_mn, b_mn, N, K):
    """D[128 x N] = A . B through dca_tc_probe (default descriptor conventions)."""
    L = _L(); lib = L.load()
    D = torch.full((128, N), float("nan"), device=DEV)
    L.check(lib.dca_tc_probe(a_store.data_ptr(), a_store.shape[0], a_store.shape[1], b_store.data_ptr(), b_store.shape[0],
                             b_store.shape[1], a_mn, b_mn, 128, N, K, -1, -1, -1, -1, D.data_ptr(), None), "dca_tc_probe")
    torch.cuda.synchronize()
    return D


def _operands(K, scale, seed):
    g = torch.Generator(device=DEV); g.manual_seed(seed)
    H = torch.relu(torch.randn(128, K, device=DEV, generator=g))
    W = torch.randn(K, 128, device=DEV, generator=g) * 0.25
    if scale == "wide":                       # exponents spread over ~2^±12: products of very different magnitude cancel
        H = torch.randn(128, K, device=DEV, generator=g) * torch.exp(torch.randn(128, K, device=DEV, generator=g) * 3)
        W = W * torch.exp(torch.randn(K, 128, device=DEV, generator=g) * 3)
    return H.to(torch.bfloat16).contiguous(), W.to(torch.bfloat16).contiguous()      # H: [cells x K], W: [K x genes]


@pytest.mark.parametrize("K", [64, 128])
def test_tc_probe_gene_major_m64n16(K):
    """D[128 genes x 16 cells] = Wᵀ . Hᵀ with A MN-major (two 64-gene boxes) and B K-major (16 rows)."""
    H, W = _operands(K, "unit", seed=K)
    Hp = H[:16].contiguous()
    ref = (W.double().t() @ Hp.double().t()).cpu().numpy()
    got = _probe(W, Hp, 1, 0, 16, K).cpu().numpy()
    assert np.isfinite(got).all()
    err = float(np.max(np.abs(got - ref)) / np.max(np.abs(ref)))
    assert err < 1e-5, err


@pytest.mark.parametrize("scale", ["unit", "wide"])
def test_gene_major_products_equal_cell_major(scale):
    """Every 16-cell piece of a 128-cell block: the m64n16 gene-major products are the transpose of the m64n128
    cell-major products, bit for bit (K = 64, the hidden width of the heads)."""
    H, W = _operands(64, scale, seed=5 if scale == "unit" else 6)
    cell = _probe(H, W, 0, 1, 128, 64)                                   # [128 cells x 128 genes]
    for piece in range(8):
        gene = _probe(W, H[16 * piece:16 * piece + 16].contiguous(), 1, 0, 16, 64)     # [128 genes x 16 cells]
        a = gene.t().contiguous().view(torch.int32)
        b = cell[16 * piece:16 * piece + 16].contiguous().view(torch.int32)
        n_diff = int((a != b).sum().item())
        assert n_diff == 0, "piece %d: %d of 2048 products differ from the cell-major ones" % (piece, n_diff)


@pytest.mark.parametrize("B,G,gather", [
    (80, 136, True),        # r = 16: the last block is one full 16-cell piece, pieces 1-3 skipped
    (81, 2000, False),      # r = 17: one row of piece 1, walked by warp 0
    (112, 8, True),         # r = 48: pieces 0-2 full, piece 3 skipped
    (127, 20000, True),     # r = 63: warp 3 walks three rows of piece 3
])
def test_cell_pieces_equal_heads_fwd_then_loss(B, G, gather):
    """The heads + loss kernel on batches whose last 64-cell block ends at or inside each 16-cell piece: dZ bit for bit
    against the heads forward followed by the loss kernel, the loss to 1e-6, three launches with identical bits."""
    from tests.test_gpu_heads_loss_pieces import _check_repeat
    _check_repeat(B, G, gather, True, 0.0, seed=B * 3 + G)
