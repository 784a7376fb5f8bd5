"""The heads + loss kernel (dca_tc_heads_loss) at the shapes its schedule makes special: four warpgroups per CTA, each
warp walking its 16 rows of a 64-cell block in four 4-row pieces.  Batches whose last block ends inside each piece, gene
counts from one partial 128-gene tile to the benchmark's, fewer units than SMs, CTAs whose unit range spans several gene
tiles.  dZ bit for bit against dca_tc_heads_fwd -> dca_zinb_loss_fwd_bwd, the loss to 1e-6, and three launches with
identical bits."""
import pytest
import torch

from tests.test_gpu_heads_loss import _check

pytestmark = pytest.mark.gpu


def _cta_ranges(B, G):
    """(first, last) gene tile of every CTA's unit range, as the kernel partitions the units."""
    nblk, tiles = -(-B // 64), -(-G // 128)
    units = tiles * nblk
    grid = min(units, torch.cuda.get_device_properties(0).multi_processor_count)
    return [((c * units // grid) // nblk, ((c + 1) * units // grid - 1) // nblk) for c in range(grid)]


def _check_repeat(B, G, gather, use_sf, ridge, seed):
    _, f, loss = _check(B, G, gather, use_sf, ridge, seed)
    dz0 = [t.clone() for t in f.dz]
    for _ in range(2):
        f.loss.zero_()
        f()
        torch.cuda.synchronize()
        assert float(f.loss.item()) == loss
        for a, b in zip(f.dz, dz0):
            assert torch.equal(a, b)


@pytest.mark.parametrize("B,G,gather,use_sf,ridge", [
    (65, 8, False, True, 0.0),          # r = 1: the last block is one row of piece 0
    (67, 136, True, True, 0.0),         # r = 3
    (132, 2000, True, False, 0.01),     # r = 4: piece 0 full, pieces 1-3 empty
    (325, 20000, True, True, 0.0),      # r = 5: one row of piece 1
    (136, 136, False, True, 0.01),      # r = 8: pieces 0 and 1 full
    (138, 2000, True, True, 0.0),       # r = 10: two rows of piece 2
    (1293, 2000, True, True, 0.0),      # r = 13: one row of piece 3
    (283, 8, True, False, 0.0),         # r = 27: warp 1, three rows of piece 2
    (4109, 20000, True, True, 0.0),     # the benchmark's genes, r = 13
    (5, 20000, False, True, 0.02),      # a single partial block
])
def test_pieces_equal_heads_fwd_then_loss(B, G, gather, use_sf, ridge):
    _check_repeat(B, G, gather, use_sf, ridge, seed=B * 7 + G)


def test_fewer_units_than_sms():
    B, G = 64, 1024                     # 8 units: 8 CTAs, one block each, one warpgroup busy per CTA
    assert len(_cta_ranges(B, G)) == 8
    _check_repeat(B, G, True, True, 0.0, seed=5)


@pytest.mark.parametrize("B,G,gather,ridge", [(65, 20000, False, 0.02), (200, 20000, True, 0.0)])
def test_cta_ranges_span_gene_tiles(B, G, gather, ridge):
    """CTAs own more units than a tile has blocks, so they load the weights of a new tile mid-range."""
    assert any(last > first for first, last in _cta_ranges(B, G)), "need CTAs spanning two gene tiles"
    _check_repeat(B, G, gather, True, ridge, seed=B + 3)
