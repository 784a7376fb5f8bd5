"""Item schedule of the head backward (gene-GEMM mode 3), no GPU needed: the band-ordered launch runs exactly the items
of the two-launch path -- every dW / db element still owned by one item over all cells, the dH partial slots the same
-- so the gradients keep their bits; only the order of the items differs."""
import ctypes as C
from collections import Counter

import numpy as np
import pytest


def schedule(B, G, nh, sm, banded):
    """(items [n x 8] int32: launch, kind, head, gb0, ng, cb0, ncb, slot), grid[2]"""
    from dca_b200 import _lib
    lib = _lib.load()
    n = C.c_int64()
    grid = (C.c_int32 * 2)()
    _lib.check(lib.dca_head_bwd_schedule(B, G, nh, sm, banded, None, 0, C.byref(n), grid), "dca_head_bwd_schedule")
    items = np.zeros((n.value, 8), np.int32)
    _lib.check(lib.dca_head_bwd_schedule(B, G, nh, sm, banded, items.ctypes.data, n.value, C.byref(n), grid),
               "dca_head_bwd_schedule")
    return items, list(grid)


def tiles(row):
    _, _, h, gb0, ng, cb0, ncb, _ = row
    return [(h, gb, cb) for cb in range(cb0, cb0 + ncb) for gb in range(gb0, gb0 + ng)]


SHAPES = [(4096, 20000, 3), (1100, 2000, 3), (4096, 20000, 1), (129, 72, 3), (1, 8, 3), (300, 1000, 2)]


@pytest.mark.parametrize("B,G,nh", SHAPES)
@pytest.mark.parametrize("sm", [1, 7, 100, 132])
def test_banded_schedule_runs_the_two_pass_items(B, G, nh, sm):
    n_cb, n_gb = -(-B // 128), -(-G // 128)
    band, bgrid = schedule(B, G, nh, sm, 1)
    two, tgrid = schedule(B, G, nh, sm, 0)
    assert (band[:, 0] == 0).all() and 1 <= bgrid[0] <= sm and bgrid[1] == 0
    assert 1 <= tgrid[0] <= sm and 1 <= tgrid[1] <= sm
    a, b = band[band[:, 1] == 0], band[band[:, 1] == 1]
    # every (a) item is one gene block over all cells, each (head, gene block) exactly once
    assert (a[:, 4] == 1).all() and (a[:, 5] == 0).all() and (a[:, 6] == n_cb).all() and (a[:, 7] == -1).all()
    assert sorted(map(tuple, a[:, [2, 3]])) == [(h, g) for h in range(nh) for g in range(n_gb)]
    # the (b) items -- gene range, cell block and partial slot -- are exactly the two-pass ones
    b_two = two[two[:, 1] == 1]
    assert sorted(map(tuple, b[:, 2:])) == sorted(map(tuple, b_two[:, 2:]))
    assert len(set(map(tuple, b[:, 2:]))) == len(b)
    # every tile of dZ is read exactly twice, once by each kind, in both schedules
    every = {(h, g, c) for h in range(nh) for g in range(n_gb) for c in range(n_cb)}
    for items in (band, two):
        for kind in (0, 1):
            cnt = Counter(t for r in items[items[:, 1] == kind] for t in tiles(r))
            assert set(cnt) == every and set(cnt.values()) == {1}, kind


def test_banded_order_and_grid_at_the_benchmark_shape():
    """4096 cells x 20000 genes, 3 heads, 132 SMs: 5 gene ranges of 32 gene blocks (15 partial slots), bands of 32 (a)
    and 32 (b) items alternating, and a grid of two whole bands."""
    items, grid = schedule(4096, 20000, 3, 132, 1)
    assert grid[0] == 128 and len(items) == 471 + 480
    first = items[:64]
    assert (first[0::2, 1] == 0).all() and (first[1::2, 1] == 1).all()
    assert list(first[0::2, 3]) == list(range(32)) and list(first[1::2, 5]) == list(range(32))
    assert (first[1::2, 3] == 0).all() and (first[1::2, 4] == 32).all() and (first[1::2, 7] == 0).all()
    assert sorted(set(items[items[:, 1] == 1, 7])) == list(range(15))
    assert list(items[:, 2]) == sorted(items[:, 2])          # head-major
