"""Row selection and concatenation of packed count matrices (io.PackedCounts.take_rows, io.concat_packed, io.pack_rows)
work on the packed arrays and give the bytes pack_counts writes for the selected / stacked matrix."""
import numpy as np
import pytest
import scipy.sparse as sp

from dca_b200 import io as dio

FORMATS = ["sparse", 4, 8, 16]


def _counts(n, g, seed, big=False):
    rng = np.random.default_rng(seed)
    C = rng.negative_binomial(1, 0.4, size=(n, g)).astype(np.float32)
    C[rng.random((n, g)) < 0.7] = 0
    C[rng.random((n, g)) < 0.01] = 40          # escapes at 4 bits
    if big:
        C[0, 3] = 1e6                          # escapes at every width
        C[n // 2, g - 1] = 70000
    return C


def _same(a, b):
    assert a.bits == b.bits and a.n_genes == b.n_genes
    for k in ("packed", "indptr", "nib_indptr", "nibbles"):
        x, y = getattr(a, k), getattr(b, k)
        if x is None or y is None:
            assert x is None and y is None, k
            continue
        assert x.dtype == y.dtype and np.array_equal(x, y), k
    assert a.entries.tobytes() == b.entries.tobytes()


@pytest.mark.parametrize("bits", FORMATS)
@pytest.mark.parametrize("big", [False, True])
def test_take_rows_is_the_pack_of_the_selected_rows(bits, big):
    C = _counts(300, 64, 1, big)
    pc = dio.pack_counts(C, bits)
    rng = np.random.default_rng(2)
    for idx in (rng.permutation(300), rng.integers(0, 300, 77), np.arange(5, 180), np.array([299])):
        sub = pc.take_rows(idx)
        _same(sub, dio.pack_counts(C[idx], bits))
        assert np.array_equal(dio.unpack_counts(sub), C[idx])
    # in blocks of rows, as for large selections
    idx = rng.permutation(300)
    _same(pc.take_rows(idx, block=37), dio.pack_counts(C[idx], bits))


@pytest.mark.parametrize("bits", FORMATS)
@pytest.mark.parametrize("big", [False, True])
def test_concatenated_chunk_packs_are_the_pack_of_the_whole(bits, big):
    C = _counts(250, 48, 3, big)
    parts = [dio.pack_counts(C[a:b], bits) for a, b in ((0, 1), (1, 100), (100, 107), (107, 250))]
    whole = dio.concat_packed(parts)
    _same(whole, dio.pack_counts(C, bits))
    assert np.array_equal(dio.unpack_counts(whole), C)


@pytest.mark.parametrize("bits", FORMATS + ["auto", "dense"])
def test_csr_packs_to_the_bytes_of_its_dense_form(bits):
    C = _counts(400, 56, 4, True)
    m = sp.csr_matrix(C)
    got = dio.pack_rows(m, bits, batch=32, chunk_rows=64)
    _same(got, dio.pack_counts(C, bits, batch=32))
    _same(dio.pack_rows(C, bits, batch=32, chunk_rows=64), dio.pack_counts(C, bits, batch=32))


def test_concat_rejects_mixed_formats():
    C = _counts(20, 16, 5)
    with pytest.raises(ValueError):
        dio.concat_packed([dio.pack_counts(C, 4), dio.pack_counts(C, 8)])
    with pytest.raises(IndexError):
        dio.pack_counts(C, 4).take_rows([20])


def test_pack_rows_needs_a_multiple_of_8_genes():
    with pytest.raises(ValueError, match="multiple of 8"):
        dio.pack_rows(sp.csr_matrix(np.ones((4, 12))), "auto")


def _deep_counts(n, g, seed):
    """Deep sequencing of few genes: ~6700 counts per cell, 4.5 % of entries >= 15."""
    rng = np.random.default_rng(seed)
    mu = np.exp(rng.normal(0.0, 1.2, size=g))
    mu *= 6400 / mu.sum()
    depth = np.exp(rng.normal(0, 0.3, (n, 1)))
    return rng.negative_binomial(2, 2 / (2 + mu[None, :] * depth), size=(n, g)).astype(np.float32)


def test_fit_batches_widens_a_packing_whose_large_batches_overflow():
    C = _deep_counts(2048, 2000, 7)
    pc = dio.pack_rows(C, "auto", batch=32)
    cap = max(4096, 1024 * 2000 // 32)                   # an engine of max_batch 1024 (engine.cu ovf_cap)
    assert pc.bits == 4 and dio._worst_batch(pc.indptr, 1024) > cap
    assert dio.fit_batches(pc, 32, cap, 1 << 30) is pc   # small batches fit as packed
    wide = dio.fit_batches(pc, 1024, cap, 1 << 30)
    assert wide.bits == 8 and dio._worst_batch(wide.indptr, 1024) <= cap
    _same(wide, dio.pack_counts(C, 8))
