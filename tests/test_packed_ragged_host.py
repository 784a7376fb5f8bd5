"""Ragged gene counts in the packed formats: io.pack_counts / io.pack_rows(..., pad_genes=True) pack a matrix whose gene
count is not a multiple of 8 as its zero-padded form, byte for byte, from dense and CSR input, in one piece and in row
chunks.  The default still refuses such a matrix."""
import numpy as np
import pytest
import scipy.sparse as sp

from dca_b200 import io as dio

WIDTHS = [4, 8, 16, "sparse", "auto"]
GENES = [1, 7, 9, 87, 89, 20001, 20004, 20007]


def _counts(n, g, seed):
    rng = np.random.default_rng(seed)
    C = rng.negative_binomial(1, 0.4, size=(n, g)).astype(np.float32)
    C[rng.random((n, g)) < 0.7] = 0
    C[rng.random((n, g)) < 0.01] = 40                    # escapes at 4 bits
    C[0, g - 1] = 1e6                                    # escapes at every width, in the last real gene
    C[n // 2, 0] = 70000
    C[n - 1, g // 2] = 300
    return C


def _padded(C):
    gp = (C.shape[1] + 7) // 8 * 8
    out = np.zeros((C.shape[0], gp), dtype=C.dtype)
    out[:, :C.shape[1]] = C
    return out


def _same(a, b):
    assert a.bits == b.bits and a.n_genes == b.n_genes and a.n_genes % 8 == 0
    for k in ("packed", "indptr", "nib_indptr", "nibbles"):
        x, y = getattr(a, k), getattr(b, k)
        if x is None or y is None:
            assert x is None and y is None, k
            continue
        assert x.dtype == y.dtype and np.array_equal(x, y), k
    assert a.entries.tobytes() == b.entries.tobytes()


@pytest.mark.parametrize("bits", WIDTHS)
@pytest.mark.parametrize("G", GENES)
def test_padded_pack_is_the_pack_of_the_zero_padded_matrix(G, bits):
    n = 40 if G > 1000 else 300
    C = _counts(n, G, G)
    ref = dio.pack_counts(_padded(C), bits)
    assert ref.genes == ref.n_genes == (G + 7) // 8 * 8
    for name, pc in (("pack_counts", dio.pack_counts(C, bits, pad_genes=True)),
                     ("pack_rows dense", dio.pack_rows(C, bits, pad_genes=True)),
                     ("pack_rows csr", dio.pack_rows(sp.csr_matrix(C), bits, pad_genes=True)),
                     ("pack_rows csr chunked", dio.pack_rows(sp.csr_matrix(C), bits, chunk_rows=7, pad_genes=True)),
                     ("pack_rows dense chunked", dio.pack_rows(C, bits, chunk_rows=13, pad_genes=True))):
        _same(pc, ref)
        assert pc.genes == G, name
        assert len(pc.entries) > 0, name                 # overflow entries at every width
        U = dio.unpack_counts(pc)
        assert U.shape == (n, pc.n_genes) and np.array_equal(U[:, :G], C), name
        assert not U[:, G:].any(), name                  # the pad columns unpack as zeros


@pytest.mark.parametrize("bits", WIDTHS)
def test_padded_rows_keep_the_gene_count_through_take_concat_and_refit(bits):
    G = 89
    C = _counts(500, G, 3)
    pc = dio.pack_rows(sp.csr_matrix(C), bits, chunk_rows=64, pad_genes=True)
    w = "sparse" if pc.bits == 1 else pc.bits
    idx = np.random.default_rng(1).permutation(500)[:333]
    sub = pc.take_rows(idx, block=50)
    _same(sub, dio.pack_counts(_padded(C[idx]), w))
    assert sub.genes == G
    whole = dio.concat_packed([pc.take_rows(np.arange(0, 200)), pc.take_rows(np.arange(200, 500))])
    assert whole.genes == G and np.array_equal(dio.unpack_counts(whole)[:, :G], C)
    refit = dio.fit_batches(pc, 64, 1, 1 << 30)          # one overflow entry per batch: repacked at a wider width
    assert refit.genes == G and refit.n_genes == 96 and np.array_equal(dio.unpack_counts(refit)[:, :G], C)
    other = dio.pack_counts(_counts(10, 90, 4), w, pad_genes=True)
    with pytest.raises(ValueError, match="width or gene count"):
        dio.concat_packed([pc.take_rows([0]), other])    # same stored width (96), different gene count


def test_multiples_of_8_are_unchanged_and_the_default_refuses_ragged():
    C = _counts(100, 64, 5)
    for bits in WIDTHS:
        _same(dio.pack_counts(C, bits, pad_genes=True), dio.pack_counts(C, bits))
        assert dio.pack_rows(C, bits, pad_genes=True).genes == 64
    for call in (lambda: dio.pack_counts(_counts(10, 12, 6)), lambda: dio.pack_rows(_counts(10, 12, 6)),
                 lambda: dio.pack_rows(sp.csr_matrix(_counts(10, 12, 6)))):
        with pytest.raises(ValueError, match="multiple of 8"):
            call()


def test_padding_does_not_densify_a_csr_matrix_whole(monkeypatch):
    """pack_rows densifies a CSR matrix chunk by chunk: no dense block larger than one chunk of rows is formed."""
    G, n, chunk = 20001, 64, 16
    C = _counts(n, G, 7)
    seen = []
    orig = dio._zero_padded

    def recording(M, gp):
        seen.append(M.shape[0])
        return orig(M, gp)
    monkeypatch.setattr(dio, "_zero_padded", recording)
    pc = dio.pack_rows(sp.csr_matrix(C), "auto", chunk_rows=chunk, pad_genes=True)
    assert seen and max(seen) <= chunk
    assert np.array_equal(dio.unpack_counts(pc)[:, :G], C)
