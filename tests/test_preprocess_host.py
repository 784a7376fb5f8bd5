"""Host-side checks of on-device preprocessing (dca_b200/device_data.py): the CLI switch, the NumPy statement of the
device arithmetic against io.normalize, and the absence of a CPU fallback."""
import numpy as np
import pytest

from tests.util import synth_counts


def test_parser_accepts_preprocess_with_host_default():
    from dca_b200.__main__ import parse_args
    assert parse_args(["in.tsv", "out"]).preprocess == "host"
    assert parse_args(["in.tsv", "out", "--preprocess", "device"]).preprocess == "device"
    with pytest.raises(SystemExit):
        parse_args(["in.tsv", "out", "--preprocess", "cpu"])


def _cases():
    yield synth_counts(4096, 2000, 0)
    Y = synth_counts(1024, 20000, 1)
    Y[3, 7] = 1e6
    yield Y


@pytest.mark.parametrize("case", [0, 1])
def test_reference_statement_is_within_bound_of_host_normalize(case):
    from dca_b200 import io
    from dca_b200.anndata_lite import AnnData
    from dca_b200.device_data import normalize_reference
    Y = list(_cases())[case]
    host = io.normalize(AnnData(Y.copy()), filter_min_counts=False)
    ref = normalize_reference(Y)
    assert np.array_equal(np.asarray(host.obs['n_counts']), ref["n_counts"])
    assert np.array_equal(np.asarray(host.obs['size_factors']), ref["size_factors"])
    Xh = np.asarray(host.X)
    bound = 4e-6 * np.maximum(1.0, np.abs(Xh))
    assert np.all(np.abs(ref["X"] - Xh) <= bound), float(np.max(np.abs(ref["X"] - Xh) / np.maximum(1.0, np.abs(Xh))))


def test_reference_statement_edge_cases():
    from dca_b200.device_data import normalize_reference
    Y = synth_counts(1, 37, 2)
    r = normalize_reference(Y)
    assert np.all(r["std"] == 1.0) and np.all(r["X"] == 0.0)          # one cell: std 1, X = l - l
    Y = synth_counts(64, 37, 3)
    Y[:, 5] = 2.0                                                      # a constant gene: std 0 -> 1
    r = normalize_reference(Y, size_factors=False)
    assert r["std"][5] == 1.0 and np.all(r["X"][:, 5] == 0.0)


def test_normalize_on_device_without_gpu_fails_loudly(monkeypatch):
    import torch
    from dca_b200 import io, _lib
    from dca_b200.anndata_lite import AnnData
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    adata = AnnData(synth_counts(32, 16, 4))
    X0 = adata.X.copy()
    with pytest.raises(_lib.DcaError, match="no CPU fallback"):
        io.normalize(adata, device="cuda:0")
    assert np.array_equal(adata.X, X0) and adata.raw is None           # nothing was mutated


def test_entry_points_without_device_return_no_device():
    import ctypes as C
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    from dca_b200 import _lib
    lib = _lib.load()
    ws = C.c_size_t()
    assert lib.dca_preprocess_workspace_bytes(100, 20, C.byref(ws)) == 0 and ws.value > 0
    st = lib.dca_count_totals(C.c_void_p(256), 20, 100, 20, None, None, None, C.c_void_p(256), ws.value, None)
    assert st == -5 and b"no CUDA device" in lib.dca_last_error()


def test_expansion_entry_points_check_arguments_and_need_a_device():
    """dca_expand_packed_counts / dca_expand_sparse_counts: malformed calls are refused before the device is looked
    at (genes % 8, bits, 16-byte alignment, the sparse format's 65536 genes); a well-formed call without a device
    returns DCA_ERR_NO_DEVICE."""
    import ctypes as C
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    from dca_b200 import _lib
    lib = _lib.load()
    p, odd = C.c_void_p(4096), C.c_void_p(4104)          # stand-in device addresses: never dereferenced here

    def packed(bits=4, genes=64, src=p, Y=p, X=p):
        return lib.dca_expand_packed_counts(src, bits, None, None, None, 3, genes, None, None, 1, 1, Y, X, _lib.F32, None, None)

    def sparse(genes=64, src=p, Y=p, X=p):
        return lib.dca_expand_sparse_counts(src, p, p, 32, None, None, None, 3, genes, None, None, 1, 1, Y, X, _lib.BF16, None,
                                            None)
    for bits in (1, 2, 5, 12, 32):
        assert packed(bits=bits) == -1 and b"bits" in lib.dca_last_error()
    for call in (packed, sparse):
        assert call(genes=60) == -1 and b"multiple of 8" in lib.dca_last_error()
        for kw in ({"src": odd}, {"Y": odd}, {"X": odd}):
            assert call(**kw) == -1 and b"aligned" in lib.dca_last_error(), kw
        assert call() == -5 and b"no CUDA device" in lib.dca_last_error()
    assert sparse(genes=65536 + 8) == -3 and b"65536" in lib.dca_last_error()
    assert sparse(genes=65536) == -5
