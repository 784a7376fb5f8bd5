"""Host-side checks of the packed device mode (packed_data.PackedDeviceDataset): CLI and training_kwds validation, the
library symbols and the dca_packed_counts layout the binding shares with the library -- no GPU needed."""
import ctypes as C
import re

import numpy as np
import pandas as pd
import pytest


def test_cli_flag():
    from dca_b200.__main__ import parse_args
    assert parse_args(["in.tsv", "out"]).packed is False
    a = parse_args(["in.tsv", "out", "--preprocess", "device", "--packed"])
    assert a.packed is True and a.preprocess == "device"


def _tsv(tmp_path):
    Y = np.arange(64 * 6).reshape(64, 6) % 5
    df = pd.DataFrame(Y, index=["g%d" % i for i in range(64)], columns=["c%d" % i for i in range(6)])
    p = tmp_path / "counts.tsv"
    df.to_csv(p, sep="\t")
    return str(p)


def test_cli_validation(tmp_path, monkeypatch):
    from dca_b200 import io
    from dca_b200.__main__ import main
    monkeypatch.setattr(io, "_cuda_available", lambda: False)        # the pandas reader: no device needed here
    inp = _tsv(tmp_path)
    with pytest.raises(ValueError, match="--preprocess device"):
        main([inp, str(tmp_path / "a"), "-e", "1", "--packed"])
    with pytest.raises(ValueError, match="exclude each other"):
        main([inp, str(tmp_path / "b"), "-e", "1", "--preprocess", "device", "--packed", "--stream"])
    genes = tmp_path / "genes.txt"
    genes.write_text("g3\ng10")
    with pytest.raises(NotImplementedError, match="denoisesubset"):
        main([inp, str(tmp_path / "c"), "-e", "1", "--preprocess", "device", "--packed", "--denoisesubset", str(genes)])


def test_training_kwds_validation():
    from dca_b200.anndata_lite import AnnData
    from dca_b200.api import dca
    ad = AnnData(np.ones((10, 8), np.float32))
    with pytest.raises(ValueError, match="'preprocess': 'device'"):
        dca(ad, training_kwds={"packed": True})
    for stream in (True, "auto"):
        with pytest.raises(ValueError, match="exclude each other"):
            dca(ad, training_kwds={"preprocess": "device", "packed": True, "stream": stream})


def test_normalize_and_train_validation():
    from dca_b200 import io
    from dca_b200.anndata_lite import AnnData
    from dca_b200.train import train
    ad = AnnData(np.ones((10, 8), np.float32))
    with pytest.raises(ValueError, match="give device="):
        io.normalize(ad, packed=True)
    with pytest.raises(ValueError, match="not both"):
        io.normalize(ad, packed=True, stream=True, device="cuda:0")
    for other in (dict(stream=True), dict(device_data=object()), dict(stream_data=object())):
        with pytest.raises(ValueError, match="cannot be combined"):
            train(None, None, packed_data=object(), verbose=False, **other)


def test_library_exports_the_packed_entry_points():
    from dca_b200 import _lib
    lib = _lib.load()
    for name in ("dca_pack_count_rows", "dca_pack_rows_device", "dca_expand_rows_exact", "dca_packed_train_step",
                 "dca_packed_eval_step", "dca_packed_predict"):
        assert name in _lib.PROTOTYPES and hasattr(lib, name), name


def test_descriptor_layout_matches_the_library():
    """The library rejects a descriptor whose struct_bytes is not its sizeof(dca_packed_counts), naming the size: the
    ctypes mirror must have the same size."""
    from dca_b200 import _lib
    lib = _lib.load()
    d = _lib.PackedCountsDesc()
    d.struct_bytes = 1
    st = lib.dca_expand_rows_exact(C.byref(d), None, 1, 1.0, 0, None, None, None, None, 0, None, None)
    assert st == -1
    size = int(re.search(r"struct_bytes must be (\d+)", lib.dca_last_error().decode()).group(1))
    assert size == C.sizeof(_lib.PackedCountsDesc) == 72
