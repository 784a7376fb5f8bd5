"""The GPU gzip compressor (dca_gzip_device, csrc/deflate.cu) and the gzip-compressed outputs built on it
(write_text_matrix_device(gzip=True), write_predictions / write(gzip=True), the CLI's --gzip): the same bytes as the
CPU encoder, files that decompress to exactly the bytes of the plain writer, and bytes that do not change run to run."""
import ctypes as C
import gzip
import os
import zlib

import numpy as np
import pandas as pd
import pytest
import torch

from tests.test_deflate_host import CASES, fixed6_text, gzip_host
from tests.util import synth_counts

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _device_gzip(data, info=None):
    from dca_b200.io import gzip_device
    return gzip_device(data, DEV, info=info).cpu().numpy().tobytes()


# ------------------------------------------------------------------------------------------------ compressor
@pytest.mark.parametrize("name", sorted(CASES))
def test_device_equals_host(name):
    data = CASES[name]
    info = np.zeros(3, dtype=np.int64)
    gz = _device_gzip(data, info)
    assert gz == gzip_host(data)
    assert gzip.decompress(gz) == data
    assert info[0] == len(gz) and info[1] == -(-len(data) // 32768)
    if name == "random":
        assert info[2] == info[1]


def test_device_equals_host_few_mb():
    rng = np.random.default_rng(11)
    text = fixed6_text(rng.lognormal(-1.0, 2.0, 400000), 2000)
    pi = fixed6_text(rng.beta(0.5, 2.0, 300000), 1000)
    noise = rng.integers(0, 256, 3 << 20, dtype=np.uint8).tobytes()
    for data in (text, pi, noise, text[:1 << 20] + noise[:1 << 20] + pi[:1 << 20]):
        gz = _device_gzip(data)
        assert gz == gzip_host(data)
        assert zlib.decompress(gz, wbits=31) == data
        assert _device_gzip(data) == gz


def test_device_member_past_4gib():
    """A member of 4 GiB + 12345 bytes: 64-bit offsets and ISIZE mod 2^32, decoded by zlib piece by piece."""
    from dca_b200.io import gzip_device
    n = (4 << 30) + 12345
    free = torch.cuda.mem_get_info(DEV)[0]
    if free < 2 * n + (4 << 30):
        pytest.skip("needs about 13 GB of free device memory")
    period = fixed6_text(np.random.default_rng(3).lognormal(-1.0, 2.0, 100003), 1000)
    pat = torch.frombuffer(bytearray(period), dtype=torch.uint8).to(DEV)
    src = pat.repeat(n // pat.numel() + 1)[:n]
    info = np.zeros(3, dtype=np.int64)
    gz = gzip_device(src, info=info)
    del src
    torch.cuda.empty_cache()
    host = gz.cpu().numpy()
    del gz
    assert info[1] == -(-n // 32768)
    assert int.from_bytes(host[-4:].tobytes(), "little") == n % (1 << 32)
    d = zlib.decompressobj(wbits=31)
    got, crc, pos = 0, 0, 0
    step = 64 << 20
    for s in range(0, host.size, step):
        out = d.decompress(host[s:s + step].tobytes())
        while out:
            k = min(len(out), len(period) - pos)
            assert out[:k] == period[pos:pos + k], got
            crc = zlib.crc32(out[:k], crc)
            got += k
            pos = (pos + k) % len(period)
            out = out[k:]
    assert d.eof and got == n
    assert crc == int.from_bytes(host[-8:-4].tobytes(), "little")


# ------------------------------------------------------------------------------------------------ matrix writer
_ODD = ["plain", "tab\there", 'quo"te', "new\nline", "cr\rx", "", "ünï"]


def _names(prefix, n):
    return [_ODD[i] if i < len(_ODD) else "%s%d" % (prefix, i) for i in range(n)]


def _matrix(shape, seed):
    rng = np.random.default_rng(seed)
    m = (rng.standard_normal(shape) * 10.0 ** rng.integers(-8, 9, shape)).astype(np.float32)
    flat = m.ravel()
    flat[::17] = np.nan
    flat[5::23] = np.inf
    flat[7::29] = -np.inf
    flat[9::31] = -0.0
    flat[11::37] = 0.0
    return m


def _gunzip_device(path):
    from dca_b200 import _lib
    lib = _lib.load()
    info = np.zeros(4, dtype=np.int64)
    stream = C.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
    _lib.check(lib.dca_gunzip(os.fsencode(path), 0, stream, None, 0, info.ctypes.data), "dca_gunzip")
    out = torch.empty(max(int(info[0]), 1), dtype=torch.uint8, device=DEV)
    _lib.check(lib.dca_gunzip(os.fsencode(path), 0, stream, C.c_void_p(out.data_ptr()), int(info[0]),
                              info.ctypes.data), "dca_gunzip")
    return out[:int(info[0])].cpu().numpy().tobytes(), int(info[3])


@pytest.mark.parametrize("shape", [(1, 1), (37, 300), (513, 7)])
@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("labels", ["none", "both"])
def test_matrix_writer_gzip_matches_plain(tmp_path, shape, transpose, labels):
    from dca_b200.io import write_text_matrix_device
    m = torch.from_numpy(_matrix(shape, shape[0] * 1000 + shape[1])).to(DEV)
    rn = _names("r", shape[0]) if labels == "both" else None
    cn = _names("c", shape[1]) if labels == "both" else None
    a, b = str(tmp_path / "plain.tsv"), str(tmp_path / "z.tsv.gz")
    write_text_matrix_device(m, a, rownames=rn, colnames=cn, transpose=transpose)
    info = np.zeros(4, dtype=np.int64)
    write_text_matrix_device(m, b, rownames=rn, colnames=cn, transpose=transpose, gzip=True, info=info)
    plain, z = open(a, "rb").read(), open(b, "rb").read()
    assert gzip.decompress(z) == plain
    assert info[0] == len(z)
    assert _gunzip_device(b) == (plain, 1)


@pytest.mark.parametrize("transpose", [False, True])
def test_matrix_writer_gzip_many_groups_and_members(tmp_path, transpose):
    """Small pieces force many line groups per member; gene-block appends give one member per call."""
    from dca_b200.io import write_text_matrix_device
    m = torch.from_numpy(_matrix((700, 900), 5)).to(DEV)
    rn, cn = _names("r", 700), _names("c", 900)
    a, b = str(tmp_path / "plain.tsv"), str(tmp_path / "z.tsv.gz")
    blocks = list(range(0, 900 if transpose else 700, 130))
    for i, g0 in enumerate(blocks):
        part = m[:, g0:g0 + 130] if transpose else m[g0:g0 + 130]
        kw = dict(rownames=rn if transpose else rn[g0:g0 + 130], colnames=cn[g0:g0 + 130] if transpose else cn,
                  transpose=transpose, append=i > 0, header=i == 0, chunk_bytes=4096)
        write_text_matrix_device(part, a, **kw)
        info = np.zeros(4, dtype=np.int64)
        write_text_matrix_device(part, b, gzip=True, info=info, **kw)
        assert info[1] > 10
    plain, z = open(a, "rb").read(), open(b, "rb").read()
    assert gzip.decompress(z) == plain
    assert _gunzip_device(b) == (plain, len(blocks))


def test_host_matrix_writer_gzip(tmp_path):
    """Host matrices (float32, float64, empty) are compressed on the device too."""
    from dca_b200.io import write_text_matrix
    for k, m in enumerate([_matrix((40, 30), 1), _matrix((40, 30), 2).astype(np.float64), np.zeros((0, 3))]):
        a, b = str(tmp_path / ("p%d.tsv" % k)), str(tmp_path / ("z%d.tsv.gz" % k))
        kw = dict(rownames=_names("r", m.shape[0]), colnames=_names("c", m.shape[1]), transpose=True)
        write_text_matrix(m, a, **kw)
        write_text_matrix(m, b, gzip=True, device=DEV, **kw)
        assert gzip.decompress(open(b, "rb").read()) == open(a, "rb").read()
    assert sorted(os.listdir(tmp_path)) == sorted(["p0.tsv", "p1.tsv", "p2.tsv", "z0.tsv.gz", "z1.tsv.gz", "z2.tsv.gz"])


# ------------------------------------------------------------------------------------------------ predictions
N_CELLS, N_GENES = 5000, 512


@pytest.fixture(scope="module")
def counts():
    return synth_counts(N_CELLS, N_GENES, 21)


def _net(ae_type):
    from dca_b200.network import AE_types
    net = AE_types[ae_type](input_size=N_GENES, output_size=N_GENES, hidden_size=(64, 32, 64))
    net.build(max_batch=256, seed=4)
    return net


def _source(kind, Y):
    from dca_b200.anndata_lite import AnnData
    from dca_b200 import io
    if kind == "host":
        return {}, io.normalize(AnnData(Y.copy()), filter_min_counts=False)
    if kind == "device":
        from dca_b200.device_data import DeviceDataset
        return {"device_data": DeviceDataset.from_counts(Y, DEV)}, None
    if kind == "stream":
        from dca_b200.stream_data import StreamedDataset
        return {"stream_data": StreamedDataset.from_counts(Y, DEV)}, None
    from dca_b200.packed_data import PackedDeviceDataset
    return {"packed_data": PackedDeviceDataset.from_counts(Y, DEV)}, None


def _same_decompressed(plain, z):
    fa, fb = sorted(os.listdir(plain)), sorted(os.listdir(z))
    assert [f + ".gz" for f in fa] == fb
    for f in fa:
        assert gzip.decompress(open(os.path.join(z, f + ".gz"), "rb").read()) == \
            open(os.path.join(plain, f), "rb").read(), f
    return fa


@pytest.mark.parametrize("ae_type", ["zinb-conddisp", "nb-conddisp", "zinb"])
@pytest.mark.parametrize("kind", ["host", "device", "stream", "packed"])
def test_write_predictions_gzip(tmp_path, counts, ae_type, kind):
    net = _net(ae_type)
    src, adata = _source(kind, counts)
    cells, genes = _names("cell", N_CELLS), _names("gene", N_GENES)
    cap = 70 * 4 * N_CELLS * 3                                    # 70 genes a block: 8 members per gene-major file
    for name, gz in (("plain", False), ("z", True)):
        net.write_predictions(str(tmp_path / name), cells, genes, mode="full", return_info=True, adata=adata,
                              max_block_bytes=cap, chunk_bytes=1 << 20, gzip=gz, **src)
    files = _same_decompressed(tmp_path / "plain", tmp_path / "z")
    assert {"mean.tsv", "latent.tsv", "dispersion.tsv"} <= set(files)


@pytest.mark.parametrize("mode", ["denoise", "latent", "full"])
def test_write_predictions_gzip_modes(tmp_path, counts, mode):
    net = _net("zinb-conddisp")
    src, adata = _source("device", counts)
    cells, genes = _names("cell", N_CELLS), _names("gene", N_GENES)
    for name, gz in (("plain", False), ("z", True)):
        net.write_predictions(str(tmp_path / name), cells, genes, mode=mode, return_info=False, gzip=gz, **src)
    _same_decompressed(tmp_path / "plain", tmp_path / "z")


def test_write_predictions_gzip_shared(tmp_path, counts):
    """zinb-shared's outputs go through predict + write, host matrices compressed on the device.  Its split-K sums
    differ run to run in the last bits, so one prediction is written twice.  (With return_info, write stops at the
    per-cell dispersion's labels with or without gzip, as test_gpu_write_outputs pins for nb-shared.)"""
    from dca_b200.anndata_lite import AnnData
    net = _net("zinb-shared")
    cells, genes = ["c%d" % i for i in range(N_CELLS)], ["g%d" % i for i in range(N_GENES)]
    adata = AnnData(np.zeros((N_CELLS, N_GENES), np.float32), obs=pd.DataFrame(index=cells),
                    var=pd.DataFrame(index=genes))
    net.predict(adata, mode="full", return_info=False, **_source("device", counts)[0])
    net.write(adata, str(tmp_path / "plain"), mode="full", colnames=genes)
    net.write(adata, str(tmp_path / "z"), mode="full", colnames=genes, gzip=True)
    files = _same_decompressed(tmp_path / "plain", tmp_path / "z")
    assert {"mean.tsv", "latent.tsv"} == set(files)


# ------------------------------------------------------------------------------------------------ CLI
def test_cli_gzip(tmp_path):
    from dca_b200.__main__ import main
    Y = synth_counts(600, 96, 23).astype(int)
    genes = _names("g", 96)
    genes[2] = "gene two"
    df = pd.DataFrame(Y.T, index=genes, columns=["c%d" % i for i in range(600)])
    inp = tmp_path / "counts.tsv"
    df.to_csv(inp, sep="\t")
    args = [str(inp), None, "--type", "zinb-conddisp", "-e", "2", "-b", "64", "--preprocess", "device"]
    runs = {}
    for name, extra in (("plain", []), ("z1", ["--gzip"]), ("z2", ["--gzip"])):
        args[1] = str(tmp_path / name)
        main(args + extra)
        runs[name] = sorted(os.listdir(tmp_path / name))
    tsv = [f for f in runs["plain"] if f.endswith(".tsv")]
    assert {"mean.tsv", "dispersion.tsv", "dropout.tsv", "latent.tsv"} == set(tsv)
    assert runs["z1"] == sorted([f + ".gz" if f in tsv else f for f in runs["plain"]]) == runs["z2"]
    for f in tsv:
        z1 = open(tmp_path / "z1" / (f + ".gz"), "rb").read()
        assert gzip.decompress(z1) == open(tmp_path / "plain" / f, "rb").read(), f
        assert open(tmp_path / "z2" / (f + ".gz"), "rb").read() == z1, f
    kw = dict(sep="\t", index_col=0)
    pd.testing.assert_frame_equal(pd.read_csv(tmp_path / "z1" / "mean.tsv.gz", **kw),
                                  pd.read_csv(tmp_path / "plain" / "mean.tsv", **kw))
