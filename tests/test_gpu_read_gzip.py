"""GPU inflate of gzip files (dca_gunzip, csrc/inflate.cu) and the readers over it (io.read_counts_gzip): the bytes
gzip.decompress gives for every stream of tests/gzip_cases.py, past 4 GiB of output, clean declines of malformed
files, and the same AnnData as today's pandas / scipy route on .tsv.gz, .txt.gz and .mtx.gz paths."""
import ctypes as C
import gzip
import os
import struct
import subprocess
import sys
import zlib

import numpy as np
import pytest
import scipy.io
import scipy.sparse as sp
import torch

from dca_b200 import _lib, io
from tests.gzip_cases import cases, count_text, member

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def gunzip(path, out=None):
    """(status, info); with out (a uint8 CUDA tensor) the second call fills it."""
    lib = _lib.load()
    info = np.zeros(4, dtype=np.int64)
    s = torch.cuda.current_stream()
    st = lib.dca_gunzip(os.fsencode(str(path)), torch.cuda.current_device(), C.c_void_p(s.cuda_stream),
                        None if out is None else C.c_void_p(out.data_ptr()), 0 if out is None else out.numel(),
                        info.ctypes.data)
    return st, info


def gunzip_bytes(path):
    st, info = gunzip(path)
    if st != 0:
        return st, None, info
    out = torch.empty(max(int(info[0]), 1), dtype=torch.uint8, device="cuda")
    st, info2 = gunzip(path, out[:int(info[0])])
    assert st == 0 and (info2[[0, 2, 3]] == info[[0, 2, 3]]).all()      # info[1]: the first call's scratch too
    return st, out[:int(info[0])].cpu().numpy().tobytes(), info


@pytest.fixture(scope="module")
def streams():
    c = cases()
    big = count_text(150 << 20, seed=3)
    c["segments_level0"] = member(big, level=0), big     # three 64 MB segments of stored blocks
    c["big_level6"] = member(big, level=6), big
    return c


# Stored blocks of count text hold many plausible dynamic-block headers, so most speculative spans there start wrong
# and each round verifies only a few blocks: a long run of them may need more rounds than a segment allows, and the
# file is then declined (and read by pandas or scipy).
MAY_DECLINE = {"segments_level0"}


def test_bytes_and_rounds(tmp_path, streams):
    rounds = {}
    for name, (gz, data) in sorted(streams.items()):
        p = tmp_path / (name + ".gz")
        p.write_bytes(gz)
        st, got, info = gunzip_bytes(p)
        if st == -3 and name in MAY_DECLINE:
            assert b"rounds" in _lib.load().dca_last_error()
            rounds[name] = "declined"
            continue
        assert st == 0, (name, _lib.load().dca_last_error())
        assert got == data == gzip.decompress(gz), name
        rounds[name] = int(info[2])
    print("rounds per stream:", rounds)
    for lv in (1, 6, 9):
        assert rounds["level%d" % lv] == 1, rounds


def test_past_4_gib(tmp_path):
    """One member of more than 2^32 output bytes (ISIZE wraps): a 64 MB TSV piece compressed once after a full flush and
    repeated; the bytes are checked piece by piece on the device and the parsed matrix against the piece's."""
    cols, reps = 64, 66
    rng = np.random.default_rng(5)
    vals = 10 ** 16 + rng.integers(0, 10 ** 6, (60000, cols))
    head = ("gene\t" + "\t".join("c%d" % j for j in range(cols)) + "\n").encode()
    piece = "".join("g\t" + "\t".join(map(str, r)) + "\n" for r in vals.tolist()).encode()
    lines = piece.count(b"\n")
    total = len(head) + reps * len(piece)
    need = total + lines * reps * cols * 4 * 2 + (4 << 30)
    if torch.cuda.mem_get_info()[0] < need:
        pytest.skip("needs %.1f GB of free device memory" % (need / 1e9))
    assert total > 2 ** 32
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    h = c.compress(head) + c.flush(zlib.Z_FULL_FLUSH)
    cp = zlib.compressobj(6, zlib.DEFLATED, -15)
    pc = cp.compress(piece) + cp.flush(zlib.Z_FULL_FLUSH)
    crc = zlib.crc32(head)
    for _ in range(reps):
        crc = zlib.crc32(piece, crc)
    p = tmp_path / "big.tsv.gz"
    with open(p, "wb") as f:
        f.write(b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\xff" + h)
        for _ in range(reps):
            f.write(pc)
        f.write(b"\x03\x00" + struct.pack("<II", crc, total & 0xffffffff))
    st, info = gunzip(p)
    assert st == 0, _lib.load().dca_last_error()
    assert info[0] == total
    out = torch.empty(total, dtype=torch.uint8, device="cuda")
    st, _ = gunzip(p, out)
    assert st == 0
    ref = torch.frombuffer(bytearray(piece), dtype=torch.uint8).cuda()
    assert bytes(out[:len(head)].cpu().numpy()) == head
    for k in range(reps):
        a = len(head) + k * len(piece)
        assert torch.equal(out[a:a + len(piece)], ref), k
    del out, ref
    torch.cuda.empty_cache()
    ad = io.read_counts_gzip(str(p))
    assert ad is not None and ad.X.shape == (lines * reps, cols)
    exp = vals.astype(np.float32)
    for k in range(reps):
        assert ad.X[k * lines:(k + 1) * lines].tobytes() == exp.tobytes(), k


def _corrupt(gz, case, seed=0):
    b = bytearray(gz)
    if case == "truncated":
        return bytes(b[:len(b) * 2 // 3])
    if case == "crc":
        b[-8] ^= 1
    elif case == "isize":
        b[-4] ^= 1
    elif case == "bitflip":
        rng = np.random.default_rng(seed)
        for i in rng.integers(12, len(b) - 8, 3):
            b[i] ^= 1 << int(rng.integers(0, 8))
    elif case == "trailing":
        b += b"garbage"
    elif case == "cm":
        b[2] = 7
    elif case == "reserved_flag":
        b[3] |= 0x20
    elif case == "fhcrc":
        return member(count_text(20000), flags=2)[:10] + b"\x00\x00" + member(count_text(20000), flags=2)[12:]
    return bytes(b)


@pytest.mark.parametrize("case", ["truncated", "crc", "isize", "bitflip", "trailing", "cm", "reserved_flag", "fhcrc"])
def test_declined(tmp_path, case):
    text = count_text(100_000)
    gz = _corrupt(member(text), case)
    p = tmp_path / "counts.tsv.gz"
    p.write_bytes(gz)
    st, info = gunzip(p)
    assert st == -3, (case, st)
    assert io.read_counts_gzip(str(p)) is None
    try:
        exp = io._read_text_pandas(str(p), "\t")
    except Exception as e:                                       # noqa: BLE001
        with pytest.raises(type(e)):
            io.read_dataset(str(p))
        return
    got = io.read_dataset(str(p))
    assert got.X.tobytes() == exp.X.tobytes()


@pytest.mark.parametrize("seed", range(4))
def test_bit_flips_decline_or_match(tmp_path, seed):
    """Seeded bit flips anywhere in the deflate data: dca_gunzip declines, or (a flip zlib also accepts) gives zlib's bytes."""
    gz = _corrupt(member(count_text(60_000), level=9), "bitflip", seed)
    p = tmp_path / "x.gz"
    p.write_bytes(gz)
    try:
        ref = gzip.decompress(gz)
    except Exception:                                            # noqa: BLE001
        ref = None
    st, got, _ = gunzip_bytes(p)
    assert (st == -3 and ref is None) or (st == 0 and got == ref)


def table(n_genes, n_cells, seed=0, sep="\t"):
    rng = np.random.default_rng(seed)
    M = (rng.poisson(2.0, (n_genes, n_cells)) * (rng.random((n_genes, n_cells)) < 0.3)).astype(np.int64)
    lines = [sep.join([""] + ["c%d" % j for j in range(n_cells)])]
    lines += [sep.join(["g%d" % i] + [str(v) for v in M[i]]) for i in range(n_genes)]
    return ("\n".join(lines) + "\n").encode()


def assert_same(ad, exp):
    assert ad.X.dtype == exp.X.dtype and ad.X.shape == exp.X.shape
    if sp.issparse(exp.X):
        for a in ("indptr", "indices", "data"):
            x, y = getattr(ad.X, a), getattr(exp.X, a)
            assert x.dtype == y.dtype and x.tobytes() == y.tobytes(), a
    else:
        assert ad.X.tobytes() == exp.X.tobytes()
    assert list(ad.obs_names) == list(exp.obs_names) and list(ad.var_names) == list(exp.var_names)


@pytest.mark.parametrize("ext", [".tsv.gz", ".txt.gz"])
@pytest.mark.parametrize("chunk_bytes", [0, 4096])
def test_text_same_as_pandas(tmp_path, monkeypatch, ext, chunk_bytes):
    p = tmp_path / ("counts" + ext)
    p.write_bytes(gzip.compress(table(300, 500)))
    ref = io._read_text_pandas(str(p), "\t")
    for tr in (False, True):
        ad = io.read_counts_gzip(str(p), tr, chunk_bytes=chunk_bytes)
        assert ad is not None
        assert_same(ad, ref.transpose() if tr else ref)

    def no_pandas(*a, **k):
        raise AssertionError("the host reader was called")
    monkeypatch.setattr(io, "_read_text_pandas", no_pandas)
    got = io.read_dataset(str(p), transpose=True)
    assert_same(got, ref.transpose())


def test_mtx_same_as_scipy(tmp_path, monkeypatch):
    M = sp.random(700, 400, density=0.08, format="csr", random_state=3, dtype=np.float64)
    M.data = np.ceil(M.data * 20)
    raw = tmp_path / "m.mtx"
    scipy.io.mmwrite(str(raw), M, field="integer")
    p = tmp_path / "matrix.mtx.gz"
    p.write_bytes(gzip.compress(raw.read_bytes()))
    ref = io._read_mtx_scipy(str(p))
    for tr in (False, True):
        exp = io._read_mtx_scipy(str(raw))
        exp = AnnDataT(exp) if tr else exp
        ad = io.read_counts_gzip(str(p), tr)
        if ad is None:                        # entries not in CSR order of this orientation: declined as for .mtx
            assert io.read_counts_mtx(str(raw), tr) is None
            continue
        assert_same(ad, exp)
    assert_same(io._read_mtx_scipy(str(p)), ref)

    def no_scipy(*a, **k):
        raise AssertionError("the host reader was called")
    monkeypatch.setattr(io, "_read_mtx_scipy", no_scipy)
    got = io.read_dataset(str(p))
    assert_same(got, ref)


def AnnDataT(ad):
    from dca_b200.anndata_lite import AnnData
    return AnnData(ad.X.T.tocsr(), keep_sparse=True)


def test_csv_gz_reads_as_today(tmp_path):
    p = tmp_path / "counts.csv.gz"
    p.write_bytes(gzip.compress(table(50, 40, sep=",")))
    assert io.read_counts_gzip(str(p)) is None            # the tab separator of today's route splits nothing
    exp = io._read_text_pandas(str(p), "\t")
    assert_same(io.read_text_or_h5ad(str(p)), exp)


def test_cli_gz_same_files(tmp_path):
    raw = tmp_path / "counts.tsv"
    raw.write_bytes(table(200, 300, seed=4))
    gz = tmp_path / "counts.tsv.gz"
    gz.write_bytes(gzip.compress(raw.read_bytes()))
    outs = []
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    for src in (raw, gz):
        run = tmp_path / ("run_" + src.name.replace(".", "_"))
        run.mkdir()
        # the same relative output directory in both runs: model.pickle holds the network's output path
        subprocess.check_call([sys.executable, "-m", "dca_b200", str(src), "out", "-e", "2"], cwd=str(run), env=env)
        outs.append(run / "out")
    files = sorted(os.listdir(outs[0]))
    assert files == sorted(os.listdir(outs[1])) and "mean.tsv" in files
    for f in files:
        assert (outs[0] / f).read_bytes() == (outs[1] / f).read_bytes(), f


def test_real_size_tsv(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from diag_read_text import write_table
    raw = tmp_path / "counts.tsv"
    write_table(str(raw), 8192, 20000)
    gz = tmp_path / "counts.tsv.gz"
    with open(raw, "rb") as f, gzip.open(gz, "wb", compresslevel=6) as g:
        while True:
            b = f.read(64 << 20)
            if not b:
                break
            g.write(b)
    a = io.read_counts_text(str(raw), "\t", True)
    b = io.read_counts_gzip(str(gz), True)
    assert b is not None
    assert_same(b, a)


def test_real_size_mtx(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from diag_read_mtx import write_mtx
    raw = tmp_path / "matrix.mtx"
    write_mtx(str(raw), 68000, 20000)
    gz = tmp_path / "matrix.mtx.gz"
    with open(raw, "rb") as f, gzip.open(gz, "wb", compresslevel=6) as g:
        while True:
            b = f.read(64 << 20)
            if not b:
                break
            g.write(b)
    a = io.read_counts_mtx(str(raw), True)
    b = io.read_counts_gzip(str(gz), True)
    assert a is not None and b is not None
    assert_same(b, a)
