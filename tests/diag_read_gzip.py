"""Reading gzip-compressed count files: the GPU inflate and the GPU readers over it (io.read_counts_gzip) against
host zlib and today's pandas / scipy route, one JSON line per size and reader.

    python tests/diag_read_gzip.py [--sizes 8192x20000,68000x20000] [--readers tsv,mtx] [--level 6]
                                   [--today-sizes 8192x20000,68000x20000]

A size is cells x genes.  The .tsv.gz is the table of diag_read_text.py (one line per gene, about 35 % non-zero), the
.mtx.gz the Cell Ranger-like file of diag_read_mtx.py (genes x cells, about 8 % non-zero), both gzip-compressed at
--level by Python's zlib in a temporary directory (not timed) and removed afterwards.  Per file, in one process:
  - inflate: dca_gunzip into device memory (after one warm-up call), as compressed and decompressed GB/s, and the
    rounds of span decoding the worst segment needed;
  - zlib: zlib.decompress of the same member on one core of this host;
  - read: read_dataset(path, transpose=True) on the .gz (the GPU route), today's route on the .gz (pandas or scipy,
    CUDA hidden from the router), and the GPU reader on the uncompressed file.
Times are wall clock up to a torch.cuda.synchronize.  The card's name and power limit are read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import shutil
import sys
import tempfile
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests.diag_read_mtx import write_mtx  # noqa: E402
from tests.diag_read_text import card, write_table  # noqa: E402


def compress(src, dst, level):
    c = zlib.compressobj(level, zlib.DEFLATED, 31)
    with open(src, "rb") as f, open(dst, "wb") as g:
        while True:
            b = f.read(64 << 20)
            if not b:
                break
            g.write(c.compress(b))
        g.write(c.flush())


def timed(fn):
    import torch
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def gunzip(path, out):
    import torch
    from dca_b200 import _lib
    info = np.zeros(4, dtype=np.int64)
    s = torch.cuda.current_stream()
    _lib.check(_lib.load().dca_gunzip(os.fsencode(path), torch.cuda.current_device(), C.c_void_p(s.cuda_stream),
                                      None if out is None else C.c_void_p(out.data_ptr()),
                                      0 if out is None else out.numel(), info.ctypes.data), "dca_gunzip")
    return info


def measure(raw, gz, today):
    import torch
    from dca_b200 import io
    rec = {"file_bytes": os.path.getsize(raw), "gz_bytes": os.path.getsize(gz)}
    info = gunzip(gz, None)
    out = torch.empty(int(info[0]), dtype=torch.uint8, device="cuda")
    gunzip(gz, out)
    t, info = timed(lambda: gunzip(gz, out))
    rec.update(inflate_s=round(t, 3), inflate_gb_s_compressed=round(rec["gz_bytes"] / t / 1e9, 3),
               inflate_gb_s_output=round(info[0] / t / 1e9, 3), rounds=int(info[2]))
    del out
    torch.cuda.empty_cache()
    with open(gz, "rb") as f:
        data = f.read()
    t0 = time.perf_counter()
    n = len(zlib.decompress(data, 31))
    tz = time.perf_counter() - t0
    assert n == rec["file_bytes"]
    rec.update(zlib_s=round(tz, 3), zlib_gb_s_output=round(n / tz / 1e9, 3))
    del data
    io.read_dataset(gz, transpose=True)                          # warm-up
    t_gpu, ad = timed(lambda: io.read_dataset(gz, transpose=True))
    shape = list(ad.shape)
    del ad
    t_raw, _ = timed(lambda: io.read_dataset(raw, transpose=True))
    rec.update(read_gz_gpu_s=round(t_gpu, 3), read_uncompressed_gpu_s=round(t_raw, 3), shape_cells_x_genes=shape)
    if today:
        real = io._cuda_available
        io._cuda_available = lambda: False
        try:
            t_host, ad = timed(lambda: io.read_dataset(gz, transpose=True))
        finally:
            io._cuda_available = real
        assert list(ad.shape) == shape
        rec.update(read_gz_today_s=round(t_host, 3))
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="8192x20000,68000x20000")
    ap.add_argument("--readers", default="tsv,mtx")
    ap.add_argument("--level", type=int, default=6)
    ap.add_argument("--today-sizes", default="8192x20000,68000x20000")
    a = ap.parse_args()
    import torch
    torch.zeros(1, device="cuda")
    name, limit = card()
    tmp = tempfile.mkdtemp(prefix="dca_read_gzip_")
    try:
        for size in a.sizes.split(","):
            n_cells, n_genes = (int(x) for x in size.split("x"))
            for reader in a.readers.split(","):
                raw = os.path.join(tmp, "counts.tsv" if reader == "tsv" else "matrix.mtx")
                gz = raw + ".gz"
                t0 = time.perf_counter()
                if reader == "tsv":
                    write_table(raw, n_cells, n_genes)
                else:
                    write_mtx(raw, n_cells, n_genes)
                compress(raw, gz, a.level)
                rec = {"size_cells_x_genes": size, "reader": reader, "gzip_level": a.level,
                       "generate_s": round(time.perf_counter() - t0, 1), "card": name, "power_limit": limit}
                try:
                    rec.update(measure(raw, gz, size in a.today_sizes.split(",")))
                except Exception as e:                           # noqa: BLE001
                    rec["error"] = repr(e)[-2000:]
                print(json.dumps(rec), flush=True)
                os.remove(raw)
                os.remove(gz)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
