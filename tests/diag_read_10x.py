"""Reading a Cell Ranger ARC-like matrix directory: the GPU route (io.read_counts_10x) against the host statement
(io._read_10x_scipy), each in a child process of its own, with its wall time, peak host RSS and peak device memory.
One JSON line per measurement.

    python tests/diag_read_10x.py [--cells 68000] [--genes 36000] [--peaks 150000] [--gene-density 0.025]
                                  [--peak-density 0.008] [--level 1]

The directory is seeded and written to a temporary directory (not timed) and removed afterwards: matrix.mtx.gz,
features.tsv.gz (six columns, the gene rows first and then the peak rows, as Cell Ranger ARC writes them) and
barcodes.tsv.gz, gzip level `--level`.  Each cell's entries are uniform draws over the gene rows and over the peak rows
at the given densities, each value 1 + a Poisson(2) count; the matrix is genes x cells in column-major order, read
with transpose as the CLI does.  The GPU route runs twice (the first a warm-up that also puts the files in the page
cache) and the host statement once; wall clock from the path to the AnnData, up to a torch.cuda.synchronize for the
GPU.  Peak host RSS is the child's ru_maxrss less its RSS before the read; peak device memory is the largest drop of
cudaMemGetInfo's free bytes below its value before the read, sampled every 2 ms (it counts the reader's own buffers,
which torch's allocator does not see).  The two results are compared array by array.  The card's name and power limit
are read in the same run.
"""
import argparse
import gzip
import json
import os
import resource
import shutil
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests.diag_read_mtx import entry_lines  # noqa: E402
from tests.diag_read_text import card  # noqa: E402


def write_dir(d, n_cells, n_genes, n_peaks, dg, dp, level, seed=0, block=4096):
    """The seeded directory; returns the number of entries."""
    rng = np.random.default_rng(seed)
    os.makedirs(d)
    nnz = 0
    body = os.path.join(d, "body.gz")
    with gzip.open(body, "wb", compresslevel=level) as f:
        for c0 in range(0, n_cells, block):
            c1 = min(n_cells, c0 + block)
            cells, rows = [], []
            for n_rows, dens, first in ((n_genes, dg, 0), (n_peaks, dp, n_genes)):
                per = rng.poisson(dens * n_rows, c1 - c0)
                c = np.repeat(np.arange(c0, c1), per)
                cells.append(c)
                rows.append(first + rng.integers(0, n_rows, c.size))
            cells, rows = np.concatenate(cells), np.concatenate(rows)
            order = np.lexsort((rows, cells))
            cells, rows = cells[order], rows[order]
            keep = np.ones(cells.size, bool)
            keep[1:] = (cells[1:] != cells[:-1]) | (rows[1:] != rows[:-1])      # no duplicate entries
            cells, rows = cells[keep], rows[keep]
            f.write(entry_lines((rows + 1, cells + 1, 1 + rng.poisson(2.0, cells.size))))
            nnz += cells.size
    with open(os.path.join(d, "matrix.mtx.gz"), "wb") as out:
        out.write(gzip.compress(b"%%%%MatrixMarket matrix coordinate integer general\n%%\n%d %d %d\n"
                                % (n_genes + n_peaks, n_cells, nnz), level))
        with open(body, "rb") as b:
            shutil.copyfileobj(b, out, 1 << 24)                  # a second gzip member
    os.remove(body)
    feats = ["ENSG%011d\tGENE%d\tGene Expression\tchr1\t%d\t%d\n" % (g, g, 1000 * g, 1000 * g + 900)
             for g in range(n_genes)]
    feats += ["chr2:%d-%d\tchr2:%d-%d\tPeaks\tchr2\t%d\t%d\n" % ((500 * p, 500 * p + 400) * 3) for p in range(n_peaks)]
    with gzip.open(os.path.join(d, "features.tsv.gz"), "wt", compresslevel=level) as f:
        f.write("".join(feats))
    with gzip.open(os.path.join(d, "barcodes.tsv.gz"), "wt", compresslevel=level) as f:
        f.write("".join("%s-1\n" % "".join(s) for s in rng.choice(list("ACGT"), (n_cells, 16))))
    return nnz


def child(route, d, out):
    """Runs one read in this process and writes its measurements and arrays to `out` (.npz)."""
    import torch
    from dca_b200 import io
    torch.zeros(1, device="cuda")
    torch.cuda.synchronize()
    rss0 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
    free0 = torch.cuda.mem_get_info()[0]
    low = [free0]
    stop = threading.Event()

    def sample():
        while not stop.is_set():
            low[0] = min(low[0], torch.cuda.mem_get_info()[0])
            time.sleep(0.002)
    th = threading.Thread(target=sample, daemon=True)
    th.start()
    t0 = time.perf_counter()
    ad = io.read_counts_10x(d, True) if route == "gpu" else io._read_10x_scipy(d, True)
    torch.cuda.synchronize()
    t = time.perf_counter() - t0
    stop.set()
    th.join()
    assert ad is not None, "the GPU reader did not take the matrix"
    rss = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss - rss0
    np.savez(out, wall_s=t, rss_growth_kb=rss, device_peak=free0 - low[0], indptr=ad.X.indptr, indices=ad.X.indices,
             data=ad.X.data, shape=np.array(ad.X.shape), obs=np.array(list(ad.obs_names)),
             var=np.array(list(ad.var_names)), gene_ids=np.array(list(ad.var["gene_ids"])))


def main():
    if len(sys.argv) > 1 and sys.argv[1] == "--child":
        return child(*sys.argv[2:5])
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=int, default=68000)
    ap.add_argument("--genes", type=int, default=36000)
    ap.add_argument("--peaks", type=int, default=150000)
    ap.add_argument("--gene-density", type=float, default=0.025)
    ap.add_argument("--peak-density", type=float, default=0.008)
    ap.add_argument("--level", type=int, default=1)
    a = ap.parse_args()
    name, limit = card()
    tmp = tempfile.mkdtemp(prefix="dca_read_10x_")
    try:
        d = os.path.join(tmp, "filtered_feature_bc_matrix")
        t0 = time.perf_counter()
        nnz = write_dir(d, a.cells, a.genes, a.peaks, a.gene_density, a.peak_density, a.level)
        base = {"cells": a.cells, "gene_rows": a.genes, "peak_rows": a.peaks, "nnz_file": nnz,
                "matrix_gz_bytes": os.path.getsize(os.path.join(d, "matrix.mtx.gz")), "gzip_level": a.level,
                "card": name, "power_limit": limit}
        print(json.dumps(dict(base, what="written", wall_s=round(time.perf_counter() - t0, 1))), flush=True)
        res = {}
        for route, label in (("gpu", "warmup"), ("gpu", "gpu"), ("scipy", "scipy")):
            out = os.path.join(tmp, label + ".npz")
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", route, d, out], cwd=ROOT,
                               capture_output=True, text=True)
            if r.returncode:
                print(json.dumps(dict(base, what=label, returncode=r.returncode, stderr=r.stderr[-1500:])), flush=True)
                return 1
            z = dict(np.load(out))
            res[label] = z
            print(json.dumps(dict(base, what=("gpu_read_10x" if route == "gpu" else "scipy_read_10x")
                                  + ("_warmup" if label == "warmup" else ""),
                                  wall_s=round(float(z["wall_s"]), 3), nnz_kept=int(z["data"].size),
                                  host_rss_growth_gb=round(float(z["rss_growth_kb"]) / 2 ** 20, 2),
                                  device_peak_gb=round(float(z["device_peak"]) / 2 ** 30, 2))), flush=True)
        g, s = res["gpu"], res["scipy"]
        same = {k: bool(g[k].dtype == s[k].dtype and g[k].tobytes() == s[k].tobytes())
                for k in ("indptr", "indices", "data", "shape")}
        same.update({k: bool(np.array_equal(g[k], s[k])) for k in ("obs", "var", "gene_ids")})
        print(json.dumps(dict(base, what="gpu_equals_scipy", speedup=round(float(s["wall_s"] / g["wall_s"]), 1),
                              **same)), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
