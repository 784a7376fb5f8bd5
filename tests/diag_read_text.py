"""Reading a gene x cell count table: the pandas reader against the GPU reader (io.read_counts_text), one JSON line per
size and reader.

    python tests/diag_read_text.py [--sizes 8192x20000,68000x20000] [--pandas-sizes 8192x20000,68000x20000]

A size is cells x genes; the file has one line per gene and one column per cell, as the CLI reads it (transposed on
read).  The tables are seeded Poisson counts with the gene means of diag_preprocess.py (about 35 % non-zero),
written in row chunks to a temporary directory (not timed) and removed afterwards.  Each reader runs in its own
subprocess: one warm-up read, then one read timed from the path to the cells x genes AnnData (wall clock, after
torch.cuda.synchronize), with the file's GB/s and the process's peak RSS.  The card's name and power limit are read
in the same run.  The GPU reader needs a GPU.
"""
import argparse
import json
import os
import resource
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def write_table(path, n_cells, n_genes, seed=0, chunk=256):
    """gene x cell TSV of Poisson counts (gene means exp(N(-1.2, 1.3)), cell depths exp(N(0, 0.3)))."""
    rng = np.random.default_rng(seed)
    gene_mean = np.exp(rng.normal(-1.2, 1.3, size=n_genes))
    depth = np.exp(rng.normal(0, 0.3, size=n_cells))
    nnz = 0
    with open(path, "wb") as f:
        f.write(("gene\t" + "\t".join("c%d" % j for j in range(n_cells)) + "\n").encode())
        for g0 in range(0, n_genes, chunk):
            g1 = min(n_genes, g0 + chunk)
            V = rng.poisson(gene_mean[g0:g1, None] * depth[None, :]).astype(np.int64)
            nnz += int(np.count_nonzero(V))
            for i in range(g1 - g0):
                f.write(b"g%d\t" % (g0 + i) + digits_line(V[i]))
    return nnz / float(n_cells * n_genes)


def digits_line(v):
    """'\\t'-joined decimal text of a non-negative int64 row, ending in '\\n'."""
    nd = np.ones(v.shape, np.int64)
    p = 10
    while True:
        more = v >= p
        if not more.any():
            break
        nd += more
        p *= 10
    ends = np.cumsum(nd + 1)
    out = np.empty(int(ends[-1]), np.uint8)
    starts = ends - nd - 1
    for k in range(int(nd.max())):
        sel = nd > k
        out[starts[sel] + nd[sel] - 1 - k] = (v[sel] // 10 ** k) % 10 + 48
    out[ends - 1] = 9
    out[-1] = 10
    return out.tobytes()


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception as e:                                   # noqa: BLE001
        return "unknown", "unknown (%s)" % e


def worker(reader, path, timed):
    import torch
    from dca_b200 import io

    def read():
        if reader == "gpu":
            ad = io.read_counts_text(path, "\t", True)
            assert ad is not None, "the GPU reader did not take the file"
            torch.cuda.synchronize()
            return ad
        return io._read_text_pandas(path, "\t").transpose()
    if reader == "gpu":
        torch.zeros(1, device="cuda")
    times = []
    for _ in range(1 + timed):
        t0 = time.perf_counter()
        ad = read()
        times.append(time.perf_counter() - t0)
        shape = ad.shape
        del ad
    rss = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1024
    print(json.dumps({"wall_s": times[1:] if timed else times, "shape": list(shape), "peak_rss_bytes": rss}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="8192x20000,68000x20000")
    ap.add_argument("--pandas-sizes", default="8192x20000,68000x20000")
    ap.add_argument("--worker", default=None)
    ap.add_argument("--path", default=None)
    ap.add_argument("--timed", type=int, default=1)
    a = ap.parse_args()
    if a.worker:
        worker(a.worker, a.path, a.timed)
        return
    name, limit = card()
    pandas_sizes = set(s for s in a.pandas_sizes.split(",") if s)
    tmp = tempfile.mkdtemp(prefix="dca_read_text_")
    try:
        for size in a.sizes.split(","):
            n_cells, n_genes = (int(x) for x in size.split("x"))
            path = os.path.join(tmp, "counts_%s.tsv" % size)
            t0 = time.perf_counter()
            density = write_table(path, n_cells, n_genes)
            gen = time.perf_counter() - t0
            nbytes = os.path.getsize(path)
            for reader in ("gpu", "pandas"):
                if reader == "pandas" and size not in pandas_sizes:
                    continue
                # pandas: the file is in the page cache from writing it, so its one read is the timed one
                timed = 1 if reader == "gpu" else 0
                r = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", reader, "--path", path,
                                    "--timed", str(timed)], capture_output=True, text=True, cwd=ROOT)
                rec = {"size_cells_x_genes": size, "reader": reader, "file_bytes": nbytes, "nonzero": round(density, 4),
                       "generate_s": round(gen, 1), "card": name, "power_limit": limit}
                if r.returncode != 0:
                    rec["error"] = r.stderr[-2000:]
                else:
                    w = json.loads(r.stdout.strip().splitlines()[-1])
                    t = min(w["wall_s"])
                    rec.update(wall_s=round(t, 3), gb_per_s=round(nbytes / t / 1e9, 3), peak_rss_gb=round(w["peak_rss_bytes"] / 1e9, 2),
                               shape=w["shape"])
                print(json.dumps(rec), flush=True)
            os.remove(path)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
