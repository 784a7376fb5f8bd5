"""Reading a 10x-like Matrix Market file: the scipy statement against the GPU reader (io.read_counts_mtx), the packed
dataset built from the CSR it returns, and the CLI from the .mtx file against the same counts as a TSV.  One JSON line
per measurement.

    python tests/diag_read_mtx.py [--sizes 8192x20000,68000x20000] [--cli-sizes 8192x20000] [--epochs 1]

A size is cells x genes.  The file is genes x cells in column-major order (Cell Ranger's layout, read with transpose
as the CLI does), seeded, about 8 % non-zero, written to a temporary directory (not timed) and removed afterwards.
Each reader runs once as a warm-up (so the file is in the page cache) and once timed, wall clock up to a
torch.cuda.synchronize, with the file's GB/s.  The GPU reader is timed with transpose=True; the scipy statement is
csr_matrix(mmread(path).astype(float32)) as scanpy runs it, and its .T.tocsr() separately.  The CLI runs with
--preprocess device --packed in a subprocess per input.  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests.diag_read_text import card, digits_line  # noqa: E402


def _ndigits(v):
    nd = np.ones(v.shape, np.int64)
    p = 10
    while True:
        more = v >= p
        if not more.any():
            return nd
        nd += more
        p *= 10


def entry_lines(fields):
    """'i j v\\n' lines of three non-negative int64 arrays, as bytes."""
    nds = [_ndigits(f) for f in fields]
    ends = np.cumsum(nds[0] + nds[1] + nds[2] + 3)
    out = np.empty(int(ends[-1]) if ends.size else 0, np.uint8)
    pos = ends - (nds[0] + nds[1] + nds[2] + 3)
    for f, nd, sep in zip(fields, nds, (32, 32, 10)):
        for k in range(int(nd.max()) if nd.size else 0):
            sel = nd > k
            out[pos[sel] + nd[sel] - 1 - k] = (f[sel] // 10 ** k) % 10 + 48
        pos = pos + nd
        out[pos] = sep
        pos = pos + 1
    return out.tobytes()


def write_mtx(path, n_cells, n_genes, seed=0, block=2048, tsv=None):
    """Seeded 10x-like counts, genes x cells, column-major; also the genes x cells TSV of the same counts when tsv."""
    rng = np.random.default_rng(seed)
    p_gene = np.clip(rng.lognormal(np.log(0.05), 1.0, n_genes), 0, 0.9)
    p_gene *= 0.08 / p_gene.mean()
    mean_gene = 1.0 + 20 * p_gene
    depth = rng.lognormal(0, 0.3, n_cells)
    blocks, nnz = [], 0
    tmp = path + ".body"
    with open(tmp, "wb") as f:
        for c0 in range(0, n_cells, block):
            c1 = min(n_cells, c0 + block)
            nz = rng.random((c1 - c0, n_genes), dtype=np.float32) < np.minimum(p_gene[None, :] * depth[c0:c1, None], 1)
            cells, genes = np.nonzero(nz)
            vals = 1 + rng.poisson(mean_gene[genes] * depth[c0 + cells])
            f.write(entry_lines((genes + 1, cells + c0 + 1, vals)))
            nnz += cells.size
            if tsv is not None:
                M = np.zeros((c1 - c0, n_genes), np.int64)
                M[cells, genes] = vals
                blocks.append(M)
    with open(path, "wb") as f, open(tmp, "rb") as b:
        f.write(b"%%%%MatrixMarket matrix coordinate integer general\n%%\n%d %d %d\n" % (n_genes, n_cells, nnz))
        shutil.copyfileobj(b, f, 1 << 24)
    os.remove(tmp)
    if tsv is not None:
        G = np.concatenate(blocks).T                            # genes x cells
        with open(tsv, "wb") as f:
            f.write(("\t" + "\t".join(str(j) for j in range(n_cells)) + "\n").encode())
            for g in range(n_genes):
                f.write(b"%d\t" % g + digits_line(G[g]))
    return nnz


def timed(fn, sync):
    fn()
    sync()
    t0 = time.perf_counter()
    out = fn()
    sync()
    return out, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="8192x20000,68000x20000")
    ap.add_argument("--cli-sizes", default="8192x20000")
    ap.add_argument("--epochs", type=int, default=1)
    a = ap.parse_args()
    import scipy.io
    import scipy.sparse as sp
    import torch
    from dca_b200 import io
    from dca_b200.packed_data import PackedDeviceDataset
    name, limit = card()
    sync = torch.cuda.synchronize
    torch.zeros(1, device="cuda")
    tmp = tempfile.mkdtemp(prefix="dca_read_mtx_")
    try:
        for size in a.sizes.split(","):
            n_cells, n_genes = (int(x) for x in size.split("x"))
            path = os.path.join(tmp, "matrix_%s.mtx" % size)
            tsv = os.path.join(tmp, "counts_%s.tsv" % size) if size in a.cli_sizes.split(",") else None
            nnz = write_mtx(path, n_cells, n_genes, tsv=tsv)
            nbytes = os.path.getsize(path)
            base = {"size_cells_x_genes": size, "nnz": nnz, "file_bytes": nbytes, "card": name, "power_limit": limit}

            def rec(what, t, **kw):
                print(json.dumps(dict(base, what=what, wall_s=round(t, 3), gb_per_s=round(nbytes / t / 1e9, 3), **kw)),
                      flush=True)
            ad, t = timed(lambda: io.read_counts_mtx(path, True), sync)
            assert ad is not None, "the GPU reader did not take the file"
            rec("gpu_reader_transpose", t)

            def scipy_read():
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore", DeprecationWarning)
                    return sp.csr_matrix(scipy.io.mmread(path).astype(np.float32))
            with warnings.catch_warnings():
                warnings.simplefilter("ignore", DeprecationWarning)
                _, t_mm = timed(lambda: scipy.io.mmread(path), lambda: None)
            ref, t = timed(scipy_read, lambda: None)
            rec("scipy_statement", t, mmread_s=round(t_mm, 3))
            refT, t = timed(lambda: ref.T.tocsr(), lambda: None)
            rec("scipy_transpose_tocsr", t)
            same = all(getattr(ad.X, f).tobytes() == getattr(refT, f).tobytes() for f in ("indptr", "indices", "data"))
            print(json.dumps(dict(base, what="gpu_equals_scipy", equal=bool(same))), flush=True)
            del ref, refT
            pdd, t = timed(lambda: PackedDeviceDataset.from_counts(ad.X, "cuda"), sync)
            rec("packed_from_counts", t, packed_bits=int(pdd.desc.bits))
            del pdd, ad
            torch.cuda.empty_cache()
            if tsv is not None:
                for inp in (path, tsv):
                    out = os.path.join(tmp, "out_" + os.path.basename(inp))
                    t0 = time.perf_counter()
                    r = subprocess.run([sys.executable, "-m", "dca_b200", inp, out, "--preprocess", "device", "--packed",
                                        "-e", str(a.epochs), "--type", "zinb-conddisp"], capture_output=True, text=True,
                                       cwd=ROOT)
                    t = time.perf_counter() - t0
                    extra = {"input": os.path.splitext(inp)[1], "input_bytes": os.path.getsize(inp), "epochs": a.epochs,
                             "returncode": r.returncode}
                    if r.returncode:
                        extra["stderr"] = r.stderr[-1500:]
                    print(json.dumps(dict(base, what="cli_packed", wall_s=round(t, 2), **extra)), flush=True)
                a_, b_ = (os.path.join(tmp, "out_" + os.path.basename(x)) for x in (path, tsv))
                same = all(open(os.path.join(a_, f), "rb").read() == open(os.path.join(b_, f), "rb").read()
                           for f in ("mean.tsv", "dispersion.tsv", "dropout.tsv", "latent.tsv"))
                print(json.dumps(dict(base, what="cli_outputs_identical", equal=bool(same))), flush=True)
                os.remove(tsv)
            os.remove(path)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
