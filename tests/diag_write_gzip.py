"""The CLI's output stage with --gzip (write_predictions(gzip=True): text compressed on the GPU) against plain TSV,
alternated in one session; then the compressed sizes against zlib, and the compressor's throughput.

Each timed run is a child process that packs the same synthetic counts, trains one epoch of zinb-conddisp with the same
seed and times the output stage alone: wall time, peak host RSS growth (sampled every 5 ms), bytes on disk and what the
writer measured.  The ratio run writes both forms at --ratio-size and compares each file's gzip size with zlib levels 1
and 6 of its text (zlib on 64 MB pieces in parallel processes: the pieces cost zlib well under 0.1 %).  The throughput
is dca_gzip_device's on 1 GiB of the mean text, already in device memory, timed around a device synchronise.

    python tests/diag_write_gzip.py --sizes 68000x20000 --ratio-size 8192x20000 --reps 1 [--out-json path]

Prints the GPU name and power limit first.  Writes its files to a temporary directory and removes them."""
import argparse
import concurrent.futures
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.diag_write_outputs import _PeakRss  # noqa: E402

PIECE = 64 << 20


def _zlib_piece(args):
    path, off, level = args
    with open(path, "rb") as f:
        f.seek(off)
        return len(zlib.compress(f.read(PIECE), level))


def _zlib_size(path, level, pool):
    offs = range(0, os.path.getsize(path), PIECE)
    return sum(pool.map(_zlib_piece, [(path, o, level) for o in offs]))


def child(mode, n, g, out):
    import numpy as np
    import torch
    from tests.util import synth_counts
    from dca_b200 import io, network
    from dca_b200.anndata_lite import AnnData
    from dca_b200.network import AE_types
    from dca_b200.train import train
    dev = torch.device("cuda", 0)
    adata = AnnData(synth_counts(n, g, 7), obs=None, var=None)
    adata = io.normalize(adata, device=dev, packed=True, filter_min_counts=False)
    pdd = adata.uns.pop("dca_packed_data")
    torch.manual_seed(42)
    np.random.seed(42)
    net = AE_types["zinb-conddisp"](input_size=g, output_size=g, hidden_size=(64, 32, 64))
    net.build(seed=0)
    train(adata, net, epochs=1, batch_size=32, verbose=False, packed_data=pdd)
    torch.cuda.synchronize()
    stats = {"mode": mode, "cells": n, "genes": g}
    writer = {"calls": 0, "bytes": 0, "kernel_us": 0, "wait_us": 0}
    orig = network.write_text_matrix_device

    def counted(t, filename, *a, **kw):
        info = np.zeros(4, dtype=np.int64)
        orig(t, filename, *a, info=info, **kw)
        writer["calls"] += 1
        writer["bytes"] += int(info[0])
        writer["kernel_us"] += int(info[2])
        writer["wait_us"] += int(info[3])
    network.write_text_matrix_device = counted

    def write(d, gz):
        net.write_predictions(d, adata.obs_names.values, adata.var_names, mode="full", return_info=True,
                              packed_data=pdd, adata=adata, gzip=gz)
        torch.cuda.synchronize()

    if mode in ("plain", "gzip"):
        with _PeakRss() as rss:
            t0 = time.perf_counter()
            write(out, mode == "gzip")
            stats["wall_s"] = time.perf_counter() - t0
        stats["rss_growth_mb"] = (rss.peak - rss.start_rss) / 2 ** 20
        stats["file_bytes"] = sum(os.path.getsize(os.path.join(out, f)) for f in os.listdir(out))
        stats["writer"] = writer
    else:
        plain, z = os.path.join(out, "plain"), os.path.join(out, "z")
        write(plain, False)
        write(z, True)
        sizes = {}
        with concurrent.futures.ProcessPoolExecutor() as pool:
            for name in ("mean", "dispersion", "dropout", "latent"):
                p = os.path.join(plain, name + ".tsv")
                sizes[name] = {"text": os.path.getsize(p), "gpu_gzip": os.path.getsize(os.path.join(z, name + ".tsv.gz")),
                               "zlib1": _zlib_size(p, 1, pool), "zlib6": _zlib_size(p, 6, pool)}
                sizes[name]["gpu_over_zlib1"] = sizes[name]["gpu_gzip"] / sizes[name]["zlib1"]
        stats["sizes"] = sizes
        with open(os.path.join(plain, "mean.tsv"), "rb") as f:
            text = f.read(1 << 30)
        src = torch.frombuffer(bytearray(text), dtype=torch.uint8).to(dev)
        del text
        io.gzip_device(src)
        times = []
        for _ in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            io.gzip_device(src)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        stats["gzip_device_gb_s"] = src.numel() / min(times) / 1e9
        stats["gzip_device_bytes"] = src.numel()
    print("RESULT " + json.dumps(stats), flush=True)


def run_child(mode, n, g):
    d = tempfile.mkdtemp(prefix="dca_gz_")
    try:
        p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", mode, "--n", str(n), "--g", str(g),
                            "--dir", d], capture_output=True, text=True, cwd=ROOT)
    finally:
        shutil.rmtree(d, ignore_errors=True)
    line = [x for x in p.stdout.splitlines() if x.startswith("RESULT ")]
    if p.returncode != 0 or not line:
        print(p.stdout[-2000:], p.stderr[-4000:], flush=True)
        raise SystemExit("child %s %dx%d failed" % (mode, n, g))
    res = json.loads(line[0][7:])
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="68000x20000")
    ap.add_argument("--ratio-size", default="8192x20000")
    ap.add_argument("--reps", type=int, default=1)
    ap.add_argument("--out-json", default=None)
    ap.add_argument("--child", default=None)
    ap.add_argument("--n", type=int, default=0)
    ap.add_argument("--g", type=int, default=0)
    ap.add_argument("--dir", default=None)
    a = ap.parse_args()
    if a.child:
        child(a.child, a.n, a.g, a.dir)
        return
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("GPU:", gpu, flush=True)
    results = {"gpu": gpu, "runs": []}
    if a.ratio_size:
        n, g = (int(x) for x in a.ratio_size.split("x"))
        results["runs"].append(run_child("ratio", n, g))
    for size in filter(None, a.sizes.split(",")):
        n, g = (int(x) for x in size.split("x"))
        for r in range(a.reps):
            for mode in ("plain", "gzip"):
                res = run_child(mode, n, g)
                res["rep"] = r
                results["runs"].append(res)
    if a.out_json:
        os.makedirs(os.path.dirname(os.path.abspath(a.out_json)), exist_ok=True)
        with open(a.out_json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
