"""Output stage of the CLI (`--preprocess device --packed -e 1 --type zinb-conddisp`), the host path
(Autoencoder.predict + write) against the GPU writer in gene blocks (Autoencoder.write_predictions), alternated in one
session.  Each run is a child process that packs the same synthetic counts, trains one epoch with the same seed and
times the output stage alone: wall time, and the peak host RSS during it (sampled every 5 ms from /proc).  The new
path's runs also report what the GPU writer measured (formatting kernel time, text bytes, time waiting for the file
writes), the number of predict passes and their device time.

    python tests/diag_write_outputs.py --sizes 8192x20000 --reps 2 [--out-json path]

Prints the GPU name and power limit first.  Writes its files to a temporary directory and removes them."""
import argparse
import json
import os
import resource
import shutil
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _rss():
    with open("/proc/self/statm") as f:
        return int(f.read().split()[1]) * os.sysconf("SC_PAGE_SIZE")


class _PeakRss:
    def __enter__(self):
        self.peak, self.stop = _rss(), False
        self.start_rss = self.peak

        def loop():
            while not self.stop:
                self.peak = max(self.peak, _rss())
                time.sleep(0.005)
        self.th = threading.Thread(target=loop)
        self.th.start()
        return self

    def __exit__(self, *a):
        self.stop = True
        self.th.join()
        self.peak = max(self.peak, _rss())


def child(path, n, g, out):
    import numpy as np
    import torch
    from tests.util import synth_counts
    from dca_b200 import io, network
    from dca_b200.anndata_lite import AnnData
    from dca_b200.network import AE_types
    from dca_b200.train import train
    dev = torch.device("cuda", 0)
    Y = synth_counts(n, g, 7)
    adata = AnnData(Y, obs=None, var=None)
    del Y
    adata = io.normalize(adata, device=dev, packed=True, filter_min_counts=False)
    pdd = adata.uns.pop("dca_packed_data")
    torch.manual_seed(42)
    np.random.seed(42)
    net = AE_types["zinb-conddisp"](input_size=g, output_size=g, hidden_size=(64, 32, 64))
    net.build(seed=0)
    train(adata, net, epochs=1, batch_size=32, verbose=False, packed_data=pdd)
    torch.cuda.synchronize()
    stats = {"path": path, "cells": n, "genes": g}
    writer = {"calls": 0, "bytes": 0, "kernel_us": 0, "wait_us": 0}
    if path == "new":
        orig = network.write_text_matrix_device

        def counted(t, filename, *a, **kw):
            info = np.zeros(4, dtype=np.int64)
            orig(t, filename, *a, info=info, **kw)
            writer["calls"] += 1
            writer["bytes"] += int(info[0])
            writer["kernel_us"] += int(info[2])
            writer["wait_us"] += int(info[3])
            if filename.endswith("mean.tsv"):
                writer["passes"] = writer.get("passes", 0) + 1
        network.write_text_matrix_device = counted
    with _PeakRss() as rss:
        t0 = time.perf_counter()
        if path == "old":
            net.predict(adata, mode="full", return_info=True, packed_data=pdd)
            net.write(adata, out, mode="full", colnames=adata.var_names)
        else:
            net.write_predictions(out, adata.obs_names.values, adata.var_names, mode="full", return_info=True,
                                  packed_data=pdd, adata=adata)
        torch.cuda.synchronize()
        stats["wall_s"] = time.perf_counter() - t0
    stats["rss_before_mb"] = rss.start_rss / 2 ** 20
    stats["rss_peak_mb"] = rss.peak / 2 ** 20
    stats["rss_growth_mb"] = (rss.peak - rss.start_rss) / 2 ** 20
    stats["file_bytes"] = sum(os.path.getsize(os.path.join(out, f)) for f in os.listdir(out))
    if path == "new":
        stats["writer"] = writer
        # one predict pass over all cells, device time (what each gene block repeats)
        eng, N = net.engine, pdd.n                # sized for predict by write_predictions above
        pdd._bind(eng)
        bs = min(network.PREDICT_BATCH, eng.max_batch)
        run, theta, session = pdd._predictor(eng, bs)
        bufs = {k: torch.empty((bs, g), device=dev) for k in ("mean", "disp", "pi")}
        bufs["latent"] = torch.empty((bs, eng.latent_dim), device=dev)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        times = []
        for _ in range(3):
            ev[0].record()
            for i, s in enumerate(range(0, N, bs)):
                run(i, s, min(s + bs, N), bufs)
            ev[1].record()
            torch.cuda.synchronize()
            times.append(ev[0].elapsed_time(ev[1]))
        stats["predict_pass_ms"] = min(times)
    stats["ru_maxrss_mb"] = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024
    print("RESULT " + json.dumps(stats), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="8192x20000")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--paths", default="old,new")
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
    for size in a.sizes.split(","):
        n, g = (int(x) for x in size.split("x"))
        for r in range(a.reps):
            for path in a.paths.split(","):
                d = tempfile.mkdtemp(prefix="dca_out_")
                try:
                    p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", path, "--n", str(n),
                                        "--g", str(g), "--dir", d], capture_output=True, text=True, cwd=ROOT)
                finally:
                    shutil.rmtree(d, ignore_errors=True)
                line = [x for x in p.stdout.splitlines() if x.startswith("RESULT ")]
                if p.returncode != 0 or not line:
                    print(p.stdout[-2000:], p.stderr[-4000:], flush=True)
                    raise SystemExit("child %s %s failed" % (path, size))
                res = json.loads(line[0][7:])
                res["rep"] = r
                results["runs"].append(res)
                print(json.dumps(res), flush=True)
    if a.out_json:
        os.makedirs(os.path.dirname(os.path.abspath(a.out_json)), exist_ok=True)
        with open(a.out_json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
