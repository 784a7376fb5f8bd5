"""Step time of the training step with the debug checks off and on, at the benchmark shape (zinb-conddisp, 20000 genes,
batch 4096), the two alternated in one process; prints one JSON line with the card's name and power limit.

    python tests/diag_debug_checks.py [--genes 20000] [--batch 4096] [--steps 50] [--rounds 4]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genes", type=int, default=20000)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=4)
    a = ap.parse_args()
    from dca_b200.engine import DeviceEngine
    G, B = a.genes, a.batch
    eng = DeviceEngine(G, G, (64, 32, 64), ae_type="zinb-conddisp", max_batch=B, seed=0)
    g = torch.Generator(device="cuda").manual_seed(0)
    Y = torch.poisson(torch.full((B, G), 1.5, device="cuda"), generator=g)
    X = torch.log1p(Y)
    X = ((X - X.mean(0)) / (X.std(0) + 1)).contiguous()
    sf = torch.ones(B, device="cuda")
    times = {False: [], True: []}
    with torch.cuda.stream(torch.cuda.Stream()):
        for r in range(a.rounds):
            for debug in (False, True):
                eng.set_debug_checks(debug)
                for _ in range(3):                   # warm-up, graph capture
                    eng.train_step(X, Y, sf)
                    eng.apply_update(1e-4, 5.0)
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.current_stream().synchronize()
                t0.record()
                for _ in range(a.steps):
                    eng.train_step(X, Y, sf)
                    eng.apply_update(1e-4, 5.0)
                t1.record()
                t1.synchronize()
                times[debug].append(t0.elapsed_time(t1) / a.steps)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"genes": G, "batch": B, "steps": a.steps, "card": card,
                      "step_ms_off": times[False], "step_ms_on": times[True],
                      "median_off": sorted(times[False])[len(times[False]) // 2],
                      "median_on": sorted(times[True])[len(times[True]) // 2]}))


if __name__ == "__main__":
    main()
