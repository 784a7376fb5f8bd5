"""Resident, streamed and packed datasets at a ragged gene count (19 999) against a multiple of 8 (20 000), one JSON
line per (genes, x_dtype).

    python tests/diag_ragged_packed.py [--cells 68000] [--genes 19999,20000] [--batch 4096] [--rounds 3]

Per case (seeded synthetic Poisson counts, tests/diag_preprocess.synth_poisson): the wall time of from_counts of
DeviceDataset, StreamedDataset and PackedDeviceDataset (synchronised host clock; the streamed and packed ones with
pad_genes=True), then the training rate in cells/s of one epoch of each dataset kind (the epoch train() runs: shuffled
batches of --batch rows and RMSprop updates, timed with device events after a warm-up epoch), the three kinds
alternated --rounds times; the median round is reported.  The card's name and power limit are read in the same run.
Needs a GPU.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tests.diag_preprocess import card, synth_poisson      # noqa: E402


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def epoch_rate(net, ds, bs):
    """Cells/s of one training epoch of dataset ds (device events around the epoch)."""
    eng = net.engine
    ds._bind(eng)
    n_tr = ds.n
    epoch, _ = ds._fit(eng, n_tr, bs, True)
    upd = lambda: eng.apply_update(1e-3, 5.0, 1.0)       # noqa: E731
    epoch(upd)                                           # warm-up: the shapes of every batch, the stream's pinning
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0.record()
    epoch(upd)
    t1.record()
    t1.synchronize()
    return n_tr / (t0.elapsed_time(t1) / 1e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=int, default=68000)
    ap.add_argument("--genes", default="19999,20000")
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    from dca_b200.device_data import DeviceDataset
    from dca_b200.network import AE_types
    from dca_b200.packed_data import PackedDeviceDataset
    from dca_b200.stream_data import StreamedDataset
    name, limit = card()
    dev = torch.device("cuda:0")
    for G in (int(g) for g in a.genes.split(",")):
        Y = synth_poisson(a.cells, G, seed=G)
        for x_dtype in ("float32", "bfloat16"):
            makers = {
                "resident": lambda: DeviceDataset.from_counts(Y, dev, x_dtype),
                "stream": lambda: StreamedDataset.from_counts(Y, dev, x_dtype, batch=a.batch, pad_genes=True),
                "packed": lambda: PackedDeviceDataset.from_counts(Y, dev, x_dtype, pad_genes=True)}
            wall(makers["packed"])                        # warm-up: module loads, first cudaHostAlloc
            prep, data = {}, {}
            for k, mk in makers.items():
                prep[k], data[k] = wall(mk)
            nets = {}
            for k in data:
                net = AE_types["zinb-conddisp"](input_size=G, output_size=G, x_dtype=x_dtype)
                net.build(max_batch=a.batch, seed=0)
                net.engine.set_optimizer("RMSprop")
                nets[k] = net
            info = nets["resident"].engine.info()
            rates = {k: [] for k in data}
            for _ in range(a.rounds):
                for k in data:
                    rates[k].append(epoch_rate(nets[k], data[k], a.batch))
            print(json.dumps({
                "card": name, "power_limit": limit, "cells": a.cells, "genes": G, "x_dtype": x_dtype,
                "batch": a.batch, "tc_heads": bool(info["tc_heads"]), "tc_encoder": bool(info["tc_encoder"]),
                "from_counts_s": {k: round(v, 3) for k, v in prep.items()},
                "train_cells_per_s": {k: round(float(np.median(v))) for k, v in rates.items()},
                "train_cells_per_s_rounds": {k: [round(x) for x in v] for k, v in rates.items()}}), flush=True)
            for net in nets.values():
                net.engine.close()
            del data, nets
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
