"""The out-of-core mode (stream_data.StreamedDataset) against the resident device path, one JSON line per size.

    python tests/diag_out_of_core.py [--sizes 68000x20000] [--epochs 5] [--batch 4096] [--steps 60]

Per size (seeded synthetic Poisson counts, tests/diag_preprocess.synth_poisson): wall time (synchronised host clock,
after a warm-up at 1/8 of the rows) of io.pack_rows, of each statistics pass over the packed counts and of
StreamedDataset.from_counts end to end, against DeviceDataset.from_counts and host io.normalize; streamed-step
cells/s with the exact transform (dca_set_input_transform_exact) against the float transform
(dca_set_input_transform) on the same packed bytes, the two alternated three times; streamed predict against
predict from the DeviceDataset; dca(epochs) with training_kwds preprocess 'host', 'device' and 'device' + stream.  The card's
name and power limit are read in the same run.  Needs a GPU.
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


def stream_rate(eng, sd, nc_pin, bs, steps, exact):
    """Cells/s of `steps` streamed training steps + updates (device events around the loop)."""
    if exact:
        eng.set_input_transform_exact(sd.mean, sd.std, sd.median, sd.flags)
        sf = None
    else:
        eng.set_input_transform(sd.mean.astype(np.float32), sd.std, True, True)
        sf = torch.from_numpy(sd.size_factors_host).pin_memory()
    nb = min(steps, (sd.n + bs - 1) // bs)
    eng.stream_begin(sd.pc, sf, bs)
    if exact:
        eng.stream_row_totals(nc_pin)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    eng.stream_step(0, 1); eng.apply_update(1e-3, 5.0)           # warm-up step
    a.record()
    for k in range(1, nb):
        eng.stream_step(k, k + 1 if k + 1 < nb else -1)
        eng.apply_update(1e-3, 5.0)
    b.record()
    eng.stream_end()
    b.synchronize()
    rows = min(sd.n, nb * bs) - bs
    return rows / (a.elapsed_time(b) / 1e3)


def measure(n, g, epochs, batch, steps):
    from dca_b200 import io
    from dca_b200.anndata_lite import AnnData
    from dca_b200.api import dca
    from dca_b200.device_data import DeviceDataset
    from dca_b200.network import AE_types
    from dca_b200.stream_data import StreamedDataset, _moments, _totals
    dev = torch.device("cuda:0")
    Y = synth_poisson(n, g)
    res = {"cells": n, "genes": g, "nonzero_frac": float(np.count_nonzero(Y) / Y.size)}
    warm = Y[: max(64, n // 8)]
    StreamedDataset.from_counts(warm, dev, batch=batch)
    DeviceDataset.from_counts(warm, dev)

    res["pack_s"], pc = wall(lambda: io.pack_rows(Y, "auto", batch=batch))
    res["packed_bytes_per_entry"] = pc.nbytes / Y.size
    res["totals_pass_s"], (nc, _, _) = wall(lambda: _totals(pc, dev))
    med = float(np.median(nc))
    res["moment_passes_s"], _ = wall(lambda: _moments(pc, nc, med, 7, dev))
    res["stream_from_counts_s"], sd = wall(lambda: StreamedDataset.from_counts(Y, dev, batch=batch))
    res["device_from_counts_s"], dd = wall(lambda: DeviceDataset.from_counts(Y, dev))
    t0 = time.perf_counter()
    io.normalize(AnnData(Y.copy()), filter_min_counts=False)
    res["host_normalize_s"] = time.perf_counter() - t0

    net = AE_types["zinb-conddisp"](input_size=g, output_size=g, hidden_size=(64, 32, 64), x_dtype="bfloat16")
    net.build(max_batch=batch, seed=0)
    eng = net.engine
    nc_pin = torch.from_numpy(np.ascontiguousarray(sd.n_counts_host)).pin_memory()
    sd16 = StreamedDataset.from_counts(Y, dev, x_dtype="bfloat16", batch=batch)
    rates = {"exact": [], "float": []}
    for _ in range(3):
        for kind in ("exact", "float"):
            rates[kind].append(stream_rate(eng, sd16, nc_pin, batch, steps, kind == "exact"))
    res["stream_step_cells_per_s"] = {k: [round(v) for v in vs] for k, vs in rates.items()}

    dd16 = DeviceDataset.from_counts(Y, dev, x_dtype="bfloat16")
    net._run_predict(None, True, False, True, True, device_data=dd16)            # warm-up (sizes the engine for predict)
    net._run_predict(None, True, False, True, True, stream_data=sd16)
    res["predict_device_s"], _ = wall(lambda: net._run_predict(None, True, False, True, True, device_data=dd16))
    res["predict_stream_s"], _ = wall(lambda: net._run_predict(None, True, False, True, True, stream_data=sd16))
    del dd, dd16, net, eng
    torch.cuda.empty_cache()

    for name, kw in (("host", {}), ("device", {"preprocess": "device"}),
                     ("device_stream", {"preprocess": "device", "stream": True})):
        a = AnnData(Y.copy())
        res["dca_%s_s" % name], _ = wall(lambda: dca(a, ae_type="zinb-conddisp", epochs=epochs, batch_size=batch,
                                                      training_kwds=kw))
        del a
        torch.cuda.empty_cache()
    name, limit = card()
    res["gpu"], res["power_limit"] = name, limit
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="68000x20000")
    ap.add_argument("--epochs", type=int, default=5)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=60)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("diag_out_of_core needs a CUDA device")
    for sz in a.sizes.split(","):
        n, g = (int(v) for v in sz.split("x"))
        print(json.dumps(measure(n, g, a.epochs, a.batch, a.steps)), flush=True)


if __name__ == "__main__":
    main()
