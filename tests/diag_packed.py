"""The packed device mode (packed_data.PackedDeviceDataset) against the resident and the streamed modes, one JSON line
per part.

    python tests/diag_packed.py [--size 68000x20000] [--big 1000000x20000] [--density 0.05] [--epochs 5] [--out DIR]

Part 1 (--size; seeded synthetic Poisson counts, tests/diag_preprocess.synth_poisson): wall time (synchronised host
clock, after a warm-up at 1/8 of the rows) of from_counts for DeviceDataset, StreamedDataset and PackedDeviceDataset and
the device bytes each holds; training cells/s at batch 4096 with bf16 X (device events around 60 steps + updates), the
three modes alternated three times; a torch.profiler table of packed steps (kernel time by name); predict time of each
mode; dca(epochs) end to end with 'preprocess': 'device' and with 'packed': True, whose weights are compared bit for bit.
Part 2 (--big): a CSR matrix built in row chunks at --density non-zeros (each entry non-zero with that probability, counts
1 + Poisson), larger than the resident dataset can hold: DeviceDataset.device_bytes against free memory, then
PackedDeviceDataset.from_counts, two training epochs and a latent-only predict, with the peak device memory.  The card's
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
from tests.diag_out_of_core import stream_rate, wall      # noqa: E402


def rate(step, n_rows, bs, steps):
    """Cells/s of `steps` calls of step(k) (training step + update), device events around the loop, one warm-up step."""
    nb = min(steps, n_rows // bs)
    step(0)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for k in range(1, nb):
        step(k)
    b.record()
    b.synchronize()
    return (nb - 1) * bs / (a.elapsed_time(b) / 1e3)


def part1(n, g, epochs, bs, steps, out_dir):
    from dca_b200.anndata_lite import AnnData
    from dca_b200.api import dca
    from dca_b200.device_data import DeviceDataset
    from dca_b200.network import AE_types
    from dca_b200.packed_data import PackedDeviceDataset
    from dca_b200.stream_data import StreamedDataset
    dev = torch.device("cuda:0")
    Y = synth_poisson(n, g)
    res = {"cells": n, "genes": g, "nonzero_frac": float(np.count_nonzero(Y) / Y.size)}
    warm = Y[: max(64, n // 8)]
    for cls in (DeviceDataset, PackedDeviceDataset):
        cls.from_counts(warm, dev, x_dtype="bfloat16")
    StreamedDataset.from_counts(warm, dev, x_dtype="bfloat16", batch=bs)
    res["device_from_counts_s"], dd = wall(lambda: DeviceDataset.from_counts(Y, dev, x_dtype="bfloat16"))
    res["stream_from_counts_s"], sd = wall(lambda: StreamedDataset.from_counts(Y, dev, x_dtype="bfloat16", batch=bs))
    res["packed_from_counts_s"], pdd = wall(lambda: PackedDeviceDataset.from_counts(Y, dev, x_dtype="bfloat16"))
    res["device_bytes"] = {"device": dd.Y.numel() * 4 + dd.X.numel() * 2 + dd.n * 20,
                           "stream": 0, "stream_host_packed": int(sd.pc.nbytes), "packed": pdd.device_bytes()}
    res["packed_bits"] = pdd.bits

    net = AE_types["zinb-conddisp"](input_size=g, output_size=g, hidden_size=(64, 32, 64), x_dtype="bfloat16")
    net.build(max_batch=bs, seed=0)
    eng = net.engine
    eng.set_optimizer("RMSprop")
    nc_pin = torch.from_numpy(np.ascontiguousarray(sd.n_counts_host)).pin_memory()
    order = torch.from_numpy(np.random.default_rng(0).permutation(n).astype(np.int32)).to(dev)
    torch.cuda.set_stream(torch.cuda.Stream(dev))         # capturable stream: step graphs as in train()

    def resident(k):
        eng.train_step(dd.X, dd.Y, dd.sf, rows=order[k * bs:(k + 1) * bs])
        eng.apply_update(1e-3, 5.0)

    def packed(k):
        eng.packed_train_step(pdd, order[k * bs:(k + 1) * bs])
        eng.apply_update(1e-3, 5.0)

    rates = {"device": [], "stream": [], "packed": []}
    for _ in range(3):
        rates["device"].append(rate(resident, n, bs, steps))
        rates["stream"].append(stream_rate(eng, sd, nc_pin, bs, steps, True))
        eng.set_input_transform_exact(pdd.mean, pdd.std, pdd.median, pdd.flags)
        rates["packed"].append(rate(packed, n, bs, steps))
    res["train_cells_per_s"] = {k: [round(v) for v in vs] for k, vs in rates.items()}

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in range(10):
            packed(k)
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
        if t:
            kern[ev.key[:60]] = round(t / 10.0, 1)
    res["packed_step_kernels_us_per_step"] = dict(sorted(kern.items(), key=lambda kv: -kv[1])[:12])

    for name, kw in (("device", dict(device_data=dd)), ("stream", dict(stream_data=sd)), ("packed", dict(packed_data=pdd))):
        net._run_predict(None, True, False, True, True, **kw)                # warm-up (sizes the engine for predict)
        res["predict_%s_s" % name], _ = wall(lambda: net._run_predict(None, True, False, True, True, **kw))
    del dd, sd, pdd, net, eng
    torch.cuda.empty_cache()

    weights = {}
    for name, kw in (("device", {"preprocess": "device"}), ("packed", {"preprocess": "device", "packed": True})):
        a = AnnData(Y.copy())
        res["dca_%s_s" % name], net = wall(lambda: dca(a, ae_type="zinb-conddisp", epochs=epochs, batch_size=bs,
                                                       network_kwds={"x_dtype": "bfloat16"}, training_kwds=kw,
                                                       return_model=True))
        weights[name] = net.engine.get_weights()
        if out_dir:
            np.savez(os.path.join(out_dir, "weights_%s.npz" % name), **{k.replace("/", "__"): v for k, v in weights[name].items()})
        del a, net
        torch.cuda.empty_cache()
    res["dca_weights_bit_identical"] = all(np.array_equal(weights["device"][k], weights["packed"][k])
                                           for k in weights["device"])
    return res


def big_csr(n, g, density, seed=1, chunk=16384):
    """n x g scipy CSR of counts 1 + Poisson(gene mean) at `density` non-zeros (each entry non-zero with that
    probability: geometric gaps between a row's genes, so every row comes out sorted), built chunk by chunk into
    preallocated arrays."""
    import scipy.sparse as sp
    rng = np.random.default_rng(seed)
    gene_mean = np.exp(rng.normal(-0.5, 1.0, size=g))
    m = int(g * density + 10 * np.sqrt(g * density) + 64)          # gaps drawn per row: their sum passes g almost surely
    cap = int(n * g * density * 1.01) + (1 << 20)
    indptr = np.zeros(n + 1, np.int64)
    indices = np.empty(cap, np.int32)
    data = np.empty(cap, np.float32)
    pos = 0
    for s in range(0, n, chunk):
        e = min(n, s + chunk)
        cols = np.cumsum(rng.geometric(density, size=(e - s, m)), axis=1) - 1
        keep = cols < g
        c = cols[keep].astype(np.int32)                           # row-major: by row, then gene
        if pos + c.size > cap:
            raise RuntimeError("capacity estimate exceeded")
        indptr[s + 1:e + 1] = pos + np.cumsum(keep.sum(1))
        indices[pos:pos + c.size] = c
        data[pos:pos + c.size] = 1 + rng.poisson(gene_mean[c])
        pos += c.size
    return sp.csr_matrix((data[:pos], indices[:pos], indptr), shape=(n, g), copy=False)


def part2(n, g, density, bs):
    from dca_b200.device_data import DeviceDataset
    from dca_b200.network import AE_types
    from dca_b200.packed_data import PackedDeviceDataset
    from dca_b200.train import train
    dev = torch.device("cuda:0")
    t0 = time.perf_counter()
    m = big_csr(n, g, density)
    res = {"cells": n, "genes": g, "nonzero_frac": m.nnz / (n * g), "generate_s": round(time.perf_counter() - t0, 1)}
    res["device_dataset_bytes"] = int(DeviceDataset.device_bytes(m, "bfloat16"))
    res["free_bytes_before"] = int(torch.cuda.mem_get_info(dev)[0])
    torch.cuda.reset_peak_memory_stats(dev)
    res["packed_from_counts_s"], pdd = wall(lambda: PackedDeviceDataset.from_counts(m, dev, x_dtype="bfloat16"))
    res["packed_bits"], res["packed_device_bytes"] = pdd.bits, pdd.device_bytes()
    res["peak_from_counts_bytes"] = int(torch.cuda.max_memory_allocated(dev))
    del m
    net = AE_types["zinb-conddisp"](input_size=g, output_size=g, hidden_size=(64, 32, 64), x_dtype="bfloat16")
    net.build(max_batch=bs, seed=0)
    np.random.seed(0)
    res["train_2_epochs_s"], hist = wall(lambda: train(None, net, packed_data=pdd, epochs=2, batch_size=bs,
                                                       verbose=False))
    res["loss"] = [round(v, 5) for v in hist.history["loss"]]
    res["predict_latent_s"], out = wall(lambda: net._run_predict(None, False, False, False, True, packed_data=pdd))
    res["latent_shape"] = list(out["latent"].shape)
    res["peak_device_bytes"] = int(torch.cuda.max_memory_allocated(dev))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", default="68000x20000")
    ap.add_argument("--big", default="1000000x20000", help="'' skips part 2")
    ap.add_argument("--density", type=float, default=0.05)
    ap.add_argument("--epochs", type=int, default=5)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("diag_packed needs a CUDA device")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    name, limit = card()
    if a.size:
        n, g = (int(v) for v in a.size.split("x"))
        print(json.dumps(dict(part1(n, g, a.epochs, a.batch, a.steps, a.out), gpu=name, power_limit=limit)), flush=True)
    if a.big:
        n, g = (int(v) for v in a.big.split("x"))
        print(json.dumps(dict(part2(n, g, a.density, a.batch), gpu=name, power_limit=limit)), flush=True)


if __name__ == "__main__":
    main()
