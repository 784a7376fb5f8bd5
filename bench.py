#!/usr/bin/env python
"""Benchmark of the DCA training hot path on H100 (see DESIGN.md).

  python bench.py --gpus N --steps K --warmup W            # our CUDA path
  python bench.py --impl reference --gpus N ...            # CPU arm: torch-CPU restatement of the
                                                           # reference step (TensorFlow is not installable)
  python bench.py ... --dump-outputs DIR                   # also write the last timed step's results as .npy

A "step" is one training batch of the hot path: forward (Dense stack, BatchNorm, three-head
output activations), ZINB loss + gradient, backward, gradient all-reduce (N > 1), clip + RMSprop.
Metric: cells/sec = steps * batch * n_gpus / device time (CUDA events, max over ranks).
Workload (``--workload auto``): at N = 1 synthetic 68k cells x 20k genes (PBMC shape), zinb-conddisp,
hidden 64,32,64 (X bf16 + Y fp32 = 8.2 GB of HBM); under torchrun (N > 1) every rank holds one shard of
1M x 20k over 8 GPUs = 125k x 20k per GPU (15 GB).  Every step trains 4096 cells per GPU in both cases (weak scaling), so the per-GPU work of
a step is identical at every N.  Both arms (ours / --impl reference) print the SAME metric string.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

WORKLOADS = {
    # name: (cells per GPU, genes, ae_type, description)
    "c2": (10000, 2000, "zinb-conddisp", "synthetic 10k cells x 2k genes ZINB-conddisp, hidden=64,32,64"),
    "c3": (68000, 20000, "zinb-conddisp", "synthetic 68k cells x 20k genes ZINB-conddisp (PBMC shape)"),
    "c5shard": (125000, 20000, "zinb-conddisp", "synthetic 125k cells x 20k genes per GPU (1M / 8 shard)"),
}
HIDDEN = (64, 32, 64)
# ONE metric string for both arms (the driver divides the two values only when metric / unit / direction agree)
METRIC = "cells/sec (ZINB AE epoch, device-timed)"
METRIC_NOTE = ("cells per second through the training step of the ZINB autoencoder epoch loop: forward + ZINB loss + backward "
               "+ gradient all-reduce (N > 1) + clip/RMSprop, batch 4096 cells per GPU; ours: CUDA events, max over ranks; "
               "reference arm: host wall clock of the torch-CPU restatement (TensorFlow is not installable in this image)")


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--workload", default=os.environ.get("DCA_BENCH_WORKLOAD", "auto"), choices=["auto"] + sorted(WORKLOADS),
                    help="auto: c3 (68k x 20k, the largest single-GPU config) at N = 1, c5shard (125k x 20k per GPU) for N > 1")
    ap.add_argument("--batch", type=int, default=4096, help="cells per GPU per step")
    ap.add_argument("--x-dtype", default="auto", choices=["auto", "float32", "bfloat16"],
                    help="storage type of the normalised input X in HBM; auto = bfloat16 on the tcgen05 path (the GEMM rounds X "
                         "to bf16 there anyway, so the results are bit-identical to float32 storage) and float32 otherwise")
    ap.add_argument("--gemm-path", default="auto", choices=["auto", "generic", "tcgen05"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--fused", action="store_true",
                    help="run head forward + loss + head backward as the ONE fused kernel (flash_zinb.cu) instead of K2 + K3 + K4")
    ap.add_argument("--e2e-format", default="auto", choices=["auto", "sparse", "dense", "u16", "4", "8", "16"],
                    help="host format of the streamed count matrix: packed bits per entry (io.pack_counts) or plain uint16")
    ap.add_argument("--cpu-seconds", type=float, default=15.0, help="budget of the CPU baseline sample")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last of them computed (loss, gradients, updated parameters, "
                         "BatchNorm moving statistics) as DIR/<name>.npy; the inputs depend only on the arguments")
    return ap.parse_args()


# ------------------------------------------------------------------------------------------------
def synth_on_device(n_cells, n_genes, device, seed, x_dtype=torch.float32, chunk=8192):
    """SURVEY.md 8d generator: gene log-means N(-2,1.5), depth LogNormal(0,.35), Gamma(2)-Poisson,
    20 % extra zeros.  Returns X = zscore(log1p(Y/sf)) (x_dtype), Y (fp32 raw counts), sf, zero fraction."""
    g = torch.Generator(device=device); g.manual_seed(seed)
    logm = torch.randn(n_genes, generator=g, device=device) * 1.5 - 2.0
    Y = torch.empty((n_cells, n_genes), dtype=torch.float32, device=device)
    for s in range(0, n_cells, chunk):
        e = min(s + chunk, n_cells)
        depth = torch.exp(torch.randn(e - s, 1, generator=g, device=device) * 0.35)
        scale = depth * torch.exp(logm)[None, :] / 2.0
        lam = torch._standard_gamma(torch.full((e - s, n_genes), 2.0, device=device), generator=g) * scale
        y = torch.poisson(lam, generator=g)
        y[torch.rand(e - s, n_genes, generator=g, device=device) < 0.2] = 0
        Y[s:e] = y
    dead = (Y.sum(0) == 0).nonzero().flatten()            # reference asserts no all-zero genes (dca/api.py:163-164)
    if dead.numel():
        Y[torch.randint(0, n_cells, (dead.numel(),), generator=g, device=device), dead] = 1
    n_counts = Y.sum(1)
    empty = (n_counts == 0).nonzero().flatten()
    if empty.numel():
        Y[empty, torch.randint(0, n_genes, (empty.numel(),), generator=g, device=device)] = 1
        n_counts = Y.sum(1)
    sf = (n_counts / n_counts.median()).float()
    # X = zscore(log1p(Y / sf)), per gene, ddof=1 -- dca/io.py:99-109
    mean = torch.zeros(n_genes, dtype=torch.float64, device=device); sq = torch.zeros_like(mean)
    for s in range(0, n_cells, chunk):
        l = torch.log1p(Y[s:s + chunk] / sf[s:s + chunk, None]).double()
        mean += l.sum(0); sq += (l * l).sum(0)
    mean /= n_cells
    var = (sq - n_cells * mean * mean) / (n_cells - 1)
    std = var.clamp_min(1e-12).sqrt()
    X = torch.empty((n_cells, n_genes), dtype=x_dtype, device=device)
    for s in range(0, n_cells, chunk):
        l = torch.log1p(Y[s:s + chunk] / sf[s:s + chunk, None]).double()
        X[s:s + chunk] = ((l - mean) / std).to(x_dtype)
    zero_frac = float((Y == 0).float().mean().item())
    return X, Y, sf.contiguous(), zero_frac, mean.float().cpu().numpy(), std.float().cpu().numpy()


class ClockSampler:
    """nvidia-smi clocks / throttle reasons DURING the timed region (read-only queries)."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index=0):
        self.p = None; self.idx = gpu_index

    def start(self):
        try:
            self.p = subprocess.Popen(["nvidia-smi", "-i", str(self.idx), "--query-gpu=" + self.Q, "--format=csv,noheader,nounits",
                                       "-lms", "100"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        except Exception:
            self.p = None

    def stop(self):
        if self.p is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.25)
        self.p.terminate()
        try:
            out = self.p.communicate(timeout=5)[0]
        except Exception:
            out = ""
        sm, mx, reasons = [], [], set()
        for line in out.strip().splitlines():
            f = [x.strip() for x in line.split(",")]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1])); mx.append(float(f[2]))
            except ValueError:
                continue
            for name, val in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[5:9]):
                if val.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


def measured_peaks():
    try:
        with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as f:
            p = json.load(f)
        return float(p["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    except Exception:
        return 3350.0, "H100 SXM data sheet (3.35 TB/s HBM3), not measured"


# ------------------------------------------------------------------------------------------------
_THREADS_CACHE = {}


def pick_cpu_threads(net_factory, Xt, Yt, sft, probe_batch=1024):
    """Thread count of the CPU arm: the fastest of a few candidates, each timed over 3 warmed steps of a reduced
    batch (per-step cost is linear in the batch), chosen ONCE per process and then kept fixed."""
    ncpu = os.cpu_count() or 1
    cands = sorted({ncpu, max(1, ncpu // 2), max(1, min(ncpu, 32)), max(1, min(ncpu, 16))}, reverse=True)
    key = (Xt.shape[1], probe_batch)
    if key in _THREADS_CACHE:
        return _THREADS_CACHE[key], cands
    net = net_factory()
    b = min(probe_batch, Xt.shape[0])
    best, threads = None, cands[0]
    for c in cands:
        torch.set_num_threads(c)
        net.train_step(Xt[:b], Yt[:b], sft[:b])                      # warm-up at this thread count
        t = time.perf_counter()
        for _ in range(3):
            net.train_step(Xt[:b], Yt[:b], sft[:b])
        el = time.perf_counter() - t
        if best is None or el < best:
            best, threads = el, c
    _THREADS_CACHE[key] = threads
    return threads, cands


def cpu_reference_arm(n_genes, ae_type, batch, seconds, steps=None, warmup=1, seed=0):
    """torch-CPU restatement of the reference training step on the box's host cores, on a bounded sample:
    batches of `batch` cells drawn from a min(16384, 4*batch)-row slice of the same synthetic shape.
    steps=None: run for about `seconds` of CPU work (the cpu_baseline leg of our arm); otherwise exactly
    `warmup` untimed + `steps` timed steps (the --impl reference arm)."""
    from oracle import dca_oracle as O
    from oracle.torch_ref import TorchRefNet
    from tests.util import synth_counts
    ncpu = os.cpu_count() or 1
    # bounded sample: the CPU needs seconds per 4096 x 20000 step, so its steps are 1024-cell batches there (cells/sec
    # does not depend on the batch a CPU step is cut into; stated in `sample`)
    gpu_batch = batch
    if n_genes >= 10000:
        batch = min(batch, 1024)
    n = min(16384, 4 * batch)
    Y = synth_counts(n, n_genes, seed)
    X, sf = O.normalize_inputs(Y)
    p0 = O.init_params(n_genes, n_genes, HIDDEN, ae_type, True, seed=0, dtype=np.float32)
    Xt, Yt, sft = torch.from_numpy(X), torch.from_numpy(Y), torch.from_numpy(sf)
    threads, cands = pick_cpu_threads(lambda: TorchRefNet(p0, HIDDEN, ae_type, True, dtype=torch.float32), Xt, Yt, sft)
    torch.set_num_threads(threads)
    net = TorchRefNet(p0, HIDDEN, ae_type, True, dtype=torch.float32)
    rng = np.random.default_rng(0)

    def one():
        idx = torch.from_numpy(rng.permutation(n)[:batch])
        return net.train_step(Xt[idx], Yt[idx], sft[idx])

    for _ in range(warmup):
        one()
    t0 = time.perf_counter(); done = 0
    while True:
        one(); done += 1
        el = time.perf_counter() - t0
        if (steps is not None and done >= steps) or (steps is None and el >= seconds):
            break
    return {"value": done * batch / el, "unit": "cells/sec", "cores": threads, "kind": "port",
            "sample": "%d timed steps (after %d warm-up) of %d-cell batches (the GPU arm steps %d cells) on a %d-cell x %d-gene "
                      "slice; torch-CPU fp32 restatement of the reference path (TensorFlow unavailable in image); %d of %d host "
                      "threads (fastest of %s over 3 warmed probe steps each, then fixed)"
                      % (done, warmup, batch, gpu_batch, n, n_genes, threads, ncpu, cands),
            "ms_per_step": 1e3 * el / done, "steps": done, "warmup": warmup}


def loss_kernel_standalone(eng, X, Y, sf, rows, genes, batch, peak):
    """The ZINB loss kernel alone (dca_zinb_loss_fwd_bwd) in the SURVEY 8d byte model: fp32 in, fp32 gradients
    out = 28 B per element, on the head outputs of a real batch; CUDA events, L2 flushed between launches."""
    import ctypes as C
    from dca_b200 import _lib
    lib = _lib.load(); dev = X.device
    m = torch.empty((batch, genes), device=dev); d = torch.empty_like(m); p = torch.empty_like(m)
    eng.predict(X, sf, rows=rows, mean=m, disp=d, pi=p)
    ones = torch.ones(sf.shape[0], device=dev)                       # mean_out above already carries sf
    gm, gd, gp = torch.empty_like(m), torch.empty_like(m), torch.empty_like(m)
    nb = C.c_size_t(); lib.dca_zinb_loss_workspace_bytes(batch, genes, C.byref(nb))
    ws = torch.empty(nb.value, dtype=torch.uint8, device=dev); loss = torch.zeros(1, dtype=torch.float64, device=dev)
    flush = torch.empty(160 * 1024 * 1024, dtype=torch.uint8, device=dev)
    st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    times = []
    for it in range(8):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rc = lib.dca_zinb_loss_fwd_bwd(Y.data_ptr(), Y.stride(0), rows.data_ptr(), ones.data_ptr(), m.data_ptr(), d.data_ptr(),
                                       p.data_ptr(), genes, batch, genes, 0, 0.0, 1.0 / (batch * genes), gm.data_ptr(),
                                       gd.data_ptr(), gp.data_ptr(), _lib.F32, None, loss.data_ptr(), ws.data_ptr(), nb.value, st)
        e1.record(); torch.cuda.synchronize(dev)
        _lib.check(rc, "dca_zinb_loss_fwd_bwd")
        if it >= 3:
            times.append(e0.elapsed_time(e1))
    ms = float(np.median(times)); byts = batch * genes * 28
    ach = byts / (ms * 1e-3) / 1e9
    return {"ms": ms, "bytes_per_element": 28, "achieved": ach, "unit": "GB/s", "frac": ach / peak,
            "note": "stand-alone launch incl. its partial-fold kernel, fp32 gradients, L2 flushed before every launch"}


DUMP_BUDGET_BYTES = 60_000_000   # all .npy payloads of one dump together stay under 64 MB


def dump_outputs(out_dir, eng):
    """The results a caller of the timed path holds after its last step: the batch loss, the gradient buffer of that
    step, the parameters after its update and the BatchNorm moving statistics.  The arrays share DUMP_BUDGET_BYTES,
    smallest first; an array that does not fit its share is replaced by a fixed, seeded sample of its elements (the
    same indices for the same array length and share)."""
    os.makedirs(out_dir, exist_ok=True)
    n = eng.n_params
    arrays = {"loss": np.array([eng.read_loss()], dtype=np.float64),
              "bn_state": eng.bn_state.float().cpu().numpy(),
              "grads": eng.grads[:n].float().cpu().numpy(),
              "params": eng.params[:n].float().cpu().numpy()}
    left = DUMP_BUDGET_BYTES
    for i, (name, v) in enumerate(arrays.items()):
        cap = left // (v.itemsize * (len(arrays) - i))            # equal share of what the earlier arrays left
        if v.size > cap:
            v = v[np.sort(np.random.default_rng(0).choice(v.size, cap, replace=False))]
        left -= v.nbytes
        np.save(os.path.join(out_dir, name + ".npy"), v)


# ------------------------------------------------------------------------------------------------
def main():
    a = parse()
    rank = int(os.environ.get("RANK", "0")); world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if a.workload == "auto":
        a.workload = "c3" if world == 1 else "c5shard"
    cells, genes, ae_type, desc = WORKLOADS[a.workload]
    batch = a.batch
    tc_shape = (a.gemm_path != "generic") and genes % 8 == 0 and HIDDEN[0] == 64 and HIDDEN[-1] == 64
    if a.x_dtype == "auto":
        a.x_dtype = "bfloat16" if tc_shape else "float32"
    # what the arithmetic really is: bf16 operands / fp32 accumulation in the gene-wide GEMMs (tensor cores), fp32 everywhere else
    dtype_label = "bf16-gemm/f32-acc/f32-loss" if tc_shape else "f32"
    config = {"workload": desc, "ae_type": ae_type, "hidden": list(HIDDEN), "cells_per_gpu": cells, "genes": genes,
              "batch_per_gpu": batch, "global_batch": batch * max(world, 1), "x_dtype": a.x_dtype,
              "optimizer": "RMSprop(lr=1e-3, clipvalue=5)", "batchnorm": "per-rank batch statistics",
              "parallelism": "dp%d" % max(world, 1),
              "l2": "dataset (X+Y %.0f MB/GPU) and per-step head tensors exceed the 50 MB L2; no explicit flush"
                    % (cells * genes * (4 + (2 if a.x_dtype == 'bfloat16' else 4)) / 1e6)}

    if a.impl == "reference":
        if rank != 0:
            return
        r = cpu_reference_arm(genes, ae_type, batch, a.cpu_seconds, steps=a.steps, warmup=a.warmup)
        line = {"impl": "reference", "metric": METRIC, "metric_note": METRIC_NOTE,
                "value": r["value"], "unit": "cells/sec", "n_gpus": a.gpus, "steps": r["steps"], "warmup": r["warmup"],
                "ms_per_step": r["ms_per_step"], "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
                "dtype": "f32", "data": "synthetic", "config": config,
                "cpu_baseline": {k: r[k] for k in ("value", "unit", "cores", "kind", "sample")},
                "e2e": {"value": r["value"], "unit": "cells/sec", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
                "gpu_launches": 0}
        print(json.dumps(line)); return

    import torch.distributed as dist
    from dca_b200.engine import DeviceEngine, launch_count
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device; the product path has no CPU fallback")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)

    X, Y, sf, zero_frac, gmean, gstd = synth_on_device(cells, genes, dev, 1234 + rank, {"float32": torch.float32, "bfloat16": torch.bfloat16}[a.x_dtype])
    n_train = int(cells * 0.9)                                  # validation_split=0.1 tail, dca/train.py:96
    if a.fused:
        from dca_b200 import _lib as _dl
        _dl.set_tunable("fused_heads", 1)
    for kv in filter(None, os.environ.get("DCA_TUNABLES", "").split(",")):     # diagnosis only: name=value,...
        from dca_b200 import _lib as _dl
        _dl.set_tunable(kv.split("=")[0], int(kv.split("=")[1]))
    eng = DeviceEngine(genes, genes, HIDDEN, ae_type, True, max_batch=batch, x_dtype=a.x_dtype,
                       gemm_path=a.gemm_path, device=dev, seed=0)
    if world > 1:
        dist.broadcast(eng.params, 0); eng.params_changed()
        if os.environ.get("DCA_BENCH_TORCH_ALLREDUCE", "0") != "1":
            eng.comm_init()      # NCCL all-reduce enqueued by the library inside the step's CUDA graph (dca_train_step_dp)
    lr, clip, gscale = 1e-3, 5.0, 1.0 / world
    total = a.steps + a.warmup
    gperm = torch.Generator(device=dev); gperm.manual_seed(99 + rank)
    need = total * batch
    stream_idx = torch.cat([torch.randperm(n_train, generator=gperm, device=dev) for _ in range(need // n_train + 1)])[:need]
    stream_idx = stream_idx.to(torch.int32).contiguous()

    # Everything below runs on a NON-default stream: the legacy default stream serialises against the engine's
    # internal copy stream (no H2D/compute overlap) and cannot be captured into a CUDA graph.
    torch.cuda.synchronize(dev)
    side = torch.cuda.Stream(dev)
    torch.cuda.set_stream(side)

    def step(i):
        rows = stream_idx[i * batch:(i + 1) * batch]
        if world > 1:
            eng.train_step_allreduce(X, Y, sf, rows=rows)     # head-gradient all-reduce overlaps the backward tail
        else:
            eng.train_step(X, Y, sf, rows=rows)
        eng.apply_update(lr, clip, gscale)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize(dev)

    for i in range(a.warmup):
        step(i)
    barrier()
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    l0 = launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    barrier()
    e0.record()
    for i in range(a.warmup, total):
        step(i)
    e1.record()
    barrier()
    ms = e0.elapsed_time(e1)
    launches = launch_count() - l0
    if a.dump_outputs and rank == 0:
        dump_outputs(a.dump_outputs, eng)
    clocks = sampler.stop() if rank == 0 else None
    final_loss = eng.read_loss()
    if world > 1:
        t = torch.tensor([ms], dtype=torch.float64, device=dev); dist.all_reduce(t, op=dist.ReduceOp.MAX); ms = float(t.item())
    value = a.steps * batch * world / (ms * 1e-3)

    # ---- profiled pass (separate from the timed region): per-phase device time, loss-kernel roofline
    _skip = os.environ.get("DCA_BENCH_SKIP", "").split(",")        # diagnosis only
    eng.profile(True)
    for i in range(a.warmup, total if "profile" not in _skip else a.warmup + 1):
        step(i)
    torch.cuda.synchronize(dev)
    prof = eng.profile_read()
    eng.profile(False)
    peak, peak_src = measured_peaks()
    nh = 3
    einfo = eng.info()
    loss_ms, loss_n = prof["loss_fwd_bwd"]
    # y (4 B) + m, d, pi in (fp32) + dzm, dzd, dzp out (fp32 generic path | bf16 tcgen05 path) -- SURVEY 8d
    loss_bytes = batch * genes * (4 + 4 * nh + einfo["grad_bytes"] * nh)
    ach = loss_bytes / (loss_ms / max(loss_n, 1) * 1e-3) / 1e9 if loss_ms > 0 else None
    step_ms_prof = sum(v[0] for v in prof.values()) / max(a.steps, 1)
    roofline = {"kernel": "zinb_loss_bwd_ring_kernel (phase loss_fwd_bwd: K3, the last block folds the partials)", "bound": "hbm", "achieved": ach,
                "peak": peak, "unit": "GB/s", "frac": (ach / peak) if ach else None,
                "peak_source": peak_src, "algorithmic_bytes_per_launch": loss_bytes,
                "bytes_per_element": 4 + 4 * nh + einfo["grad_bytes"] * nh, "engine": einfo,
                "share_of_step": (loss_ms / max(loss_n, 1)) / step_ms_prof if step_ms_prof > 0 else None}
    phases = {k: (v[0] / max(v[1], 1)) for k, v in prof.items()}
    if a.fused:
        # the fused kernel moves 4 B / element (the counts) and is bound by the fp32 / MUFU loss arithmetic, not by HBM
        # or the tensor pipe: its HBM fraction is reported for completeness only
        roofline["kernel"] = "flash_zinb_kernel (heads forward + ZINB loss/gradient + heads backward fused; issue-bound)"
        roofline["bytes_per_element"] = 4
        roofline["algorithmic_bytes_per_launch"] = batch * genes * 4
        roofline["achieved"] = (batch * genes * 4) / (loss_ms / max(loss_n, 1) * 1e-3) / 1e9 if loss_n else None
        roofline["frac"] = roofline["achieved"] / peak if roofline["achieved"] else None
    roofline["loss_kernel_fp32_io"] = (loss_kernel_standalone(eng, X, Y, sf, stream_idx[:batch], genes, batch, peak)
                                       if "standalone" not in _skip else None)

    # ---- end to end through the public streaming API: the raw counts live in pinned HOST memory (bit-packed by
    # io.pack_counts: 4/8/16 bits per entry + overflow list, or plain uint16), every step copies its batch
    # host->device (double-buffered, overlapping the previous step's compute), the device expands / normalises it
    # (dca/io.py:99-109 restated), runs the full training step, and the step's loss is read back device->host.
    e2e = None
    if not a.no_e2e:
        nb = max(2, min(8, cells // batch, (1 << 26) // (batch * genes)))    # host copy of <= 64 M entries (packing time)
        from dca_b200 import io as dio
        from dca_b200.hostmem import pin_near_gpu, near_gpu
        counts_np = Y[: nb * batch].cpu().numpy()
        t_pack = time.perf_counter()
        if a.e2e_format == "u16":
            assert float(counts_np.max()) < 65536
            cnt_h = pin_near_gpu(counts_np.astype(np.uint16), dev.index)
            fmt = "uint16 raw counts"; tile_bytes = batch * genes * 2
        else:
            cnt_h = dio.pack_counts(counts_np, a.e2e_format if a.e2e_format in ("auto", "sparse", "dense") else int(a.e2e_format),
                                    batch=batch)
            fmt = ("sparse raw counts: 1-bit non-zero map + 4-bit codes of the non-zero entries" if cnt_h.bits == 1
                   else "%d-bit packed raw counts" % cnt_h.bits) + " + overflow list (%d entries of %d, io.pack_counts)" % (
                len(cnt_h.entries), counts_np.size)
            tile_bytes = max(cnt_h.bytes_for_rows(i * batch, (i + 1) * batch) for i in range(nb))
        t_pack = time.perf_counter() - t_pack
        sf_h = pin_near_gpu(sf[: nb * batch].cpu(), dev.index)
        loss_h = pin_near_gpu(torch.zeros(64, dtype=torch.float32), dev.index)
        eng.set_input_transform(gmean, gstd, True, True)
        k_e2e = max(3, min(a.steps, 40))
        P = eng.n_params

        def e2e_run(k):
            eng.set_loss_ring(loss_h)           # the step's result, D2H: the update kernel stores the (all-reduced)
            eng.stream_begin(cnt_h, sf_h, batch)  # batch loss into this pinned host ring every step
            for i in range(k):
                eng.stream_step(i % nb, (i + 1) % nb if i + 1 < k else -1)
                if world > 1:
                    eng.allreduce_grads() if getattr(eng, "_comm", False) else dist.all_reduce(eng.grads)
                eng.apply_update(lr, clip, gscale)
            eng.stream_end()
            eng.set_loss_ring(None)

        # context: raw pinned host->device copy bandwidth of this box (64 MiB, best of 5)
        probe_h = pin_near_gpu(torch.empty(64 << 20, dtype=torch.uint8), dev.index); probe_d = torch.empty(64 << 20, dtype=torch.uint8, device=dev)
        h2d_best = 0.0
        for _ in range(5 if "probe" not in _skip else 0):
            p0, p1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            p0.record(); probe_d.copy_(probe_h, non_blocking=True); p1.record(); torch.cuda.synchronize(dev)
            h2d_best = max(h2d_best, (64 << 20) / (p0.elapsed_time(p1) * 1e-3) / 1e9)
        e2e_run(6)            # warm-up: both staging buffers have been through direct call + graph capture
        barrier()
        # three timed passes of k_e2e steps each (max over ranks per pass); the median pass is reported, all are kept
        runs = []
        for _ in range(3):
            f0, f1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            f0.record()
            e2e_run(k_e2e)
            f1.record(); barrier()
            t_run = f0.elapsed_time(f1)
            if world > 1:
                t = torch.tensor([t_run], dtype=torch.float64, device=dev); dist.all_reduce(t, op=dist.ReduceOp.MAX); t_run = float(t.item())
            runs.append(t_run)
        ems = float(np.median(runs))
        e2e = {"value": k_e2e * batch * world / (ems * 1e-3), "unit": "cells/sec", "steps": k_e2e,
               "h2d_bytes_per_step": tile_bytes + 4 * batch, "d2h_bytes_per_step": 4,
               "host_format": fmt + " + float32 size factors in pinned memory; Y and X are derived on the device",
               "host_pack_seconds_once": round(t_pack, 3), "host_rows": nb * batch,
               "api": "DeviceEngine.stream_begin / stream_step / apply_update (C ABI dca_stream_*, dca_set_loss_ring); "
                      "every step's loss lands in pinned host memory (written by the update kernel)",
               "last_loss": float(loss_h[(k_e2e - 1) % 64]), "h2d_gbs_measured": h2d_best,
               "ms_per_step": ems / k_e2e, "ms_per_step_passes": [round(r / k_e2e, 4) for r in runs]}

    cpu = None
    if rank == 0 and world == 1 and not a.no_cpu_baseline:
        cpu = cpu_reference_arm(genes, ae_type, batch, a.cpu_seconds)
        cpu = {k: cpu[k] for k in ("value", "unit", "cores", "kind", "sample")}

    if rank == 0:
        line = {"metric": METRIC, "metric_note": METRIC_NOTE,
                "value": value, "unit": "cells/sec", "n_gpus": world, "steps": a.steps, "warmup": a.warmup,
                "ms_per_step": ms / a.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
                "dtype": dtype_label, "data": "synthetic (zero fraction %.3f)" % zero_frac,
                "config": config, "clocks": clocks, "e2e": e2e, "gpu_launches": int(launches),
                "roofline": roofline, "cpu_baseline": cpu, "phase_ms": phases, "final_loss": final_loss,
                "impl": "ours"}
        print(json.dumps(line))
    if world > 1:
        dist.barrier(); dist.destroy_process_group()


if __name__ == "__main__":
    main()
