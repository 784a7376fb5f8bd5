"""2-rank (or N-rank) NUMERICAL parity of the data-parallel step on real GPUs over NCCL -- launched under torchrun
(tests/test_gpu_dist.py does it when >= 2 GPUs are visible):
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 tests/run_dist_parity.py

Every rank runs dca_train_step_dp (phase 1 -> all-reduce(head bucket) || phase 2 -> all-reduce(rest), one CUDA graph)
on ITS slice of a global batch; the all-reduced gradient x 1/R must equal
  (a) the gradient a single engine computes on the WHOLE global batch on one GPU, and
  (b) the float64 oracle's gradient of the global batch (SURVEY.md 8e: the loss is a mean over (cell, gene) elements,
      so the global gradient is the mean of the shard gradients),
with BatchNorm off (per-rank batch statistics are the documented default with BatchNorm on, which is deliberately not
the global-batch model).  Also: direct call, graph capture and graph replay give the same numbers, the replicas stay
bit-identical after the update, and dca_allreduce alone sums the buffer."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import dca_oracle as O          # noqa: E402  (test infrastructure: the checker)
from tests.util import synth_counts         # noqa: E402


def main():
    rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"]); local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from dca_b200.engine import DeviceEngine
    ok = True
    msgs = []
    # batchnorm off: plain data parallelism; batchnorm on + sync_bn: BatchNorm statistics all-reduced over the ranks
    # (forward and backward), i.e. exactly the single-GPU model at the global batch size (SURVEY.md 8e)
    # tcgen05 self-consistency 2e-3: the encoder backward rounds dA1 to bf16; the two runs sum dH3 in different orders
    # (per-rank partials plus the all-reduce against one engine's slots, 1e-7), which flips single bf16 roundings of dA1
    # (2^-9 of that element)
    for gemm_path, G, hidden, bn, tol_self, tol_oracle in (("generic", 200, (16, 8, 16), False, 2e-5, 2e-3),
                                                           ("tcgen05", 264, (64, 32, 64), False, 2e-3, 3e-2),
                                                           ("generic", 200, (16, 8, 16), True, 5e-5, 2e-3),
                                                           ("tcgen05", 264, (64, 32, 64), True, 2e-3, 3e-2)):
        B = 96
        Y = synth_counts(world * B, G, 7); X, sf = O.normalize_inputs(Y)
        p0 = O.init_params(G, G, hidden, "zinb-conddisp", bn, seed=1, dtype=np.float32)
        eng = DeviceEngine(G, G, hidden, "zinb-conddisp", bn, max_batch=B, seed=None, gemm_path=gemm_path, device=dev, sync_bn=bn)
        eng.set_weights(p0)
        assert eng.comm_init()
        lo, hi = rank * B, (rank + 1) * B
        Xd = torch.from_numpy(X[lo:hi]).to(dev); Yd = torch.from_numpy(Y[lo:hi]).to(dev); sfd = torch.from_numpy(sf[lo:hi]).to(dev)
        side = torch.cuda.Stream(dev)
        grads = []
        with torch.cuda.stream(side):
            for it in range(3):                                   # direct call, graph capture, graph replay
                eng.train_step_allreduce(Xd, Yd, sfd)
                side.synchronize()
                grads.append(eng.grads.clone())
        P = eng.n_params
        for it in (1, 2):
            d = (grads[it][:P] - grads[0][:P]).abs().max().item() / grads[0][:P].abs().max().item()
            if d > 2e-5:           # (the step sums every gradient in a fixed order, so the calls are expected to agree exactly)
                ok = False; msgs.append("%s: call %d differs from the direct call by %.2e" % (gemm_path, it, d))
        g_dp = (grads[2][:P] / world).cpu().numpy()
        loss_dp = float(grads[2][P].item()) / world
        # (a) one engine, whole global batch, one GPU
        big = DeviceEngine(G, G, hidden, "zinb-conddisp", bn, max_batch=world * B, seed=None, gemm_path=gemm_path, device=dev)
        big.set_weights(p0)
        big.train_step(torch.from_numpy(X).to(dev), torch.from_numpy(Y).to(dev), torch.from_numpy(sf).to(dev))
        torch.cuda.synchronize(dev)
        g_one = big.grads[:P].cpu().numpy(); loss_one = big.read_loss()
        # (b) float64 oracle of the global batch (same bf16 rounding points on the tcgen05 path)
        net = O.OracleNet(G, G, hidden, "zinb-conddisp", bn, dtype=np.float64, params=p0, emulate_bf16=(gemm_path == "tcgen05"))
        loss_o, g_o = net.loss_and_grads(X.astype(np.float64), Y.astype(np.float64), sf.astype(np.float64))
        worst_self = worst_or = 0.0
        for name, off, r, c in eng.param_info:
            if bn and name.endswith("/bias") and not name.startswith(("mean", "dispersion", "pi")):
                continue                                  # exactly zero in exact arithmetic (BatchNorm removes it): pure noise
            a = g_dp[off: off + r * c]; b = g_one[off: off + r * c]; o = g_o[name].reshape(-1)
            worst_self = max(worst_self, float(np.max(np.abs(a - b)) / (np.max(np.abs(b)) + 1e-30)))
            worst_or = max(worst_or, float(np.max(np.abs(a - o)) / (np.max(np.abs(o)) + 1e-30)))
        if worst_self > tol_self or abs(loss_dp - loss_one) > 1e-5 * abs(loss_one):
            ok = False
        if worst_or > tol_oracle or abs(loss_dp - loss_o) > 2e-4 * abs(loss_o):
            ok = False
        msgs.append("%s%s: all-reduced/R vs one-GPU global batch: grads %.2e (tol %.0e), loss %.2e; vs float64 oracle: grads %.2e "
                    "(tol %.0e), loss %.2e" % (gemm_path, " + sync_bn" if bn else "", worst_self, tol_self, abs(loss_dp - loss_one) / abs(loss_one), worst_or,
                                                tol_oracle, abs(loss_dp - loss_o) / abs(loss_o)))
        # replicas identical after the update
        eng.apply_update(1e-3, 5.0, 1.0 / world)
        torch.cuda.synchronize(dev)
        ref = eng.params.clone(); dist.broadcast(ref, 0)
        if not torch.equal(ref, eng.params):
            ok = False; msgs.append("%s: replicas differ after the update" % gemm_path)
        # dca_allreduce alone
        eng.grads.fill_(float(rank + 1)); eng.allreduce_grads(); torch.cuda.synchronize(dev)
        if abs(eng.grads[0].item() - world * (world + 1) / 2) > 1e-6:
            ok = False; msgs.append("%s: dca_allreduce sum wrong" % gemm_path)
        eng.close(); big.close()
    flag = torch.tensor([1.0 if ok else 0.0], device=dev); dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        for m in msgs:
            print("dist parity:", m)
        print("DIST PARITY %s (world=%d)" % ("OK" if flag.item() == 1.0 else "FAILED", world))
    dist.barrier(); dist.destroy_process_group()
    sys.exit(0 if flag.item() == 1.0 else 1)


if __name__ == "__main__":
    main()
