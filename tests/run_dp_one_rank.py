"""The data-parallel step (dca_train_step_dp) on ONE GPU over a one-rank NCCL communicator, for the launch plans only
that step selects:
  DCA_DP_RESERVE_SMS=n  the hidden-stack backward runs at most SMs - n CTAs (its strips then differ from the forward's)
                        and the encoder backward's grid is SMs - n CTAs;
  DCA_DP_SPLIT_HEADS=1  one head-backward launch per head (n_heads = 1 each).
The library reads these switches once per process, so tests/test_gpu_parity.py runs this script once per setting:
    python tests/run_dp_one_rank.py OUT.npz
Three steps on the same batch and weights (direct call, graph capture, graph replay; no update in between) save their
gradient buffers, the BatchNorm state after the first step and the number of captured step graphs to OUT.npz."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle import dca_oracle as O          # noqa: E402
from tests.util import synth_counts         # noqa: E402

B, G, N, HIDDEN = 4096, 2000, 4600, (64, 32, 64)


def problem():
    """Batch of B rows gathered from N cells, zinb-conddisp weights with non-zero biases (seeded: the same in every
    process)."""
    Y = synth_counts(N, G, 61); X, sf = O.normalize_inputs(Y)
    rows = np.random.default_rng(4).permutation(N)[:B].astype(np.int32)
    p0 = O.init_params(G, G, HIDDEN, "zinb-conddisp", True, seed=6, dtype=np.float32)
    rng = np.random.default_rng(7)
    for k in p0:
        if k.endswith(("/bias", "/bn_beta")):
            p0[k] = rng.normal(0, 0.2, p0[k].shape).astype(np.float32)
    return X, Y, sf, rows, p0


def main(out_path):
    from dca_b200.engine import DeviceEngine
    X, Y, sf, rows, p0 = problem()
    dev = torch.device("cuda", 0)
    eng = DeviceEngine(G, G, HIDDEN, "zinb-conddisp", True, max_batch=B, seed=None, device=dev)
    eng.set_weights(p0)
    assert eng.comm_init(single_rank=True)
    Xd, Yd, sfd = (torch.from_numpy(a).to(dev) for a in (X, Y, sf))
    rd = torch.from_numpy(rows).to(dev)
    side = torch.cuda.Stream(dev)            # (the legacy default stream cannot be captured)
    grads, bn = [], None
    with torch.cuda.stream(side):
        for it in range(3):
            eng.train_step_allreduce(Xd, Yd, sfd, rows=rd)
            side.synchronize()
            grads.append(eng.grads.cpu().numpy())
            if it == 0:
                bn = eng.bn_state.cpu().numpy()
    np.savez(out_path, grads=np.stack(grads), bn_state=bn, step_graphs=eng.info()["step_graphs"])
    eng.close()


if __name__ == "__main__":
    main(sys.argv[1])
