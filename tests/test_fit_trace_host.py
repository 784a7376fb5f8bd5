"""The engine calls train() makes for every input kind, against traces recorded once (tests/golden/fit_traces.json).

train() is driven on the CPU with a recording engine: every call and its arguments (small tensors as lists, large ones
as a digest) go into a trace, and ``read_epoch_acc`` returns a scripted sequence that makes ReduceLROnPlateau and
EarlyStopping fire.  The epoch part of a trace (from the first ``read_epoch_acc`` on) must equal the recorded one
call for call; the set-up before it must hold the same calls, with ``reset_optimizer`` after ``set_optimizer`` and
after every broadcast.  Rejected keyword combinations record the exception type and message.

Re-record with ``DCA_RECORD_TRACES=1 pytest tests/test_fit_trace_host.py``; the stream=True case packs its counts with
the native host packer of libdca_b200.so (built by the csrc Makefile), no device is used."""
import collections
import hashlib
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from tests.util import synth_counts

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fit_traces.json")
RECORD = os.environ.get("DCA_RECORD_TRACES") == "1"
N, G, BATCH = 40, 8, 8
# validation loss per epoch: best at epoch 1, then a plateau (reduce_lr=2 fires twice, early_stop=4 stops at epoch 5)
VAL = [1.0, 0.9, 0.95, 0.96, 0.97, 0.98, 0.99, 1.0]


def _enc(a):
    if isinstance(a, np.ndarray):
        a = torch.from_numpy(np.ascontiguousarray(a))
    if isinstance(a, torch.Tensor):
        t = a.detach().cpu().contiguous()
        if t.numel() <= 16:
            return {"dtype": str(t.dtype), "v": (t.float() if t.dtype == torch.bfloat16 else t).tolist()}
        return {"dtype": str(t.dtype), "shape": list(t.shape), "sha1": hashlib.sha1(t.view(torch.uint8).numpy()).hexdigest()}
    if isinstance(a, np.generic):
        return a.item()
    if a is None or isinstance(a, (bool, int, float, str)):
        return a
    if hasattr(a, "bits") and hasattr(a, "indptr"):                    # io.PackedCounts
        h = hashlib.sha1()
        for x in (a.packed, a.indptr, a.entries, getattr(a, "nib_indptr", None), getattr(a, "nibbles", None)):
            if x is not None:
                h.update(np.ascontiguousarray(x).tobytes())
        return {"packed_counts": a.bits, "rows": a.n_rows, "sha1": h.hexdigest()}
    return {"object": type(a).__name__}


class _Engine:
    def __init__(self, trace, n_in=G, n_out=G):
        self.trace, self.n_in, self.n_out = trace, n_in, n_out
        self.device, self.x_dtype, self.max_batch = torch.device("cpu"), torch.float32, BATCH
        self.params, self.grads, self.bn_state = torch.zeros(16), torch.zeros(18), torch.ones(4)
        self._acc = 0

    def _rec(self, name, *args, **kw):
        self.trace.append([name, [_enc(a) for a in args], {k: _enc(v) for k, v in sorted(kw.items())}])

    def set_optimizer(self, name):
        self._rec("set_optimizer", name)
        return 1e-3

    def read_epoch_acc(self, reset=True):
        self._rec("read_epoch_acc", reset=reset)
        k, self._acc = self._acc, self._acc + 1
        v = VAL[min(k // 2, len(VAL) - 1)]
        return [2.0 * (k + 1), 4.0, 3.0 * v, 3.0]

    def stream_capacity(self):
        self._rec("stream_capacity")
        return 4096, 4096

    def __getattr__(self, name):                # every other engine call is recorded and returns None
        if name.startswith("_"):
            raise AttributeError(name)
        return lambda *a, **kw: self._rec(name, *a, **kw)


class _Net:
    def __init__(self, eng):
        self.eng = eng

    def ensure_engine(self, max_batch):
        self.eng._rec("ensure_engine", max_batch=max_batch)
        return self.eng

    def penalty_value(self):
        return 0.0

    def summary(self):
        return "model summary"

    def save_weights(self, path):
        self.eng._rec("save_weights")


@pytest.fixture
def no_cuda(monkeypatch):
    """torch.cuda's stream calls as no-ops (recorded into the trace of the active case)."""
    state = SimpleNamespace(trace=None)

    def rec(name):
        def f(*a, **kw):
            if state.trace is not None:
                state.trace.append([name, [], {}])
        return f
    monkeypatch.setattr(torch.cuda, "synchronize", rec("cuda.synchronize"))
    monkeypatch.setattr(torch.cuda, "set_stream", rec("cuda.set_stream"))
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **kw: None)
    monkeypatch.setattr(torch.cuda, "Stream", lambda *a, **kw: None)
    return state


def _world2(monkeypatch, trace):
    from dca_b200 import dist as D

    def rec(name):
        def f(t, *a, **kw):
            trace.append([name, [_enc(t)], {}])
            return t
        return f
    monkeypatch.setattr(D, "rank_world", lambda: (0, 2))
    monkeypatch.setattr(D, "broadcast_", rec("dist.broadcast_"))
    monkeypatch.setattr(D, "all_reduce_sum_", rec("dist.all_reduce_sum_"))
    monkeypatch.setattr(D, "all_reduce_sum_host", lambda a, dev: (trace.append(["dist.all_reduce_sum_host", [_enc(a)], {}]),
                                                                 a)[1])
    monkeypatch.setattr(torch.distributed, "get_backend", lambda *a: "nccl")


# ---------------------------------------------------------------------- data
def _counts():
    return synth_counts(N, G, seed=3)


def _host_adata():
    from dca_b200 import io
    from dca_b200.anndata_lite import AnnData
    ad = AnnData(_counts())
    io.normalize(ad, filter_min_counts=False)
    return ad


def _device_data():
    from dca_b200.device_data import DeviceDataset, normalize_reference
    Y = _counts()
    r = normalize_reference(Y)
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a)).to(dt)     # noqa: E731
    return DeviceDataset(t(Y, torch.float32), t(r["X"], torch.float32), t(r["size_factors"], torch.float32),
                         t(r["n_counts"], torch.float64), t(r["mean"], torch.float64), t(r["std"], torch.float64),
                         torch.arange(N, dtype=torch.int32))


def _y_cols(cols):
    dd = _device_data()
    return dd._derive(Y=dd.Y[:, cols].contiguous(), y_cols=np.array(cols))


def _stats(ds):
    from dca_b200.device_data import normalize_reference
    r = normalize_reference(_counts())
    ds.n_counts_host, ds.size_factors_host = r["n_counts"], r["size_factors"]
    ds.mean, ds.std, ds.median, ds.flags = r["mean"], r["std"], float(np.median(r["n_counts"])), 7
    return ds


def _stream_data():
    from dca_b200 import io
    from dca_b200.stream_data import StreamedDataset
    sd = StreamedDataset(io.pack_counts(_counts(), native=False), None, None, None, None, None, None, torch.float32,
                         torch.device("cpu"))
    return _stats(sd)


def _packed_data():
    from dca_b200.packed_data import PackedDeviceDataset
    pd = PackedDeviceDataset.__new__(PackedDeviceDataset)
    pd.rows, pd.desc = torch.arange(N, dtype=torch.int32), SimpleNamespace(genes=G, n_rows=N)
    pd.x_dtype, pd.device = torch.float32, torch.device("cpu")
    return _stats(pd)


# ---------------------------------------------------------------------- cases
FIT = dict(epochs=8, reduce_lr=2, early_stop=4, batch_size=BATCH, verbose=False)


def _host(shuffle, split):
    return lambda: (_host_adata(), dict(shuffle=shuffle, validation_split=split))


CASES = {
    "host_shuffle_split": _host(True, 0.1),
    "host_shuffle_nosplit": _host(True, 0.0),
    "host_inorder_split": _host(False, 0.1),
    "host_inorder_nosplit": _host(False, 0.0),
    "host_world2": lambda: (_host_adata(), dict(world=2)),
    "host_stream": lambda: (_host_adata(), dict(stream=True)),
    "host_stream_inorder": lambda: (_host_adata(), dict(stream=True, shuffle=False)),
    "device_data_take": lambda: (None, dict(device_data=_device_data().take(np.arange(N - 1, 3, -1)))),
    "device_data_inorder": lambda: (None, dict(device_data=_device_data(), shuffle=False)),
    "device_data_y_cols": lambda: (_host_adata(), dict(device_data=_y_cols([1, 4, 6]), output_subset=["1", "4", "6"])),
    "stream_data": lambda: (None, dict(stream_data=_stream_data())),
    "stream_data_inorder": lambda: (None, dict(stream_data=_stream_data().take(np.arange(N)[::-1]), shuffle=False)),
    "packed_data": lambda: (None, dict(packed_data=_packed_data().take(np.arange(N)[::-1]))),
    "packed_data_inorder": lambda: (None, dict(packed_data=_packed_data(), shuffle=False)),
}

REJECTED = {
    "packed+device": lambda: dict(packed_data=_packed_data(), device_data=_device_data()),
    "packed+stream_data": lambda: dict(packed_data=_packed_data(), stream_data=_stream_data()),
    "packed+stream": lambda: dict(packed_data=_packed_data(), stream=True),
    "stream_data+device": lambda: dict(stream_data=_stream_data(), device_data=_device_data()),
    "device+stream": lambda: dict(device_data=_device_data(), stream=True),
    "device_world2": lambda: dict(device_data=_device_data(), world=2),
    "stream_data_world2": lambda: dict(stream_data=_stream_data(), world=2),
    "packed_world2": lambda: dict(packed_data=_packed_data(), world=2),
    "device_not_raw": lambda: dict(device_data=_device_data(), use_raw_as_output=False),
    "stream_data_not_raw": lambda: dict(stream_data=_stream_data(), use_raw_as_output=False),
    "packed_not_raw": lambda: dict(packed_data=_packed_data(), use_raw_as_output=False),
    "device_subset_no_adata": lambda: dict(device_data=_device_data(), output_subset=["1"]),
    "device_subset_wrong_y": lambda: dict(adata=_host_adata(), device_data=_device_data(), output_subset=["1"]),
    "device_y_cols_no_subset": lambda: dict(device_data=_y_cols([0, 1])),
    "stream_data_subset": lambda: dict(stream_data=_stream_data(), output_subset=["1"]),
    "packed_subset": lambda: dict(packed_data=_packed_data(), output_subset=["1"]),
    "device_cells": lambda: dict(adata=_host_adata()[np.arange(5)], device_data=_device_data()),
    "stream_data_cells": lambda: dict(adata=_host_adata()[np.arange(5)], stream_data=_stream_data()),
    "packed_cells": lambda: dict(adata=_host_adata()[np.arange(5)], packed_data=_packed_data()),
    "stream_data_genes": lambda: dict(stream_data=_stream_data(), n_in=16),
    "packed_genes": lambda: dict(packed_data=_packed_data(), n_out=4),
    "device_dtype": lambda: dict(device_data=_device_data(), x_dtype=torch.bfloat16),
    "stream_data_dtype": lambda: dict(stream_data=_stream_data(), x_dtype=torch.bfloat16),
    "packed_dtype": lambda: dict(packed_data=_packed_data(), x_dtype=torch.bfloat16),
    "device_device": lambda: dict(device_data=_device_data(), device=torch.device("meta")),
    "stream_data_device": lambda: dict(stream_data=_stream_data(), device=torch.device("meta")),
    "packed_device": lambda: dict(packed_data=_packed_data(), device=torch.device("meta")),
    "host_stream_subset": lambda: dict(adata=_host_adata(), stream=True, output_subset=["1"]),
    "unknown_keyword": lambda: dict(device_data=_device_data(), steps_per_epoch=3),
    "optimizer": lambda: dict(device_data=_device_data(), optimizer="LBFGS"),
    "tensorboard": lambda: dict(device_data=_device_data(), tensorboard=True),
}


def _run(monkeypatch, no_cuda, adata, kw):
    from dca_b200.train import train
    trace = []
    no_cuda.trace = trace
    kw = dict(kw)
    eng = _Engine(trace, kw.pop("n_in", G), kw.pop("n_out", G))
    eng.x_dtype = kw.pop("x_dtype", eng.x_dtype)
    eng.device = kw.pop("device", eng.device)
    if kw.pop("world", 1) > 1:
        _world2(monkeypatch, trace)
    np.random.seed(7)
    hist = train(adata, _Net(eng), **dict(FIT, **kw))
    trace.append(["history", [], {k: _enc(np.asarray(v)) for k, v in sorted(hist.history.items())}])
    trace.append(["rng_after", [int(np.random.randint(1 << 30))], {}])
    return trace


def _run_rejected(monkeypatch, no_cuda, kw):
    kw = dict(kw)
    adata = kw.pop("adata", None)
    try:
        _run(monkeypatch, no_cuda, adata, kw)
    except Exception as e:                      # noqa: BLE001 -- the type and message are what is recorded
        return [type(e).__name__, str(e)]
    return None


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


def _split(trace):
    k = next(i for i, c in enumerate(trace) if c[0] == "read_epoch_acc")
    return trace[:k], trace[k:]


@pytest.mark.skipif(not RECORD, reason="records the golden traces (DCA_RECORD_TRACES=1)")
def test_record_traces(monkeypatch, no_cuda):
    out = {"fit": {}, "rejected": {}}
    for name, make in CASES.items():
        with monkeypatch.context() as m:
            out["fit"][name] = _run(m, no_cuda, *make())
    for name, make in REJECTED.items():
        with monkeypatch.context() as m:
            out["rejected"][name] = _run_rejected(m, no_cuda, make())
    with open(GOLDEN, "w") as f:                # one call per line, so that a re-recording diffs call by call
        f.write('{"fit": {\n%s\n},\n"rejected": %s}\n' % (",\n".join(
            "%s: [\n%s]" % (json.dumps(k), ",\n".join(json.dumps(c, sort_keys=True) for c in t))
            for k, t in sorted(out["fit"].items())), json.dumps(out["rejected"], indent=0, sort_keys=True)))


@pytest.mark.skipif(RECORD, reason="recording")
@pytest.mark.parametrize("name", sorted(CASES))
def test_fit_trace(name, monkeypatch, no_cuda):
    want = _golden()["fit"][name]
    got = json.loads(json.dumps(_run(monkeypatch, no_cuda, *CASES[name]())))
    (ws, we), (gs, ge) = _split(want), _split(got)
    assert ge == we
    key = lambda c: json.dumps(c, sort_keys=True)                   # noqa: E731
    assert collections.Counter(map(key, gs)) == collections.Counter(map(key, ws))
    names = [c[0] for c in gs]
    last_reset = max(i for i, n in enumerate(names) if n == "reset_optimizer")
    assert all(i < last_reset for i, n in enumerate(names) if n in ("set_optimizer", "dist.broadcast_"))
    # the set-up (exact transform, take, ...) runs before the switch to the side stream
    assert names[-1] == "cuda.set_stream"


@pytest.mark.skipif(RECORD, reason="recording")
@pytest.mark.parametrize("name", sorted(REJECTED))
def test_rejected(name, monkeypatch, no_cuda):
    got = _run_rejected(monkeypatch, no_cuda, REJECTED[name]())
    assert got is not None and got == _golden()["rejected"][name]
