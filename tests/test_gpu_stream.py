"""The host-streaming path (dca_stream_*) element by element and bit for bit.

(a) The two expansion kernels (dca_expand_packed_counts / dca_expand_sparse_counts, the calls dca_stream_step makes)
    against a float64 statement of the input transform, for every format, at the shapes where the sparse kernel's
    span scan, its shared-memory sizing and its global-memory fallback change.
(b) dca_stream_step against the resident dca_train_step on the expanded matrix: the expansion is per row, so the
    tensor-core step must see the same bytes and give bit-identical losses, gradients and weights in every batch order.
(c) train(stream=True, shuffle=True) against a replay of its batches on the resident path.
(d) dca_train_step_host against train_step + apply_update.  Needs an H100: -m gpu."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
SPECIAL = np.array([14, 15, 16, 254, 255, 256, 65534, 65535, 65536, 1e6])   # around every escape value, and a large count


def _L():
    from dca_b200 import _lib
    return _lib


def _dev(a):
    """numpy -> device (structured arrays as their bytes); torch allocations are 512-byte aligned."""
    a = np.ascontiguousarray(a)
    if a.dtype.names:
        a = a.view(np.uint8)
    return torch.from_numpy(a).to(DEV)


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _spans(G):
    """Genes where the sparse kernel's per-thread spans of S bitmap bytes start and end, plus both ends of the row."""
    S = -(-(G // 8) // 256)
    starts = [8 * S * t for t in range(256) if 8 * S * t < G]
    return sorted(set([0, G - 1] + starts + [g - 1 for g in starts if g > 0]))


def _counts(n, G, seed, density=0.3):
    """Counts with an empty row (row 0), a row with every gene non-zero (row 1), a row with an odd number of non-zeros
    (row 2) and the counts of SPECIAL at gene 0, gene G-1 and both ends of every span in the other rows."""
    rng = np.random.default_rng(seed)
    Y = np.where(rng.random((n, G)) < density, rng.geometric(0.25, (n, G)), 0).astype(np.float64)
    spots = np.array(_spans(G))
    k = np.arange(len(spots))[None, :] + np.arange(n)[:, None]
    Y[:, spots] = SPECIAL[k % len(SPECIAL)]
    if n >= 3:
        Y[1] = np.maximum(Y[1], rng.integers(1, 14, G))
        Y[0] = 0
        free = np.setdiff1d(np.arange(G), spots)
        if np.count_nonzero(Y[2]) % 2 == 0 and len(free):
            Y[2, free[0]] = 0 if Y[2, free[0]] else 3
    return Y.astype(np.float32)


def _pack(Y, fmt, ovf):
    """Packed form of Y; without an overflow list the counts are first clipped to the format's largest code, which is
    then a literal.  Returns (packed counts, the counts the expansion must reproduce)."""
    from dca_b200 import io
    top = 15 if fmt == "sparse" else (1 << fmt) - 1
    Yw = Y if ovf else np.minimum(Y, top)
    pc = io.pack_counts(Yw, fmt, native=True)
    assert np.array_equal(io.unpack_counts(pc), Yw)
    return pc, Yw


class _Dev:
    """Device copy of a PackedCounts (rows r0:r1), in the layout the expansion entry points take."""

    def __init__(self, pc, ovf, r0=0, r1=None):
        r1 = pc.n_rows if r1 is None else r1
        self.bits, self.n, self.G = pc.bits, r1 - r0, pc.n_genes
        self.packed = _dev(pc.packed[r0:r1].view(np.uint8))
        e0, e1 = int(pc.indptr[r0]), int(pc.indptr[r1])
        self.ovp = _dev(pc.indptr[r0:r1 + 1]) if ovf else None
        self.ove = _dev(pc.entries[e0:e1] if e1 > e0 else np.zeros(1, pc.entries.dtype)) if ovf else None
        if pc.bits == 1:
            n0, n1 = int(pc.nib_indptr[r0]), int(pc.nib_indptr[r1])
            self.nibp = _dev(pc.nib_indptr[r0:r1 + 1])
            self.nib = _dev(pc.nibbles[n0:n1 + 16])
            self.max_nib = int(np.max(np.diff(pc.nib_indptr[r0:r1 + 1])))


GUARD = 64


def _expand(d, sf, mean, inv, use_sf, log1p, x_bf16, max_nib=None):
    """Run one expansion into NaN-filled buffers with GUARD elements after Y, X and sf_out; checks the guards and returns
    (Y, X, sf_out) device tensors of the real extent."""
    L = _L(); lib = L.load()
    n, G = d.n, d.G
    Y = torch.full((n * G + GUARD,), float("nan"), device=DEV)
    X = torch.full((n * G + GUARD,), float("nan"), device=DEV, dtype=torch.bfloat16 if x_bf16 else torch.float32)
    so = torch.full((n + GUARD,), float("nan"), device=DEV)
    xd = L.BF16 if x_bf16 else L.F32
    sp = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    if d.bits == 1:
        st = lib.dca_expand_sparse_counts(_ptr(d.packed), _ptr(d.nibp), _ptr(d.nib), d.max_nib if max_nib is None else max_nib,
                                          _ptr(d.ovp), _ptr(d.ove), _ptr(sf), n, G, _ptr(mean), _ptr(inv), int(use_sf),
                                          int(log1p), _ptr(Y), _ptr(X), xd, _ptr(so), sp)
    else:
        st = lib.dca_expand_packed_counts(_ptr(d.packed), d.bits, _ptr(d.ovp), _ptr(d.ove), _ptr(sf), n, G, _ptr(mean),
                                          _ptr(inv), int(use_sf), int(log1p), _ptr(Y), _ptr(X), xd, _ptr(so), sp)
    L.check(st, "expand")
    torch.cuda.synchronize()
    for buf, m in ((Y, n * G), (X, n * G), (so, n)):
        assert bool(torch.isnan(buf[m:].float()).all()), "the expansion wrote past its output"
    return Y[:n * G].view(n, G), X[:n * G].view(n, G), so[:n]


def _x_bound_check(Yw, sf, mean, inv, use_sf, log1p, Xf, tag, chunk=256):
    """fp32 X against X64 = (l64 - mean) * inv_std, l64 = log1p(y / sf) in float64 from the same float32 sf, mean, inv_std.

    normalise_count (layers.cu) computes v = y * (1/s), l = ln2 * __log2f(1 + v), X = (l - mean) * inv_std in fp32:
      v:       two roundings, relative 2^-23                    -> l off by <= v/(1+v) 2^-23 <= 2^-23 absolute
      1 + v:   one rounding, relative 2^-24                      -> l off by <= 2^-24 absolute
      __log2f: 2^-22 absolute on [0.5, 2] (CUDA Programming Guide, intrinsic functions), 2 ulp elsewhere
                                                                 -> l off by <= ln2 2^-22 absolute or 2^-22 relative
      * ln2f:  the rounded constant and the product, relative 2^-23 of l
    so |l - l64| <= 2^-23 + 2^-24 + ln2 2^-22 + (2^-22 + 2^-23) l64 < 4e-7 + 4e-7 l64 (without log1p: 2^-23 v).  The
    subtraction and the product round once each (relative 2^-24 of X), and the error of l is scaled by inv_std:
      |X - X64| <= inv_std (4e-7 + 4e-7 l64) + 2^-23 |X64|.
    Returns the worst err / bound."""
    n, G = Yw.shape
    m64 = mean.astype(np.float64) if mean is not None else np.zeros(G)
    i64 = inv.astype(np.float64) if inv is not None else np.ones(G)
    worst = 0.0
    for r0 in range(0, n, chunk):
        y = Yw[r0:r0 + chunk].astype(np.float64)
        v = y / sf[r0:r0 + chunk, None].astype(np.float64) if (use_sf and sf is not None) else y
        l64 = np.log1p(v) if log1p else v
        X64 = (l64 - m64) * i64
        bound = i64 * (4e-7 + 4e-7 * l64) + 2.0 ** -23 * np.abs(X64)
        err = np.abs(Xf[r0:r0 + chunk].astype(np.float64) - X64)
        ratio = err / bound
        k = np.unravel_index(np.argmax(ratio), ratio.shape)
        assert ratio[k] <= 1.0, (tag, r0 + k[0], k[1], float(y[k]), float(Xf[r0 + k[0], k[1]]), float(X64[k]), float(bound[k]))
        worst = max(worst, float(ratio[k]))
    return worst


def _transform(G, seed):
    rng = np.random.default_rng(seed)
    mean = rng.normal(1.0, 0.7, G).astype(np.float32)
    inv = np.exp(rng.normal(0.0, 0.7, G)).astype(np.float32)
    return mean, inv


def _check_case(Y, fmt, ovf, use_sf, log1p, scale, sf_given, seed, max_nib_list=()):
    n, G = Y.shape
    pc, Yw = _pack(Y, fmt, ovf)
    d = _Dev(pc, ovf)
    rng = np.random.default_rng(seed)
    sf = np.exp(rng.normal(0.0, 0.5, n)).astype(np.float32) if sf_given else None
    mean, inv = _transform(G, seed) if scale else (None, None)
    sfd, md, vd = (None if a is None else _dev(a) for a in (sf, mean, inv))
    Yf, Xf, so = _expand(d, sfd, md, vd, use_sf, log1p, False)
    Yb, Xb, sob = _expand(d, sfd, md, vd, use_sf, log1p, True)
    tag = (fmt, ovf, n, G, use_sf, log1p, scale, sf_given)
    Yh = Yf.cpu().numpy()
    assert np.array_equal(Yh.view(np.int32), Yw.view(np.int32)), tag             # counts bit for bit, escapes included
    assert torch.equal(Yb, Yf), tag
    want_sf = sf if sf is not None else np.ones(n, np.float32)
    for s in (so, sob):
        assert np.array_equal(s.cpu().numpy().view(np.int32), want_sf.view(np.int32)), tag
    # bf16 X is the same call's fp32 X rounded to nearest even (torch's float -> bfloat16 cast)
    assert torch.equal(Xb.view(torch.int16), Xf.to(torch.bfloat16).view(torch.int16)), tag
    worst = _x_bound_check(Yw, sf, mean, inv, use_sf, log1p, Xf.cpu().numpy(), tag)
    for cap in max_nib_list:                        # rows above the cap read their codes from global memory: same bits
        for x_bf16, (Yr, Xr) in ((False, (Yf, Xf)), (True, (Yb, Xb))):
            Y2, X2, _ = _expand(d, sfd, md, vd, use_sf, log1p, x_bf16, max_nib=cap)
            assert torch.equal(Y2, Yr) and torch.equal(X2.view(torch.int16 if x_bf16 else torch.int32),
                                                       Xr.view(torch.int16 if x_bf16 else torch.int32)), (tag, cap)
    print("X err / bound %s: worst %.3f" % (tag, worst))
    return worst


SHAPES = [(1, 8), (3, 8), (4096, 8), (1, 264), (3, 264), (4096, 264), (3, 2048), (1024, 2048), (3, 2056), (1024, 2056),
          (1, 20000), (3, 20000), (256, 20000), (3, 65536)]
FORMATS = [4, 8, 16, "sparse"]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "%dx%d" % s)
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("ovf", [True, False], ids=["ovf", "no_ovf"])
def test_expansion_matches_float64(shape, fmt, ovf):
    """Y == the counts, sf_out == sf, bf16 X == RNE(fp32 X), fp32 X within the derived bound of the float64 transform,
    nothing written past the outputs; sparse rows also through the global-memory fallback for their codes."""
    n, G = shape
    Y = _counts(n, G, seed=n * 7 + G)
    caps = (0, 16, 48) if fmt == "sparse" else ()
    _check_case(Y, fmt, ovf, True, True, True, True, seed=G, max_nib_list=caps)


FLAGS = [(1, 1, 1, 1), (0, 1, 1, 1), (1, 0, 1, 1), (1, 1, 0, 1), (1, 1, 1, 0), (0, 0, 0, 0), (1, 0, 0, 1), (0, 1, 0, 0)]


@pytest.mark.parametrize("flags", FLAGS, ids=lambda f: "sf%d_log%d_scale%d_sfgiven%d" % f)
@pytest.mark.parametrize("fmt", FORMATS)
def test_expansion_transform_flags(fmt, flags):
    """Every combination the input transform allows: size factors used or not, log1p on or off, mean / inv_std given or
    NULL, size factors given or NULL (sf_out is then 1)."""
    use_sf, log1p, scale, sf_given = flags
    Y = _counts(64, 2056, seed=11)
    _check_case(Y, fmt, True, use_sf, log1p, scale, sf_given, seed=5)
    _check_case(Y, fmt, False, use_sf, log1p, scale, sf_given, seed=6)


def test_expansion_benchmark_shape():
    """The benchmark's 4096 x 20000 batch (S = 10 bitmap bytes per thread of the sparse kernel), 4-bit and sparse."""
    rng = np.random.default_rng(3)
    Y = _counts(4096, 20000, seed=3, density=0.15)
    Y[rng.integers(0, 4096, 3000), rng.integers(0, 20000, 3000)] = 1e6
    for fmt in (4, "sparse"):
        _check_case(Y, fmt, True, True, True, True, True, seed=7, max_nib_list=(256,) if fmt == "sparse" else ())


# ------------------------------------------------------------------------------------------------------------ pipeline
def _engine(G, B, gemm_path, x_dtype, seed=None):
    from dca_b200.engine import DeviceEngine
    return DeviceEngine(G, G, (64, 32, 64), "zinb-conddisp", max_batch=B, seed=seed, gemm_path=gemm_path, x_dtype=x_dtype)


def _stream_counts(N, G, seed):
    """Sparse-looking counts (about 12 % non-zero) generated in row blocks, with counts that need every escape."""
    rng = np.random.default_rng(seed)
    Y = np.empty((N, G), np.float32)
    for r0 in range(0, N, 1024):
        r1 = min(N, r0 + 1024)
        blk = np.where(rng.random((r1 - r0, G), dtype=np.float32) < 0.12, rng.geometric(0.35, (r1 - r0, G)), 0)
        Y[r0:r1] = blk
    k = rng.integers(0, len(SPECIAL), 4 * N)
    Y[rng.integers(0, N, 4 * N), rng.integers(0, G, 4 * N)] = SPECIAL[k]
    Y[np.arange(N), 0] = np.maximum(Y[:, 0], 1)             # no empty row (the size factors below stay finite)
    return Y


def _resident(src, ovf, G, sf, mean, inv, x_bf16):
    """Whole-matrix expansion (X, Y, sf_out) of a packed matrix, or of a uint16 matrix given as 16-bit packed counts."""
    d = _Dev(src, ovf)
    Y, X, so = _expand(d, _dev(sf), _dev(mean), _dev(inv), True, True, x_bf16)
    return X, Y, so


def _equal_state(es, er, tag):
    assert es.read_loss() == er.read_loss(), tag
    for name in ("grads", "params", "rms", "bn_state"):
        assert torch.equal(getattr(es, name), getattr(er, name)), (tag, name)


ORDERS = {                          # (batch, next) per call; 4 batches, batch 3 is the partial one
    "in_sequence": [(0, 1), (1, 2), (2, 3), (3, -1)],
    "partial_in_middle": [(2, 3), (3, 0), (0, 1), (1, -1)],
    "next_not_followed": [(1, 3), (0, 2), (3, 1), (2, -1)],
    "no_next_mid_epoch": [(0, 1), (1, -1), (2, 3), (3, -1)],
    "epoch_a": [(3, 1), (1, 0), (0, 2), (2, -1)],
    "epoch_b": [(1, 2), (2, 3), (3, 0), (0, -1)],
}


def _run_pipeline(G, B, N, src, ovf, sf, mean, inv, gemm_path, stream_src=None):
    """Stream engine (fp32 x_dtype) against a resident engine on the whole-matrix expansion: bf16 X on the tensor-core
    path (the bytes the stream's expansion writes), fp32 X on the generic path.  Every order is one epoch inside
    stream_begin / stream_end, all on the same pair of engines."""
    tc = gemm_path == "tcgen05"
    es = _engine(G, B, gemm_path, "float32", seed=3)
    er = _engine(G, B, gemm_path, "bfloat16" if tc else "float32", seed=None)
    er.set_weights(es.get_weights())
    Xr, Yr, sfr = _resident(src, ovf, G, sf, mean, inv, x_bf16=tc)
    std = (1.0 / inv.astype(np.float64))
    es.set_input_transform(mean, std, True, True)
    sfh = torch.from_numpy(sf).pin_memory()
    torch.cuda.synchronize()
    for oname, order in ORDERS.items():
        es.stream_begin(src if stream_src is None else stream_src, sfh, B)
        for k, (i, nxt) in enumerate(order):
            r0, r1 = i * B, min(N, (i + 1) * B)
            es.stream_step(i, nxt)
            er.train_step(Xr[r0:r1], Yr[r0:r1], sfr[r0:r1])
            tag = (gemm_path, oname, k, i, nxt)
            if tc:
                _equal_state(es, er, tag)
            else:               # split-K atomics: the bounds of test_two_phase_step_equals_single_call
                l1, l2 = es.read_loss(), er.read_loss()
                assert abs(l1 - l2) <= 1e-5 * abs(l2), (tag, l1, l2)
                g1, g2 = es.grads.cpu().numpy(), er.grads.cpu().numpy()
                assert np.max(np.abs(g1 - g2)) <= 1e-5 * np.max(np.abs(g2)) + 1e-12, tag
            es.apply_update(1e-3, 5.0); er.apply_update(1e-3, 5.0)
            torch.cuda.synchronize()
            if tc:
                _equal_state(es, er, tag + ("update",))
            else:               # keep the replicas identical: RMSprop amplifies order noise in near-zero gradients
                es.params.copy_(er.params); es.rms.copy_(er.rms); es.bn_state.copy_(er.bn_state); es.params_changed()
        es.stream_end()
    es.close(); er.close()


@pytest.fixture(scope="module")
def big_counts():
    N, G, B = 3 * 4096 + 123, 20000, 4096
    Y = _stream_counts(N, G, 17)
    from dca_b200 import io
    pc = io.pack_counts(Y, "sparse", batch=B)
    assert pc.bits == 1 and len(pc.entries) > 0
    rng = np.random.default_rng(4)
    sf = np.exp(rng.normal(0, 0.3, N)).astype(np.float32)
    mean, inv = _transform(G, 8)
    return N, G, B, pc, sf, mean, inv


@pytest.fixture(scope="module")
def mid_counts():
    N, G, B = 3 * 1024 + 123, 2048, 1024
    Y = _stream_counts(N, G, 19)
    rng = np.random.default_rng(5)
    sf = np.exp(rng.normal(0, 0.3, N)).astype(np.float32)
    mean, inv = _transform(G, 9)
    return N, G, B, Y, sf, mean, inv


@pytest.mark.parametrize("bufs", ["2", "3"])
def test_stream_sparse_benchmark_shape_bit_identical(big_counts, bufs, monkeypatch):
    """G = 20000, batch 4096, 3 full batches and one of 123 rows, sparse format with escapes."""
    monkeypatch.setenv("DCA_STREAM_BUFS", bufs)
    N, G, B, pc, sf, mean, inv = big_counts
    _run_pipeline(G, B, N, pc, True, sf, mean, inv, "tcgen05")


@pytest.mark.parametrize("bufs", ["2", "3"])
def test_stream_4bit_overflow_bit_identical(mid_counts, bufs, monkeypatch):
    monkeypatch.setenv("DCA_STREAM_BUFS", bufs)
    from dca_b200 import io
    N, G, B, Y, sf, mean, inv = mid_counts
    pc = io.pack_counts(Y, 4, batch=B)
    assert len(pc.entries) > 0
    _run_pipeline(G, B, N, pc, True, sf, mean, inv, "tcgen05")


@pytest.mark.parametrize("bufs", ["2", "3"])
def test_stream_strided_uint16_bit_identical(mid_counts, bufs, monkeypatch):
    """A column slice of a wider pinned uint16 tensor: the pitched-copy branch of the prefetch."""
    monkeypatch.setenv("DCA_STREAM_BUFS", bufs)
    from dca_b200 import io
    N, G, B, Y, sf, mean, inv = mid_counts
    Y16 = np.minimum(Y, 65535).astype(np.uint16)
    wide = np.zeros((N, G + 24), np.uint16)
    wide[:, 8:8 + G] = Y16
    counts = torch.from_numpy(wide).pin_memory()[:, 8:8 + G]
    assert counts.stride(0) == G + 24
    pc16 = io.PackedCounts(Y16, 16, G, np.zeros(N + 1, np.int64), np.zeros(0, io.OVERFLOW_ENTRY))
    _run_pipeline(G, B, N, pc16, False, sf, mean, inv, "tcgen05", stream_src=counts)


def test_stream_generic_path_within_tolerance(mid_counts):
    from dca_b200 import io
    N, G, B, Y, sf, mean, inv = mid_counts
    _run_pipeline(G, B, N, io.pack_counts(Y, "sparse", batch=B), True, sf, mean, inv, "generic")


# ------------------------------------------------------------------------------------------------------ public route
def test_train_stream_replays_on_resident_path(monkeypatch):
    """train(stream=True, shuffle=True): the batches it streams, replayed in the recorded order with resident train_step
    on the whole-matrix expansion from the same initial weights, give bit-identical final weights, loss and val_loss."""
    from dca_b200.anndata_lite import AnnData
    from dca_b200 import io
    from dca_b200.engine import DeviceEngine
    from dca_b200.network import AE_types
    from dca_b200.train import train
    from tests.util import synth_counts
    N, G, bs, epochs = 1000, 2000, 128, 3
    Y = synth_counts(N, G, 29); Y[5, 3] = 300.0; Y[7, 1999] = 70000.0
    ad = io.normalize(io.read_dataset(AnnData(Y.copy())), filter_min_counts=False)
    log = []
    first = {}

    def wrap(name, keep_result=False):
        orig = getattr(DeviceEngine, name)

        def f(self, *a, **k):
            if name == "stream_begin" and not first:
                torch.cuda.synchronize()
                first.update(params=self.params.clone(), bn=self.bn_state.clone())
            out = orig(self, *a, **k)
            log.append((name, a, k, out if keep_result else None))
            return out
        monkeypatch.setattr(DeviceEngine, name, f)
    for name in ("set_input_transform", "stream_begin", "stream_step", "apply_update", "eval_step"):
        wrap(name)
    wrap("read_epoch_acc", keep_result=True)
    np.random.seed(0)
    net = AE_types["zinb-conddisp"](input_size=G, output_size=G, hidden_size=(64, 32, 64), gemm_path="tcgen05")
    net.build(max_batch=bs, seed=3)
    hist = train(ad, net, epochs=epochs, batch_size=bs, verbose=False, stream=True, shuffle=True).history
    monkeypatch.undo()
    orders = [a for n, a, k, _ in log if n == "stream_step"]
    assert sorted(set(i for i, _ in orders)) == list(range(8)) and len(orders) == 8 * epochs
    assert any(i == 7 and nxt >= 0 for i, nxt in orders), "the partial batch was never in the middle of an epoch"
    (mean, std, use_sf, log1p), = [a for n, a, k, _ in log if n == "set_input_transform"]
    assert use_sf and log1p
    pc, sfh, B = [a for n, a, k, _ in log if n == "stream_begin"][0]
    assert B == bs
    std64 = np.asarray(std, np.float64)                   # what DeviceEngine.set_input_transform uploads
    inv = (1.0 / np.where(std64 == 0, 1.0, std64)).astype(np.float32)
    Xr, Yr, sfr = _resident(pc, True, G, sfh.numpy(), np.asarray(mean, np.float32), inv, x_bf16=False)
    net2 = AE_types["zinb-conddisp"](input_size=G, output_size=G, hidden_size=(64, 32, 64), gemm_path="tcgen05")
    net2.build(max_batch=bs, seed=3)                      # an engine of the same configuration, fp32 X
    er = net2.engine
    er.params.copy_(first["params"]); er.bn_state.copy_(first["bn"]); er.params_changed()
    er.set_optimizer("RMSprop"); er.reset_optimizer()
    n_acc = 0
    replay_hist = {"loss": [], "val_loss": []}
    for name, a, k, out in log:
        if name == "stream_step":
            r0, r1 = a[0] * B, min(pc.n_rows, (a[0] + 1) * B)
            er.train_step(Xr[r0:r1], Yr[r0:r1], sfr[r0:r1])
        elif name == "apply_update":
            er.apply_update(*a, **k)
        elif name == "eval_step":
            er.eval_step(*a, **k)
        elif name == "read_epoch_acc":
            acc = er.read_epoch_acc(*a, **k)
            assert acc == out, (n_acc, acc, out)
            n_acc += 1
            if n_acc % 2 == 0:                     # the second read of an epoch is its result
                replay_hist["loss"].append(acc[0] / acc[1]); replay_hist["val_loss"].append(acc[2] / acc[3])
    torch.cuda.synchronize()
    assert torch.equal(er.params, net.engine.params) and torch.equal(er.bn_state, net.engine.bn_state)
    assert replay_hist["loss"] == hist["loss"] and replay_hist["val_loss"] == hist["val_loss"], (replay_hist, hist)
    er.close()


# ------------------------------------------------------------------------------------------------ dca_train_step_host
@pytest.mark.parametrize("x_dtype", ["float32", "bfloat16"])
def test_train_step_host_equals_device_step(x_dtype):
    """dca_train_step_host == train_step + apply_update on device copies: bit for bit on the tensor-core path (full and
    partial batch, size factors given and NULL), within tolerance on the generic path; refused while a host stream is
    active, accepted again after stream_end; host tensors of the wrong dtype or shape are refused."""
    from tests.util import synth_counts
    from oracle import dca_oracle as O
    G, B = 264, 256
    Y = synth_counts(B, G, 41); X, sf = O.normalize_inputs(Y)
    tdt = torch.bfloat16 if x_dtype == "bfloat16" else torch.float32
    for gemm_path in ("tcgen05", "generic"):
        eh = _engine(G, B, gemm_path, x_dtype, seed=5)
        ed = _engine(G, B, gemm_path, x_dtype, seed=5)
        for step, (nb, with_sf) in enumerate([(B, True), (B, True), (B - 56, True), (B, False), (B - 56, False)]):
            xh = torch.from_numpy(X[:nb]).to(tdt).pin_memory(); yh = torch.from_numpy(Y[:nb]).pin_memory()
            sh = torch.from_numpy(sf[:nb]).pin_memory() if with_sf else None
            loss = eh.train_step_host(xh, yh, sh, 1e-3, 5.0)
            ed.train_step(xh.to(DEV), yh.to(DEV), None if sh is None else sh.to(DEV)); ed.apply_update(1e-3, 5.0)
            torch.cuda.synchronize()
            tag = (gemm_path, x_dtype, step, nb, with_sf)
            if gemm_path == "tcgen05":
                assert loss == ed.read_loss(), tag
                for name in ("grads", "params", "rms", "bn_state"):
                    assert torch.equal(getattr(eh, name), getattr(ed, name)), (tag, name)
            else:
                assert abs(loss - ed.read_loss()) <= 1e-5 * abs(loss), tag
                g1, g2 = eh.grads.cpu().numpy(), ed.grads.cpu().numpy()
                assert np.max(np.abs(g1 - g2)) <= 1e-5 * np.max(np.abs(g2)) + 1e-12, tag
                eh.params.copy_(ed.params); eh.rms.copy_(ed.rms); eh.bn_state.copy_(ed.bn_state); eh.params_changed()
        # the host-buffer step shares its staging with the streaming path: refused while a stream is active
        eh.set_input_transform(None, None, True, True)
        eh.stream_begin(torch.from_numpy(Y.astype(np.uint16)).pin_memory(), torch.from_numpy(sf).pin_memory(), B)
        eh.stream_step(0, -1); eh.apply_update(1e-3, 5.0)
        with pytest.raises(ValueError, match="stream"):
            eh.train_step_host(xh, yh, sh, 1e-3, 5.0)
        eh.stream_end()
        assert np.isfinite(eh.train_step_host(xh, yh, sh, 1e-3, 5.0))
        other = torch.bfloat16 if tdt == torch.float32 else torch.float32
        for bad in ((xh.to(other), yh, sh), (xh[:, :-8].contiguous(), yh, sh), (xh, yh[:-1], sh),
                    (xh, yh.double(), sh), (xh, yh, torch.ones(3)), (xh.to(DEV), yh, sh)):
            with pytest.raises(ValueError, match="train_step_host"):
                eh.train_step_host(*bad, 1e-3, 5.0)
        eh.close(); ed.close()
