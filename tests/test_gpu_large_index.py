"""Every whole-dataset kernel past 2^31 entries and 4 GiB of one matrix.

The training step, predict and the preprocessing read the dataset in place, by row index, from the whole matrix
(``rows[r] * ld + col``).  A 110 000 x 20 000 count matrix (2.2e9 entries) puts rows on both sides of each place where
such an address leaves 32 bits: fp32 byte offsets from row ROW_F32_BYTES, element offsets (and bf16 byte offsets) from
row ROW_ELEMS.  The checks, and the kernels each one reads the big matrix with:

 * resident preprocessing (DeviceDataset.from_counts, bf16 and fp32 X): dca_counts_csr_to_dense, dca_count_totals,
   dca_log_moments, dca_normalize_write against a float64 reference computed from the CSR on the host; take() and
   dca_gather_counts on rows past the boundaries;
 * the step reading rows in place (train_step / eval_step / predict with rows=) against the same engine state fed
   contiguous copies of the rows: K1 / K5 (gene_gemm_tc.cu), the heads + loss kernel and the ZINB loss kernel
   (zinb_loss.cu), the fused heads kernel (flash_zinb.cu), the generic GEMM's row gather
   (dense_generic.cu), an extra AE type (extra_types.cu), input dropout (activations.cu), the fp32 X gather + convert
   (layers.cu);
 * packed in HBM (PackedDeviceDataset, 16-bit dense and sparse): the GPU packer's bytes against io.pack_rows,
   dca_expand_rows_exact and dca_packed_train_step against the resident rows and step;
 * out of core (StreamedDataset): the chunked statistics passes with row0 past the boundaries, and a streamed predict
   batch holding the last rows.

Every row of the matrix is different (a marker count per row, and a fingerprint check), so a read of the wrong row
changes bits.  The GPU tests need about 30 GB of free device memory and skip with the reason when it is not there; the
large device objects are built one at a time.  The float64 reference and the boundary arithmetic are CPU tests."""
import gc

import numpy as np
import pytest
import torch

N, G = 110_000, 20_000
DENSITY = 0.05
SEED = 11
DEV = torch.device("cuda:0")

ROW_F32_BYTES = -(-2 ** 32 // (4 * G))       # 53 688: first row whose fp32 byte offset is >= 2^32
ROW_ELEMS = -(-2 ** 31 // G)                 # 107 375: first row whose element offset is >= 2^31 (bf16 bytes >= 2^32)
EDGES = [0, N - 1]
NEAR = list(range(ROW_F32_BYTES - 2, ROW_F32_BYTES + 2)) + list(range(ROW_ELEMS - 2, ROW_ELEMS + 2))
DEEP_ROWS = [0, ROW_F32_BYTES - 1, ROW_F32_BYTES, ROW_ELEMS - 1, ROW_ELEMS, N - 1]   # counts 20, 300 and 70000
DEEP_COUNTS = (20.0, 300.0, 70000.0)        # past the 4-, 8- and 16-bit packing widths


def _samples():
    """A seeded sample of 40 rows from each region: below ROW_F32_BYTES, between the two boundaries, past ROW_ELEMS."""
    rng = np.random.default_rng(SEED + 1)
    return np.concatenate([rng.choice(np.arange(a, b), 40, replace=False)
                           for a, b in ((1, ROW_F32_BYTES - 2), (ROW_F32_BYTES + 2, ROW_ELEMS - 2), (ROW_ELEMS + 2, N - 1))])


BOUNDARY = np.unique(np.concatenate([EDGES, NEAR, _samples()])).astype(np.int64)
# the training batch: every boundary row in a seeded order, N - 1 and ROW_ELEMS twice
BATCH = np.random.default_rng(SEED + 2).permutation(np.concatenate([BOUNDARY, [N - 1, ROW_ELEMS]])).astype(np.int64)
STREAM_BS = 4096
STREAM_BATCH = (N - 1) // STREAM_BS          # the streamed predict batch holding ROW_ELEMS and N - 1


def _assert_past_boundaries(rows, both_sides=True):
    """rows hold N - 1 and rows whose fp32 byte, element and bf16 byte offsets are past 2^32, 2^31 and 2^32; with
    both_sides, also rows below each boundary."""
    r = np.asarray(rows, dtype=np.int64)
    assert (r * G * 4 >= 2 ** 32).any(), "fp32 byte offsets past 2^32"
    assert (r * G >= 2 ** 31).any(), "element offsets past 2^31"
    assert (r * G * 2 >= 2 ** 32).any(), "bf16 byte offsets past 2^32"
    assert (r == N - 1).any()
    if both_sides:
        assert (r * G * 4 < 2 ** 32).any() and (r * G < 2 ** 31).any(), "rows below the boundaries"


# ---------------------------------------------------------------------------------------------- the counts
def _counts():
    """N x G scipy CSR of counts 1 + Poisson(gene mean) at DENSITY non-zeros (the geometric gaps of
    tests/diag_packed.big_csr), built in row chunks.  Row r also holds the count 1 + r // G at gene r % G (rows r and
    r + k G differ there), and the rows DEEP_ROWS hold DEEP_COUNTS (so that the overflow lists of every packing width
    have entries on both sides of each boundary)."""
    import scipy.sparse as sp
    rng = np.random.default_rng(SEED)
    gene_mean = np.exp(rng.normal(-0.5, 1.0, size=G))
    m = int(G * DENSITY + 10 * np.sqrt(G * DENSITY) + 64)        # gaps drawn per row: their sum passes G almost surely
    cap = int(N * G * DENSITY * 1.01) + N + (1 << 20)
    indptr = np.zeros(N + 1, np.int64)
    indices = np.empty(cap, np.int32)
    data = np.empty(cap, np.float32)
    pos = 0
    for s in range(0, N, 8192):
        e = min(N, s + 8192)
        r = np.arange(s, e)
        mark = (r % G)[:, None]
        cols = np.cumsum(rng.geometric(DENSITY, size=(e - s, m)), axis=1) - 1
        cols[(cols >= G) | (cols == mark)] = G                      # past the row, or the marker's gene: dropped
        cols = np.sort(np.concatenate([cols, mark], axis=1), axis=1)
        keep = cols < G
        c = cols[keep].astype(np.int32)                              # row-major: by row, then gene
        v = (1 + rng.poisson(gene_mean[c])).astype(np.float32)
        v[(cols == mark)[keep]] = 1 + r // G                         # one marker per row, in row order
        if pos + c.size > cap:
            raise RuntimeError("capacity estimate exceeded")
        indptr[s + 1:e + 1] = pos + np.cumsum(keep.sum(1))
        indices[pos:pos + c.size] = c
        data[pos:pos + c.size] = v
        pos += c.size
    for r in DEEP_ROWS:
        a, b = indptr[r], indptr[r + 1]
        slots = a + np.flatnonzero(indices[a:b] != r % G)[:len(DEEP_COUNTS)]
        data[slots] = DEEP_COUNTS
    return sp.csr_matrix((data[:pos], indices[:pos], indptr), shape=(N, G), copy=False)


def sparse_reference(csr):
    """device_data.normalize_reference (default flags) from the non-zeros of a CSR matrix, in float64, without a dense
    pass: n_counts from row sums (exact: integer counts), sf = float32(n_counts / median), the gene mean and two-pass
    variance of l = float32(log1p(float64(float32(y / sf64)))) over the non-zeros, the zeros adding (N - nnz_g) mean^2.
    Returns the statistics and x_rows(rows), the X rows normalize_reference computes."""
    import scipy.sparse as sp
    n, g = csr.shape
    lens = np.diff(csr.indptr)
    y = csr.data.astype(np.float64)
    n_counts = np.bincount(np.repeat(np.arange(n, dtype=np.int32), lens), weights=y, minlength=n)
    med = np.median(n_counts)
    sf64 = n_counts / med
    q = (y / np.repeat(sf64, lens)).astype(np.float32)
    del y
    l = np.log1p(q.astype(np.float64)).astype(np.float32)
    del q
    mean = np.bincount(csr.indices, weights=l, minlength=g) / n
    nnz_g = np.bincount(csr.indices, minlength=g)
    if n > 1:
        var = (np.bincount(csr.indices, weights=(l - mean[csr.indices]) ** 2, minlength=g) + (n - nnz_g) * mean ** 2) / (n - 1)
    else:
        var = np.ones(g)
    std = np.sqrt(var)
    std[std == 0] = 1.0
    logs = sp.csr_matrix((l, csr.indices, csr.indptr), shape=(n, g))

    def x_rows(rows):
        return ((logs[np.asarray(rows)].toarray() - mean) / std).astype(np.float32)
    return dict(n_counts=n_counts, median=med, size_factors=sf64.astype(np.float32), mean=mean, std=std, x_rows=x_rows)


# ---------------------------------------------------------------------------------------------- CPU tests
def test_boundary_rows_lie_where_they_claim():
    assert N * G > 2 ** 31 and N < 2 ** 31
    assert (ROW_F32_BYTES - 1) * G * 4 < 2 ** 32 <= ROW_F32_BYTES * G * 4
    assert (ROW_ELEMS - 1) * G < 2 ** 31 <= ROW_ELEMS * G
    assert (ROW_ELEMS - 1) * G * 2 < 2 ** 32 <= ROW_ELEMS * G * 2
    assert ROW_F32_BYTES - 1 in NEAR and ROW_F32_BYTES in NEAR and ROW_ELEMS - 1 in NEAR and ROW_ELEMS in NEAR
    _assert_past_boundaries(BOUNDARY)
    _assert_past_boundaries(BATCH)
    assert len(set(BATCH.tolist())) == len(BATCH) - 2
    s0 = STREAM_BATCH * STREAM_BS
    _assert_past_boundaries(np.arange(s0, min(N, s0 + STREAM_BS)), both_sides=False)
    assert s0 < ROW_ELEMS                                           # ... and rows below 2^31 elements


def test_sparse_reference_is_normalize_reference():
    """The float64 reference of the large tests, computed from the non-zeros, against the dense statement of the device
    arithmetic: n_counts, median and size factors bit for bit, mean and std to float64 reassociation noise, X to one
    float32 ulp (the mean moves by reassociation noise)."""
    import scipy.sparse as sp
    from dca_b200.device_data import normalize_reference
    from tests.util import synth_counts
    Y = synth_counts(700, 96, 3)
    Y[5, :3] = DEEP_COUNTS
    Y[:, 40] = 0
    Y[0, 40] = 1                                                    # a gene with one non-zero
    ref = normalize_reference(Y)
    got = sparse_reference(sp.csr_matrix(Y))
    assert np.array_equal(got["n_counts"], ref["n_counts"])
    assert got["median"] == np.median(ref["n_counts"])
    assert np.array_equal(got["size_factors"], ref["size_factors"])
    np.testing.assert_allclose(got["mean"], ref["mean"], rtol=1e-12, atol=0)
    np.testing.assert_allclose(got["std"], ref["std"], rtol=1e-12, atol=0)
    rows = np.array([0, 5, 699, 5, 300])
    X = got["x_rows"](rows)
    assert X.dtype == np.float32 and X.shape == (5, 96)
    Xr = ref["X"][rows]
    assert np.all(np.abs(X.astype(np.float64) - Xr) <= np.spacing(np.maximum(np.abs(X), np.abs(Xr))))


# ---------------------------------------------------------------------------------------------- fixtures
@pytest.fixture(scope="module")
def counts():
    m = _counts()
    fp = m @ np.random.default_rng(SEED + 3).standard_normal(G)   # equal rows have equal fingerprints
    assert np.unique(fp).size == N, "two rows of the matrix are equal"
    for r in DEEP_ROWS:
        row = m.data[m.indptr[r]:m.indptr[r + 1]]
        assert (row >= 15).any() and (row >= 255).any() and (row >= 65535).any(), r
    return m


@pytest.fixture(scope="module")
def ref(counts):
    return sparse_reference(counts)


_BIG = {}            # the one large device object alive: building another frees it first
_SNAP = {}           # host copies of the resident dataset's statistics and boundary rows


def _free_big():
    for obj in _BIG.values():
        obj.__dict__.clear()                                        # (also when a failed test's frame still holds it)
    _BIG.clear()
    gc.collect()
    torch.cuda.empty_cache()


def _require(nbytes, what):
    free = torch.cuda.mem_get_info(DEV)[0]
    if free < nbytes:
        pytest.skip("%s needs %.1f GB of free device memory, %.1f GB are free" % (what, nbytes / 1e9, free / 1e9))


def _big(name, need, build):
    if name not in _BIG:
        _free_big()
        _require(need, name)
        _BIG[name] = build()
    return _BIG[name]


@pytest.fixture(scope="module", autouse=True)
def _peak_memory():
    if torch.cuda.is_available():
        torch.empty(0, device=DEV)                                  # (the allocator's statistics exist from here on)
        torch.cuda.reset_peak_memory_stats(DEV)
    yield
    _SNAP.clear()
    if torch.cuda.is_available():
        _free_big()
        print("\n[large index] peak device memory allocated: %.2f GB" % (torch.cuda.max_memory_allocated(DEV) / 1e9))


def _resident(counts, x_dtype):
    from dca_b200.device_data import DeviceDataset
    dd = _big("resident " + x_dtype, DeviceDataset.device_bytes(counts, x_dtype),
              lambda: DeviceDataset.from_counts(counts, DEV, x_dtype=x_dtype))
    if x_dtype == "bfloat16" and not _SNAP:
        r = torch.from_numpy(BOUNDARY).to(DEV)
        s0 = STREAM_BATCH * STREAM_BS
        _SNAP.update(n_counts=dd.n_counts.cpu().numpy(), sf=dd.sf.cpu().numpy(), mean=dd.mean.cpu().numpy(),
                     std=dd.std.cpu().numpy(), median=dd.median, flags=dd.flags, Y=dd.Y[r].cpu(), X=dd.X[r].cpu(),
                     stream_X=dd.X[s0:s0 + STREAM_BS].cpu(), stream_sf=dd.sf[s0:s0 + STREAM_BS].cpu())
    return dd


def _snapshot(counts):
    if not _SNAP:
        _resident(counts, "bfloat16")
    return _SNAP


def _snap_rows(snap, rows):
    """(Y, X, sf) of the resident dataset at rows (a subset of BOUNDARY, any order), contiguous on the device."""
    i = torch.from_numpy(np.searchsorted(BOUNDARY, rows))
    r = torch.from_numpy(np.asarray(rows))
    return (snap["Y"][i].contiguous().to(DEV), snap["X"][i].contiguous().to(DEV),
            torch.from_numpy(snap["sf"])[r].contiguous().to(DEV))


def _same_bits(a, b):
    a, b = (t.detach().cpu().contiguous() for t in (a, b))
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.reshape(-1).view(torch.uint8),
                                                                     b.reshape(-1).view(torch.uint8))


def _rows_d(rows):
    return torch.from_numpy(np.asarray(rows, dtype=np.int32)).to(DEV)


# ---------------------------------------------------------------------------------------------- 1. resident
def _bf16_bracket(x32):
    """The bf16 values of fp32 numbers within one ulp of x32 (rounded to nearest even): (low, high) as float32."""
    lo = torch.from_numpy(np.nextafter(x32, np.float32(-np.inf))).to(torch.bfloat16).float().numpy()
    hi = torch.from_numpy(np.nextafter(x32, np.float32(np.inf))).to(torch.bfloat16).float().numpy()
    return lo, hi


@pytest.mark.gpu
def test_resident_preprocessing_bf16(counts, ref):
    """dca_counts_csr_to_dense, dca_count_totals, dca_log_moments and dca_normalize_write over the whole matrix:
    n_counts and size factors bit for bit, mean and std to 1e-12 (float64 sums in another order), the boundary rows of Y
    equal to the CSR rows and of X within one fp32 ulp of the reference before the bf16 rounding."""
    dd = _resident(counts, "bfloat16")
    assert tuple(dd.Y.shape) == (N, G) and dd.X.dtype == torch.bfloat16
    assert np.array_equal(dd.n_counts.cpu().numpy(), ref["n_counts"])
    assert np.array_equal(dd.sf.cpu().numpy(), ref["size_factors"]) and dd.median == ref["median"]
    np.testing.assert_allclose(dd.mean.cpu().numpy(), ref["mean"], rtol=1e-12, atol=0)
    np.testing.assert_allclose(dd.std.cpu().numpy(), ref["std"], rtol=1e-12, atol=0)
    _assert_past_boundaries(BOUNDARY)
    r = torch.from_numpy(BOUNDARY).to(DEV)
    assert np.array_equal(dd.Y[r].cpu().numpy(), counts[BOUNDARY].toarray())
    X = dd.X[r].float().cpu().numpy()
    lo, hi = _bf16_bracket(ref["x_rows"](BOUNDARY))
    bad = ~((lo <= X) & (X <= hi))
    assert not bad.any(), "X rows %s off the reference" % np.unique(BOUNDARY[np.nonzero(bad)[0]])


@pytest.mark.gpu
def test_take_and_gather_past_the_boundaries(counts):
    """take() composes the rows a mask keeps; dca_gather_counts copies those rows, a set of columns over every row
    (with_output_genes) and both at once, reading Y at offsets past 2^31 elements."""
    from dca_b200 import _lib
    from dca_b200.device_data import _gather
    dd = _resident(counts, "bfloat16")
    mask = np.zeros(N, bool)
    mask[BOUNDARY] = True
    sub = dd.take(mask)
    assert np.array_equal(sub.rows.cpu().numpy(), BOUNDARY)
    _assert_past_boundaries(sub.rows.cpu().numpy())
    lib = _lib.load()
    assert np.array_equal(_gather(lib, dd.Y, sub.rows.cpu().numpy(), None, DEV).cpu().numpy(),
                          counts[BOUNDARY].toarray())
    cols = np.array([0, 7, 8, 4093, 12345, G - 9, G - 1, 3], np.int64)
    ys = dd.with_output_genes(cols)
    assert np.array_equal(ys.Y.cpu().numpy(), counts[:, cols].toarray())
    del ys
    _assert_past_boundaries(BATCH)
    both = _gather(lib, dd.Y, BATCH, cols, DEV).cpu().numpy()             # duplicate rows, any order
    assert np.array_equal(both, counts[BATCH][:, cols].toarray())


def _loss_call(lib, L, Y, rows, sf, m, d, pi, gdt):
    B = m.shape[0]
    tdt = torch.bfloat16 if gdt == L.BF16 else torch.float32
    dz = [torch.zeros((B, G), dtype=tdt, device=DEV) for _ in range(3)]
    loss = torch.zeros(1, dtype=torch.float64, device=DEV)
    nb = _lib_size(lib, B)
    ws = torch.zeros(nb, dtype=torch.uint8, device=DEV)
    L.check(lib.dca_zinb_loss_fwd_bwd(Y.data_ptr(), G, None if rows is None else rows.data_ptr(), sf.data_ptr(),
                                      m.data_ptr(), d.data_ptr(), pi.data_ptr(), G, B, G, L.AE_TYPE_IDS["zinb-conddisp"],
                                      0.0, 1.0 / (B * G), dz[0].data_ptr(), dz[1].data_ptr(), dz[2].data_ptr(), gdt, None,
                                      loss.data_ptr(), ws.data_ptr(), nb, None), "dca_zinb_loss_fwd_bwd")
    torch.cuda.synchronize()
    return loss, dz


def _lib_size(lib, B):
    import ctypes as C
    nb = C.c_size_t()
    assert lib.dca_zinb_loss_workspace_bytes(B, G, C.byref(nb)) == 0
    return nb.value


@pytest.mark.gpu
def test_loss_kernel_rows_equals_gathered(counts):
    """dca_zinb_loss_fwd_bwd (the per-thread cp.async ring kernel) reading the batch's counts and size factors by row
    index from the whole Y against the call on the gathered Y and sf: loss and fp32 / bf16 gradients bit for bit."""
    from dca_b200 import _lib as L
    lib = L.load()
    dd = _resident(counts, "bfloat16")
    _assert_past_boundaries(BATCH)
    B = len(BATCH)
    g = torch.Generator(device=DEV); g.manual_seed(1)
    m = torch.exp(torch.randn(B, G, device=DEV, generator=g) * 0.7 - 1.0).clamp(1e-5, 1e6)
    d = torch.nn.functional.softplus(torch.randn(B, G, device=DEV, generator=g) * 2.0).clamp(1e-4, 1e4)
    p = torch.sigmoid(torch.randn(B, G, device=DEV, generator=g) * 2.0)
    rows = _rows_d(BATCH)
    Yg, sfg = dd.Y[rows.long()].contiguous(), dd.sf[rows.long()].contiguous()
    for gdt in (L.F32, L.BF16):
        la, za = _loss_call(lib, L, dd.Y, rows, dd.sf, m, d, p, gdt)
        lb, zb = _loss_call(lib, L, Yg, None, sfg, m, d, p, gdt)
        assert torch.isfinite(la).all() and torch.equal(la, lb), (gdt, la.item(), lb.item())
        for k in range(3):
            assert torch.equal(za[k], zb[k]), (gdt, k)


def _engine(B, x_dtype="bfloat16", ae_type="zinb-conddisp", **kw):
    from dca_b200.engine import DeviceEngine
    return DeviceEngine(G, G, (64, 32, 64), ae_type, True, max_batch=B, x_dtype=x_dtype, device=DEV, seed=5, **kw)


def _outputs(eng, B):
    cond = eng.ae_type not in ("zinb", "nb", "poisson", "normal")
    out = {"mean": torch.empty((B, G), device=DEV), "latent": torch.empty((B, eng.latent_dim), device=DEV)}
    if cond:
        out["disp"] = torch.empty((B, G), device=DEV)
        out["pi"] = torch.empty((B, G), device=DEV)
    return out


def _compare(a, b, exact, what):
    """Bit for bit when exact; else (split-K or gradient sums with atomics: two runs of one arm differ in the last bits)
    within 1e-5 norm-wise -- a row read from the wrong place moves a batch of 132 rows by far more."""
    if exact:
        assert _same_bits(a, b), what
        return
    a, b = a.double().cpu(), b.double().cpu()
    assert a.shape == b.shape, what
    err = float((a - b).norm() / max(float(b.norm()), 1e-30))
    assert err <= 1e-5, (what, err)


def _step_pair(X, Y, sf, rows, gathered, make, exact):
    """train_step / eval_step / predict on the big (X, Y, sf) with rows= against a second engine in the same state fed
    the gathered contiguous rows: predict outputs, eval loss, training loss, gradients and BatchNorm state; when exact,
    also the parameters after apply_update and two more steps (the step graph's capture and a replay) on new batches
    drawn from the same rows."""
    a, b = make(), make()
    Xg, Yg, sfg = gathered
    B = rows.numel()
    side = torch.cuda.Stream(DEV)
    with torch.cuda.stream(side):
        oa, ob = _outputs(a, B), _outputs(b, B)
        a.predict(X, sf, rows=rows, **oa)
        b.predict(Xg, sfg, **ob)
        side.synchronize()
        for k in oa:
            _compare(oa[k], ob[k], exact, "predict " + k)
        a.read_epoch_acc(reset=True); b.read_epoch_acc(reset=True)
        a.eval_step(X, Y, sf, rows=rows)
        b.eval_step(Xg, Yg, sfg)
        ea, eb = a.read_epoch_acc(), b.read_epoch_acc()
        assert ea[3] == eb[3] == B * G
        assert (ea[2] == eb[2]) if exact else abs(ea[2] - eb[2]) <= 1e-5 * abs(eb[2]), ("eval loss", ea, eb)
        perm = np.random.default_rng(SEED + 4).permutation(B)
        rows_s = torch.empty_like(rows); Xs, Ys, sfs = (torch.empty_like(t) for t in (Xg, Yg, sfg))
        for it in range(3 if exact else 1):             # direct call, graph capture, replay
            p = torch.from_numpy(np.roll(perm, it) if it else np.arange(B)).to(DEV)
            rows_s.copy_(rows[p]); Xs.copy_(Xg[p]); Ys.copy_(Yg[p]); sfs.copy_(sfg[p])
            a.train_step(X, Y, sf, rows=rows_s)
            b.train_step(Xs, Ys, sfs)
            side.synchronize()
            la, lb = a.read_loss(), b.read_loss()
            assert np.isfinite(la), (it, la)
            assert (la == lb) if exact else abs(la - lb) <= 1e-5 * abs(lb), ("loss", it, la, lb)
            _compare(a.grads, b.grads, exact, "gradients, step %d" % it)
            _compare(a.bn_state, b.bn_state, exact, "BatchNorm state, step %d" % it)
            if exact:
                a.apply_update(1e-3, 5.0); b.apply_update(1e-3, 5.0)
                side.synchronize()
                assert torch.equal(a.params, b.params), "parameters after step %d" % it
    if exact:
        assert a.info()["step_graphs"] >= 1
    a.close(); b.close()


STEP_CASES = {
    # name: (engine keywords, bit-identical)
    "tc": (dict(), True),                                            # K1 / K5 rows, heads + loss kernel
    "tc_fused_heads": (dict(), False),                               # flash_zinb.cu (fused_heads): gradient atomics
    "input_dropout": (dict(input_dropout=0.1), True),                # activations.cu gathers + masks the rows
    "generic": (dict(gemm_path="generic"), False),                   # dense_generic.cu a_rows
    "poisson": (dict(ae_type="poisson"), False),                     # extra_types.cu
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(STEP_CASES))
def test_step_rows_equals_gathered_batch(counts, case):
    """The step, eval and predict reading the boundary batch in place from the bf16 dataset (13 GB: X past 2^32 bytes,
    Y past 2^31 elements) against the gathered rows, on the tensor-core path (K1 / K5 with rows, the heads + loss kernel
    on aligned counts), the fused heads kernel, input dropout, the generic GEMMs and the poisson extra type."""
    from dca_b200 import _lib
    kw, exact = STEP_CASES[case]
    dd = _resident(counts, "bfloat16")
    _assert_past_boundaries(BATCH)
    rows = _rows_d(BATCH)
    gathered = tuple(t[rows.long()].contiguous() for t in (dd.X, dd.Y, dd.sf))

    def make():
        eng = _engine(len(BATCH), **kw)
        if case == "tc":
            assert eng.info()["tc_heads"] and eng.info()["tc_encoder"]
        return eng
    if case == "tc_fused_heads":
        _lib.set_tunable("fused_heads", 1)
    try:
        _step_pair(dd.X, dd.Y, dd.sf, rows, gathered, make, exact)
    finally:
        if case == "tc_fused_heads":
            _lib.set_tunable("fused_heads", 0)


@pytest.mark.gpu
def test_resident_fp32_x(counts, ref):
    """X in fp32 (8.8 GB, byte offsets past 2^32 from ROW_F32_BYTES): the boundary rows within one ulp of the reference
    and equal, rounded to bf16, to the bf16 dataset's rows; the step reading fp32 rows in place (layers.cu: gather +
    convert for the tensor-core encoder) bit-identical to the step on the gathered rows."""
    snap = _snapshot(counts)
    dd = _resident(counts, "float32")
    assert dd.X.dtype == torch.float32
    _assert_past_boundaries(BOUNDARY)
    r = torch.from_numpy(BOUNDARY).to(DEV)
    X = dd.X[r].cpu()
    Xr = ref["x_rows"](BOUNDARY)
    Xn = X.numpy()
    assert np.all(np.abs(Xn.astype(np.float64) - Xr) <= np.spacing(np.maximum(np.abs(Xn), np.abs(Xr))))
    assert torch.equal(X.to(torch.bfloat16), snap["X"])
    assert _same_bits(dd.mean, torch.from_numpy(snap["mean"])) and _same_bits(dd.std, torch.from_numpy(snap["std"]))
    rows = _rows_d(BATCH)
    gathered = tuple(t[rows.long()].contiguous() for t in (dd.X, dd.Y, dd.sf))
    _step_pair(dd.X, dd.Y, dd.sf, rows, gathered, lambda: _engine(len(BATCH), x_dtype="float32"), True)


# ---------------------------------------------------------------------------------------------- 3. packed in HBM
def _packed_rows_host(pdd, rows):
    """(packed bytes [rows x row bytes], overflow entry bytes per row, nibble bytes per row or None) of the storage rows
    ``rows``, read at their absolute offsets in the device arrays."""
    rb = G // 8 if pdd.bits == 1 else G * pdd.bits // 8
    r = torch.from_numpy(np.asarray(rows, np.int64)).to(DEV)
    idx = r[:, None] * rb + torch.arange(rb, device=DEV)[None, :]
    packed = pdd.packed[idx].cpu().numpy()
    ip = pdd.ovf_indptr.cpu().numpy()
    ent = [pdd.entries[8 * ip[x]: 8 * ip[x + 1]].cpu().numpy() for x in rows]
    nib = None
    if pdd.bits == 1:
        np_ = pdd.nib_indptr.cpu().numpy()
        nib = [pdd.nibbles[np_[x]: np_[x + 1]].cpu().numpy() for x in rows]
    return packed, ent, nib


@pytest.mark.gpu
@pytest.mark.parametrize("bits", [16, "sparse"])
def test_packed_in_hbm(counts, bits):
    """PackedDeviceDataset.from_counts (16 bits: 4.4 GB of packed bytes, offsets past 2^32 from ROW_ELEMS): statistics
    bit-identical to the resident dataset; the boundary rows' packed bytes, overflow entries and nibbles those io.pack_rows
    writes for the same rows (offsets relative there, absolute here); dca_expand_rows_exact over the boundary rows
    (duplicates included) the resident Y, X and sf rows; dca_packed_train_step on them the resident step."""
    from dca_b200 import io
    from dca_b200.packed_data import PackedDeviceDataset
    snap = _snapshot(counts)
    need = N * G * 2 + (3 << 30) if bits == 16 else N * G // 2 + (3 << 30)
    pdd = _big("packed %s" % bits, need,
               lambda: PackedDeviceDataset.from_counts(counts, DEV, x_dtype="bfloat16", bits=bits))
    assert pdd.bits == (1 if bits == "sparse" else bits)
    if bits == 16:
        assert pdd.packed.numel() == N * G * 2 > 2 ** 32
    assert np.array_equal(pdd.n_counts_host, snap["n_counts"]) and np.array_equal(pdd.size_factors_host, snap["sf"])
    assert _same_bits(torch.from_numpy(pdd.mean), torch.from_numpy(snap["mean"]))
    assert _same_bits(torch.from_numpy(pdd.std), torch.from_numpy(snap["std"]))
    assert pdd.median == snap["median"] and pdd.flags == snap["flags"]

    # the packer's bytes
    _assert_past_boundaries(BOUNDARY)
    want = io.pack_rows(counts[BOUNDARY], bits, batch=None)
    assert want.bits == pdd.bits
    packed, ent, nib = _packed_rows_host(pdd, BOUNDARY)
    assert np.array_equal(packed, np.ascontiguousarray(want.packed).view(np.uint8).reshape(len(BOUNDARY), -1))
    want_ent = want.entries.view(np.uint8)
    for i, r in enumerate(BOUNDARY):
        assert np.array_equal(ent[i], want_ent[8 * want.indptr[i]: 8 * want.indptr[i + 1]]), r
        if nib is not None:
            assert np.array_equal(nib[i], want.nibbles[want.nib_indptr[i]: want.nib_indptr[i + 1]]), r
    deep = [i for i, r in enumerate(BOUNDARY) if r in DEEP_ROWS]
    assert len(deep) == len(DEEP_ROWS) and all(len(ent[i]) > 0 for i in deep)

    # the row-indexed exact expansion
    _assert_past_boundaries(BATCH)
    Yp, Xp, sfp = pdd.take(BATCH).expand()
    Ys, Xs, sfs = _snap_rows(snap, BATCH)
    assert _same_bits(Yp, Ys) and _same_bits(Xp, Xs) and _same_bits(sfp, sfs)
    del Yp, Xp, sfp

    # one packed training step against the resident step on the gathered rows
    rows = _rows_d(BATCH)
    a, b = _engine(len(BATCH)), _engine(len(BATCH))
    a.set_input_transform_exact(pdd.mean, pdd.std, pdd.median, pdd.flags)
    a.packed_train_step(pdd, rows)
    b.train_step(Xs, Ys, sfs)
    torch.cuda.synchronize()
    assert a.read_loss() == b.read_loss()
    assert torch.equal(a.grads, b.grads) and torch.equal(a.bn_state, b.bn_state)
    a.apply_update(1e-3, 5.0); b.apply_update(1e-3, 5.0)
    torch.cuda.synchronize()
    assert torch.equal(a.params, b.params)
    a.close(); b.close()


# ---------------------------------------------------------------------------------------------- 4. out of core
@pytest.mark.gpu
def test_streamed_statistics_and_predict(counts):
    """StreamedDataset.from_counts: the chunked statistics passes (dca_count_totals_rows, dca_log_moments_rows), whose
    chunks start past both boundaries, bit-identical to the resident dataset; one streamed predict batch (the last: it
    holds ROW_ELEMS and N - 1) bit-identical to predict on the resident rows."""
    from dca_b200.stream_data import StreamedDataset
    snap = _snapshot(counts)
    chunk = 3000
    starts = np.arange(0, N, chunk)
    assert (starts * G * 4 >= 2 ** 32).any() and (starts * G >= 2 ** 31).any()
    sd = _big("streamed", 4 << 30, lambda: StreamedDataset.from_counts(counts, DEV, x_dtype="bfloat16", batch=STREAM_BS,
                                                                       chunk_rows=chunk))
    assert np.array_equal(sd.n_counts_host, snap["n_counts"]) and np.array_equal(sd.size_factors_host, snap["sf"])
    assert _same_bits(torch.from_numpy(sd.mean), torch.from_numpy(snap["mean"]))
    assert _same_bits(torch.from_numpy(sd.std), torch.from_numpy(snap["std"]))
    assert sd.median == snap["median"] and sd.flags == snap["flags"]

    s0 = STREAM_BATCH * STREAM_BS
    nb = min(N, s0 + STREAM_BS) - s0
    _assert_past_boundaries(np.arange(s0, s0 + nb), both_sides=False)
    eng = _engine(STREAM_BS)
    out_s, out_r = _outputs(eng, STREAM_BS), _outputs(eng, STREAM_BS)
    sd.stream_batches(eng, STREAM_BS)
    try:
        eng.stream_predict(STREAM_BATCH, -1, **out_s)
    finally:
        eng.stream_end()
    Xr, sfr = snap["stream_X"].to(DEV), snap["stream_sf"].to(DEV)
    assert Xr.shape[0] == sfr.shape[0] == nb
    eng.predict(Xr, sfr, **out_r)
    torch.cuda.synchronize()
    for k in out_s:
        assert _same_bits(out_s[k][:nb], out_r[k][:nb]), k
    eng.close()
