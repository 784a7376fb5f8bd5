"""--debug without a GPU: the NumPy statement of the checked terms, the FloatingPointError message, the fit loop's check
before every update, and the C ABI of the report."""
import ctypes as C
import re

import numpy as np
import pytest

from tests.debug_terms import debug_report, debug_terms


def _batch(B=5, G=7, seed=0):
    r = np.random.default_rng(seed)
    y = r.poisson(2.0, (B, G)).astype(np.float32)
    m = r.uniform(0.1, 10, (B, G)).astype(np.float32)
    th = r.uniform(0.1, 100, (B, G)).astype(np.float32)
    sf = r.uniform(0.5, 2, B).astype(np.float32)
    return y, m, sf, th


def test_finite_batch_reports_nothing():
    assert debug_report(*_batch()) == {"count": [0, 0, 0], "first": [None, None, None]}


def test_huge_count_flags_t1_at_that_element_only():
    y, m, sf, th = _batch()
    y[3, 4] = 1e38                                   # float32 lgamma(1e38) is inf
    r = debug_report(y, m, np.ones_like(sf), th)
    assert r["count"][0] == 0 and r["first"][0] is None
    assert r["count"][1] == 1 and r["first"][1] == (3, 4)
    yp, t1, t2 = debug_terms(y, m, None, th)
    assert np.isfinite(np.delete(t2.ravel(), 3 * 7 + 4)).all()


def test_nan_mean_column_flags_y_pred_and_t2_not_t1():
    y, m, sf, th = _batch()
    m[:, 2] = np.nan
    r = debug_report(y, m, sf, th)
    assert r["count"] == [5, 0, 5] and r["first"] == [(0, 2), None, (0, 2)]


def test_nan_theta_flags_t1_t2_not_y_pred():
    y, m, sf, th = _batch()
    g = np.ones(7, np.float32); g[5] = np.nan            # const-disp: one theta per gene
    r = debug_report(y, m, sf, g)
    assert r["count"] == [0, 5, 5] and r["first"] == [None, (0, 5), (0, 5)]
    th[2, 1] = np.nan                                    # per element
    assert debug_report(y, m, sf, th)["first"][1] == (2, 1)


def test_message_names_first_failing_term_in_reference_order():
    from dca_b200.train import debug_message
    rep = {"count": [0, 2, 3], "first": [None, (1, 4), (0, 6)]}
    msg = debug_message(rep, 3, "training", 7, np.array([10, 42, 11]), ["c%d" % i for i in range(50)],
                        ["g%d" % i for i in range(9)])
    assert msg.startswith("t1 has inf/nans")
    assert "epoch 3" in msg and "training batch 7" in msg
    assert "cell 42 (c42)" in msg and "gene 4 (g4)" in msg
    assert "y_pred 0, t1 2, t2 3" in msg
    msg = debug_message({"count": [1, 1, 0], "first": [(0, 0), (2, 1)]  + [None]}, 1, "validation", 0, [5, 6, 7])
    assert msg.startswith("y_pred has inf/nans") and "validation batch 0" in msg and "cell 5, gene 0;" in msg
    msg = debug_message({"count": [0, 0, 4], "first": [None, None, None]}, 2, "training", 1, [])
    assert msg.startswith("t2 has inf/nans") and "another rank" in msg


def test_check_runs_before_the_update():
    """A failing check stops the epoch before that batch's update: the updates of the batches before it only."""
    import torch
    from dca_b200.device_data import _resident_fit

    class Eng:
        device = torch.device("cpu")
    steps, updates, seen = [], [], []
    epoch, validate = _resident_fit(Eng(), 10, 14, 4, False, lambda rows: steps.append(rows.tolist()),
                                    lambda s, e: steps.append((s, e)))

    def check(pos):
        seen.append(list(pos))
        if len(seen) == 2:
            raise FloatingPointError("t1 has inf/nans")
    with pytest.raises(FloatingPointError):
        epoch(lambda: updates.append(len(steps)), check)
    assert steps == [[0, 1, 2, 3], [4, 5, 6, 7]] and updates == [1] and seen == [[0, 1, 2, 3], [4, 5, 6, 7]]
    seen.clear()
    validate(seen.append)
    assert [list(p) for p in seen] == [[10, 11, 12, 13]]
    epoch(lambda: None)                                  # without a check: as before


def test_abi_symbols_and_struct_guard():
    from dca_b200 import _lib
    lib = _lib.load()
    assert {"dca_set_debug_checks", "dca_read_debug_report"} <= set(_lib.PROTOTYPES)
    r = _lib.DebugReport()
    r.struct_bytes = 1
    assert lib.dca_read_debug_report(None, C.byref(r), None) == -1
    size = int(re.search(r"struct_bytes must be (\d+)", lib.dca_last_error().decode()).group(1))
    assert size == C.sizeof(_lib.DebugReport) == 56
    r.struct_bytes = size
    assert lib.dca_read_debug_report(None, C.byref(r), None) == -1
    assert "handle is NULL" in lib.dca_last_error().decode()
    assert lib.dca_set_debug_checks(None, 1) == -1
