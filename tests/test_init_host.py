"""Kernel initializers without a GPU (include/dca_b200.h, "initializers"): the Keras name table, the fan rules of every
kernel of the eleven AE types, and the host restatement of the draws (dca_init_fill_host, the same source as the
device code) against oracle/init_ref.py, a NumPy restatement of the formulas.  Reference behaviour: --init
(dca/__main__.py:82), Dense(kernel_initializer=init) (dca/network.py:124-126)."""
import ctypes as C

import numpy as np
import pytest

from dca_b200 import _lib
from oracle import init_ref as R

AE_TYPES = list(_lib.AE_TYPE_IDS)
NAMES = sorted(R.SPECS)


def _fill(name_or_spec, seed, sid, shape):
    lib = _lib.load()
    spec = _lib.initializer(name_or_spec) if isinstance(name_or_spec, str) else name_or_spec
    ndim, rows, cols = (1, 1, shape[0]) if len(shape) == 1 else (2, shape[0], shape[1])
    out = np.empty(rows * cols, np.float32)
    st = lib.dca_init_fill_host(C.byref(spec), C.c_uint64(seed), C.c_uint64(sid), ndim, rows, cols,
                                out.ctypes.data_as(C.c_void_p))
    return st, out


def _ulps(a, b):
    a = np.asarray(a, np.float32).view(np.int32).astype(np.int64)
    b = np.asarray(b, np.float32).view(np.int32).astype(np.int64)
    a = np.where(a < 0, -(a & 0x7FFFFFFF), a)
    b = np.where(b < 0, -(b & 0x7FFFFFFF), b)
    return np.abs(a - b)


def test_every_keras_name_and_alias_resolves_to_the_table():
    kinds = {R.VS: _lib.INIT_VARIANCE_SCALING, "random_normal": _lib.INIT_RANDOM_NORMAL,
             "random_uniform": _lib.INIT_RANDOM_UNIFORM, "truncated_normal": _lib.INIT_TRUNCATED_NORMAL,
             "constant": _lib.INIT_CONSTANT, "orthogonal": _lib.INIT_ORTHOGONAL, "identity": _lib.INIT_IDENTITY}
    names = list(R.SPECS) + list(R.ALIASES) + list(R.CAMEL)
    assert len(set(names)) == 34
    for name in names:
        spec = _lib.initializer(name)
        kind, a = R.SPECS[R.canonical(name)]
        assert spec.struct_bytes == C.sizeof(_lib.Initializer)
        assert spec.kind == kinds[kind], name
        if kind == R.VS:
            assert (spec.scale, spec.mode, spec.distribution) == (
                a["scale"], _lib.FAN_MODES[a["mode"]], _lib.DISTRIBUTIONS[a["distribution"]]), name
        for field in ("stddev", "minval", "maxval", "value", "gain"):
            if field in a:
                assert getattr(spec, field) == np.float32(a[field]), (name, field)
    assert set(_lib.INITIALIZERS) == set(names)


@pytest.mark.parametrize("bad", ["he_normall", "Glorot_Uniform", "", "softmax", None, 3])
def test_unknown_initializer_is_a_value_error_listing_the_names(bad):
    with pytest.raises(ValueError) as e:
        _lib.initializer(bad)
    msg = str(e.value)
    assert "unknown initializer" in msg and all(n in msg for n in ("glorot_uniform", "he_normal", "orthogonal"))


def test_unknown_initializer_stops_the_model_build_before_any_device_work():
    from dca_b200.network import AE_types
    with pytest.raises(ValueError, match="unknown initializer"):
        AE_types["zinb-conddisp"](40, init="he_norm").build()


def test_cli_passes_init_through():
    from dca_b200.__main__ import build_parser
    assert build_parser().parse_args(["in.tsv", "out", "--init", "he_normal"]).init == "he_normal"


def test_invalid_specs_are_rejected():
    lib = _lib.load()
    out = np.empty(8, np.float32)
    spec = _lib.initializer("he_normal")
    spec.struct_bytes = 4
    assert lib.dca_init_fill_host(C.byref(spec), 0, 0, 2, 2, 4, out.ctypes.data_as(C.c_void_p)) == -1
    for field, value in (("kind", 7), ("scale", 0.0), ("mode", 3), ("distribution", 5)):
        spec = _lib.initializer("he_normal")
        setattr(spec, field, value)
        assert _fill(spec, 0, 0, (2, 4))[0] == -1, field
    spec = _lib.initializer("random_uniform"); spec.minval, spec.maxval = 1.0, -1.0
    assert _fill(spec, 0, 0, (2, 4))[0] == -1
    assert lib.dca_init_fill_host(C.byref(_lib.initializer("ones")), 0, 0, 1, 2, 4, out.ctypes.data_as(C.c_void_p)) == -1


@pytest.mark.parametrize("name", ["orthogonal", "identity", "Orthogonal", "Identity"])
def test_orthogonal_and_identity_refuse_a_1d_kernel(name):
    st, _ = _fill(name, 0, 0, (16,))
    assert st == -1 and b"2-D" in _lib.load().dca_last_error()
    with pytest.raises(ValueError):
        R.target(name, (16,))
    assert _fill(name, 0, 0, (16, 4))[0] == 0


@pytest.mark.parametrize("ae_type", AE_TYPES)
def test_fan_rules_for_every_kernel_of_every_type(ae_type):
    """fan_in / fan_out / fan_avg of each kernel, seen through the draws: the uniform variance-scaling limits follow the
    fans, and the library's draws match the restatement bit for bit."""
    G, hidden = 48, (16, 8, 16)
    table = R.kernels(ae_type, G, G, hidden, sharedpi=False)
    names = [n for n, _, _ in table]
    assert len(set(sid for _, _, sid in table)) == len(table)
    for name, shape, sid in table:
        fi, fo = R.fans(shape)
        if name == "pi/kernel" and ae_type == "zinb-elempi":
            assert shape == (G,) and (fi, fo) == (G, G)
        else:
            assert len(shape) == 2 and (fi, fo) == shape
        for mode, n in (("fan_in", fi), ("fan_out", fo), ("fan_avg", (fi + fo) / 2)):
            spec = _lib.initializer("variance_scaling")
            spec.mode, spec.distribution, spec.scale = _lib.FAN_MODES[mode], _lib.DISTRIBUTIONS["uniform"], 2.0
            st, w = _fill(spec, 5, sid, shape)
            assert st == 0
            assert np.abs(w).max() <= np.sqrt(6.0 / n) * (1 + 1e-6), (ae_type, name, mode)
        for init in ("glorot_uniform", "he_uniform", "lecun_uniform"):
            st, w = _fill(init, 5, sid, shape)
            np.testing.assert_array_equal(w, R.draw(init, 5, sid, shape).ravel(), err_msg="%s %s" % (name, init))
    if ae_type == "zinb-elempi":
        assert R.kernels(ae_type, G, G, hidden, sharedpi=True)[-1][1] == (1,)
    assert any(n.endswith("/kernel") for n in names)


@pytest.mark.parametrize("name", NAMES)
def test_host_draws_match_the_float64_formulas(name):
    shape, seed, sid = (64, 3000), 11, 101
    kind = R.target(name, shape)[0]
    st, w = _fill(name, seed, sid, shape)
    assert st == 0
    if kind == "orthogonal":
        A = R.normal_matrix(seed, sid, shape)
        assert A.shape == (3000, 64)
        assert _ulps(w, A.ravel()).max() <= 1
        return
    ref = R.draw(name, seed, sid, shape).ravel()
    if kind in ("uniform", "constant", "identity"):
        np.testing.assert_array_equal(w, ref)
    else:
        assert _ulps(w, ref).max() <= 1, name
    if kind == "truncated":
        sigma = R.target(name, shape)[1]
        assert np.abs(w.astype(np.float64)).max() <= 2 * sigma * (1 + 2.0 ** -23)
    if kind in ("normal", "truncated", "uniform"):
        # a sample of 192 000 draws: its moments are those of the target distribution
        t = R.target(name, shape)
        var = {"uniform": lambda: (t[2] - t[1]) ** 2 / 12, "normal": lambda: t[1] ** 2,
               "truncated": lambda: (t[1] * R.TRUNC_SD) ** 2}[kind]()
        assert abs(w.mean()) < 5 * np.sqrt(var / w.size)
        assert abs(w.astype(np.float64).var() / var - 1) < 0.02, name


def test_identity_is_eye_of_any_shape():
    for shape in ((4, 7), (7, 4), (5, 5)):
        st, w = _fill("identity", 0, 0, shape)
        np.testing.assert_array_equal(w.reshape(shape), np.eye(*shape, dtype=np.float32))


def test_draws_are_keyed_by_seed_stream_and_element():
    a = _fill("he_normal", 1, 0, (64, 500))[1]
    assert np.array_equal(a, _fill("he_normal", 1, 0, (64, 500))[1])
    assert not np.array_equal(a, _fill("he_normal", 2, 0, (64, 500))[1])
    assert not np.array_equal(a, _fill("he_normal", 1, 1, (64, 500))[1])
    # element i does not depend on the tensor's shape
    b = _fill("he_normal", 1, 0, (32, 1000))[1]
    s = R.target("he_normal", (32, 1000))[1] / R.target("he_normal", (64, 500))[1]
    assert _ulps(b, (a.astype(np.float64) * s).astype(np.float32)).max() <= 2
