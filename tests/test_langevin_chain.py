"""The Langevin chain's host side on the CPU: the per-level coefficients and the collection rows smd_langevin_setup
uploads against the float32 formulas of utils/ebm_utils.py:89-271, the rejections of the new entry points, and the
DenseNCSN workspace, which the chain reuses without growing.  Squares are written as products: the jitted reference's
`x ** 2` is lax.integer_pow, i.e. x * x, while numpy's float32 power can be one ulp away from it."""
import ctypes

import numpy as np
import pytest

from smd_b200 import Engine, ModelConfig
from smd_b200 import lib as L


def _tables(sigmas, T, epsilon, kind, rows):
    lib = L.load_library()
    s = np.ascontiguousarray(sigmas, np.float32)
    n = len(s)
    steps = n * T if kind == 0 else n
    coef = np.zeros((n, 4), np.float32)
    slots = np.zeros((steps,), np.int32)
    L.check(lib.smd_langevin_tables(s.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), n, T, float(epsilon), kind,
                                    rows, coef.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
                                    slots.ctypes.data_as(ctypes.POINTER(ctypes.c_int))))
    return coef, slots


def _schedule(L_, lo=0.01):
    from smd_b200 import ebm_utils
    return ebm_utils.create_noise_schedule(1.0, lo, L_, "geometric")


@pytest.mark.parametrize("L_,T,epsilon,denoise", [(2, 3, 2e-6, True), (5, 7, 1e-5, False), (20, 100, 2e-6, True),
                                                  (500, 100, 2e-6, True), (10, 10, 3e-5, False), (4, 1, 2e-6, True)])
def test_annealed_tables_match_float32_formulas(lib, L_, T, epsilon, denoise):
    from smd_b200 import ebm_utils
    sig = _schedule(L_)
    rows = 101 + int(denoise)
    coef, slots = _tables(sig, T, epsilon, 0, rows)
    for si in range(L_):
        s = np.float32(sig[si])
        q = s / np.float32(sig[-1])
        alpha = np.float32(epsilon) * (q * q)
        assert coef[si, 0] == s and coef[si, 1] == alpha, si
        assert coef[si, 2] == np.sqrt(np.float32(2) * alpha), si
    slot_of = ebm_utils._collection_slot_fn(L_ * T, 100)
    want = np.array([slot_of(j + 1) for j in range(L_ * T)], np.int32)
    want[want >= rows] = -1          # a repeated linspace index sums past the end: the update is dropped
    np.testing.assert_array_equal(slots, want)
    if L_ * T >= 100:
        assert sorted(slots[slots >= 0].tolist()) == list(range(1, 101))
    else:
        assert (slots >= 0).sum() <= L_ * T


@pytest.mark.parametrize("L_,epsilon", [(2, 2e-6), (10, 1e-4), (500, 2e-6)])
def test_consistent_tables_match_float32_formulas(lib, L_, epsilon):
    sig = _schedule(L_, 0.05)
    coef, _ = _tables(sig, 1, epsilon, 1, 101)
    r = np.float32(1) - np.float32(epsilon) / (sig[-1] * sig[-1])
    beta = np.sqrt(np.float32(1) - r * r).astype(np.float32)
    for i in range(L_):
        nxt = np.float32(sig[i + 1]) if i < L_ - 1 else np.float32(0)
        q = np.float32(sig[i]) / np.float32(sig[-1])
        alpha = np.float32(epsilon) * (q * q)
        assert coef[i, 0] == sig[i] and coef[i, 1] == alpha and coef[i, 2] == beta * nxt, i
    assert coef[-1, 2] == 0


def _engine(arch, **kw):
    cfg = dict(channels=512, mlp_dims=2048, num_layers=3) if arch == "DenseNCSN" else dict(channels=42)
    if arch == "TransformerMDN":
        cfg.update(num_layers=1, num_mlp_layers=1)
    return Engine(ModelConfig(arch=arch, **cfg), **kw)


def test_rejections(lib):
    key = (ctypes.c_uint32 * 2)(0, 1)
    sig = np.asarray([1.0, 0.5, 0.1], np.float32)
    fp = sig.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
    eng = _engine("TransformerDDPM", max_batch=4)
    bad = [(fp, 1, 10, 0), (fp, 8193, 10, 0), (fp, 3, 10, 2), (fp, 3, 10, -1), (fp, 3, 0, 0)]
    for args in bad:
        with pytest.raises(ValueError):
            L.check(lib.smd_langevin_setup(eng._plan, args[0], args[1], args[2], 1e-5, args[3], key, None))
        with pytest.raises(ValueError):
            L.check(lib.smd_langevin_tables(args[0], args[1], args[2], 1e-5, args[3], 101, None, None))
    # the consistent chain ignores steps_per_level
    L.check(lib.smd_langevin_tables(fp, 3, 0, 1e-5, 1, 101, None, None))
    # more samples than the plan holds; the schedule check comes after it
    with pytest.raises(ValueError, match="n out of range"):
        L.check(lib.smd_langevin_sample(eng._plan, None, None, 5, None, None, 1, None, None, 1, None))
    with pytest.raises(L.SmdError, match="smd_langevin_setup"):
        L.check(lib.smd_langevin_sample(eng._plan, None, None, 4, None, None, 1, None, None, 1, None))
    mdn = _engine("TransformerMDN", max_batch=4)
    with pytest.raises(ValueError, match="TransformerMDN"):
        L.check(lib.smd_langevin_setup(mdn._plan, fp, 3, 10, 1e-5, 0, key, None))
    with pytest.raises(ValueError, match="TransformerMDN"):
        L.check(lib.smd_langevin_sample(mdn._plan, None, None, 4, None, None, 1, None, None, 1, None))
    with pytest.raises(ValueError, match="unknown Langevin sampler"):
        eng.langevin_setup(sig, 10, 1e-5, "ddpm")


# smd_workspace_bytes of DenseNCSN plans recorded at the commit before the Langevin chain: the chain reuses the
# sampler regions (coef, slots, t_ptr, ftab*) and adds none
PARENT_WORKSPACE_BYTES = {
    (128, False, "bf16"): 143292416,
    (128, True, "bf16"): 153101312,
    (128, False, "bf16x3"): 292876288,
    (1000, False, "bf16"): 225754112,
}


def test_dense_ncsn_workspace_is_unchanged(lib):
    for (mb, training, precision), want in PARENT_WORKSPACE_BYTES.items():
        assert _engine("DenseNCSN", max_batch=mb, training=training, precision=precision).workspace_bytes == want
