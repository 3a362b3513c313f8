"""The DPM-Solver++ chain's host side on the CPU: the coefficient / key / slot tables smd_dpm_tables builds against
the float64 restatement, the order rule, the identity of order 1 with the DDIM eta = 0 step, the observed order of
convergence on Gaussian data, the rejections of the new entry points and the command-line flags."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import ddpm_oracle as O
from smd_b200 import Engine, ModelConfig, ebm_utils
from smd_b200 import lib as L
from tests import ddim_reference as DR
from tests import dpm_reference as R

BETAS = O.create_noise_schedule(1e-4, 0.02, 1000, "linear")


def _fp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))


def _ip(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_int))


def _tables(betas, steps, order, key=(0, 7)):
    lib = L.load_library()
    b = np.ascontiguousarray(betas, np.float32)
    s = np.ascontiguousarray(steps, np.int32)
    K = len(s)
    coef = np.zeros((K, 8), np.float32)
    keys = np.zeros((K, 4), np.uint32)
    slots = np.zeros((K,), np.int32)
    k = (ctypes.c_uint32 * 2)(*key)
    L.check(lib.smd_dpm_tables(_fp(b), len(b), _ip(s), K, int(order), k, _fp(coef),
                               keys.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)), _ip(slots)))
    return coef, keys, slots


def _ddim_tables(betas, steps, key=(0, 7)):
    lib = L.load_library()
    b = np.ascontiguousarray(betas, np.float32)
    s = np.ascontiguousarray(steps, np.int32)
    K = len(s)
    coef = np.zeros((K, 8), np.float32)
    keys = np.zeros((K, 4), np.uint32)
    slots = np.zeros((K,), np.int32)
    k = (ctypes.c_uint32 * 2)(*key)
    L.check(lib.smd_ddim_tables(_fp(b), len(b), _ip(s), K, 0.0, k, _fp(coef),
                                keys.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)), _ip(slots)))
    return coef, keys, slots


SCHEDULES = {
    "uniform50": ebm_utils.ddim_schedule(1000, 50),
    "quadratic20": ebm_utils.ddim_schedule(1000, 20, "quadratic"),
    "one": np.asarray([999]),
    "irregular": np.asarray([3, 17, 500, 501, 640, 998]),
    "full": np.arange(1000),
}


# --------------------------------------------------------------------------------------------------------- tables
@pytest.mark.parametrize("order", [1, 2, 3])
@pytest.mark.parametrize("name", sorted(SCHEDULES))
def test_coefficient_table_matches_float64(lib, name, order):
    steps = SCHEDULES[name]
    coef, keys, slots = _tables(BETAS, steps, order)
    tab = R.tables(BETAS, steps, order)
    for j, key in [(0, "sqrt_recip"), (1, "sqrt_m1"), (5, "sqrt_a"), (7, "a")]:
        np.testing.assert_allclose(coef[:, j], tab[key], rtol=1e-6, atol=0, err_msg=key)
    np.testing.assert_array_equal(coef[:, 7], DR.alpha_bar(BETAS)[steps])        # alpha_bar as the ddpm chain
    # the four solver coefficients, each against the size of the step's largest one: the order-3 ones are
    # differences of terms up to ~1/r larger than the result, which the float64 restatement and the library's
    # gathered closed form round differently
    got = coef[:, [2, 3, 4, 6]].astype(np.float64)
    want = np.stack([tab["c_x"], tab["c_0"], tab["c_1"], tab["c_2"]], axis=1)
    scale = np.abs(want).max(axis=1, keepdims=True)
    err = np.abs(got - want) / scale
    assert err.max() < 2e-6, (float(err.max()), np.unravel_index(err.argmax(), err.shape))
    # the key and slot tables are the DDIM chain's
    _, dkeys, dslots = _ddim_tables(BETAS, steps)
    np.testing.assert_array_equal(keys, dkeys)
    np.testing.assert_array_equal(slots, dslots)


@pytest.mark.parametrize("order", [1, 2, 3])
def test_order_rule(lib, order):
    steps = SCHEDULES["uniform50"]
    coef, _, _ = _tables(BETAS, steps, order)
    K = len(steps)
    for i in range(K):
        o = R.step_order(i, K, order)
        assert (coef[i, 4] != 0) == (o >= 2), (i, coef[i])
        assert (coef[i, 6] != 0) == (o >= 3), (i, coef[i])
        if o < 2:
            assert coef[i, 4] == 0.0 and coef[i, 6] == 0.0      # exactly: the kernel then leaves the history unread
    # the first step has no history; the second has one estimate
    assert coef[K - 1, 4] == 0 and coef[K - 1, 6] == 0
    assert coef[K - 2, 6] == 0
    # the last step lands on the data: x' = m0
    np.testing.assert_array_equal(coef[0, [2, 3, 4, 6]], [0.0, 1.0, 0.0, 0.0])
    one, _, _ = _tables(BETAS, [999], order)
    np.testing.assert_array_equal(one[0, [2, 3, 4, 6]], [0.0, 1.0, 0.0, 0.0])


@pytest.mark.parametrize("name", ["uniform50", "quadratic20", "irregular", "full"])
def test_order_one_is_the_ddim_eta_zero_step(lib, name):
    """c_x x + c_0 m0 = sqrt(a') m0 + sqrt(1-a') (x - sqrt(a) m0) / sqrt(1-a) for every (x, m0)."""
    steps = SCHEDULES[name]
    g = np.random.default_rng(len(steps))
    x = g.standard_normal((len(steps), 64)) * 1.5
    m0 = g.uniform(-1, 1, (len(steps), 64))
    dd = DR.tables(BETAS, steps, 0.0)

    def ddim(t):
        return (t["c_x0"][:, None] * m0 + t["c_dir"][:, None] * (x - t["sqrt_a"][:, None] * m0)
                / t["sqrt_1m"][:, None])
    want = ddim(dd)
    tab = R.tables(BETAS, steps, 1)
    got = tab["c_x"][:, None] * x + tab["c_0"][:, None] * m0
    err = np.abs(got - want).max() / np.abs(want).max()
    assert err < 1e-12, err
    # the library's float32 tables: the same step to float32 rounding of the coefficients
    coef, _, _ = _tables(BETAS, steps, 1)
    lt = R.library_tables(coef)
    got32 = lt["c_x"][:, None] * x + lt["c_0"][:, None] * m0
    dcoef, _, _ = _ddim_tables(BETAS, steps)
    want32 = (dcoef[:, 2, None] * m0 + dcoef[:, 3, None] * (x - dcoef[:, 5, None] * m0) / dcoef[:, 6, None])
    assert np.abs(got32 - want32).max() / np.abs(want32).max() < 1e-6


# ------------------------------------------------------------------------------------------------- convergence
MU, S = 0.3, 2.0        # data N(MU, S^2) per element; the clipping is off, so the data may pass [-1, 1]


def _gauss_eps(x, cond):
    """The exact noise prediction for data N(MU, S^2): sqrt(1-a) (x - sqrt(a) MU) / (a S^2 + 1 - a)."""
    a = cond * cond
    return torch.sqrt(1 - a) * (x - cond * MU) / (a * S * S + 1 - a)


def _ode_error(K, order, init):
    """rel-L2 of the chain's state at level tau_0 (before the final step) against the probability-flow ODE's exact
    solution, on the library's own tables with the clipping off."""
    steps = ebm_utils.ddim_schedule(1000, K)
    coef, _, _ = _tables(BETAS, steps, order)
    x, _, _ = R.dpm_chain(_gauss_eps, BETAS, steps, order, init, (0, 0), tab=R.library_tables(coef), clip=False,
                          stop_before_last=True)
    a = R.levels(BETAS, steps)
    aT, a0 = a[-1], a[0]
    # the ODE keeps (x - sqrt(a) MU) / sqrt(a S^2 + 1 - a) constant
    exact = np.sqrt(a0) * MU + np.sqrt(a0 * S * S + 1 - a0) * (init - np.sqrt(aT) * MU) / np.sqrt(aT * S * S + 1 - aT)
    return float((x - exact).norm() / exact.norm())


def test_convergence_order_on_gaussian_data(lib):
    init = torch.from_numpy(np.random.default_rng(0).standard_normal((16, 64)))
    Ks = (10, 20, 40, 80)
    e = {o: [_ode_error(K, o, init) for K in Ks] for o in (1, 2, 3)}
    p = {o: [float(np.log2(e[o][k] / e[o][k + 1])) for k in range(3)] for o in (1, 2, 3)}
    # the restatement shows, on the uniform schedule over this T = 1000 linear schedule:
    #   order 1: 1.5e-1 7.6e-2 3.8e-2 1.9e-2 (observed order 1.02 1.01 1.00)
    #   order 2: 1.7e-1 3.9e-2 8.6e-3 1.9e-3 (2.13 2.20 2.15)
    #   order 3: 3.7e-1 8.6e-2 1.2e-2 1.7e-3 (2.12 2.79 2.90)
    assert all(0.9 < v < 1.15 for v in p[1]), e
    assert all(1.8 < v < 2.5 for v in p[2]), e
    assert all(e[2][k] < e[1][k] for k in range(1, 4)), e
    # order 3 starts with a first- and a second-order step, which caps its global order: on this schedule it is
    # less accurate than order 2 up to K = 40 and passes it at K = 80, converging faster
    assert e[3][3] < e[2][3], e
    assert all(v > 2.4 for v in p[3][1:]), e


# --------------------------------------------------------------------------------------------------- rejections
def _engine(arch="TransformerDDPM", **kw):
    cfg = dict(channels=42)
    if arch == "TransformerMDN":
        cfg.update(num_layers=1, num_mlp_layers=1)
    return Engine(ModelConfig(arch=arch, **cfg), **kw)


def test_rejections(lib):
    key = (ctypes.c_uint32 * 2)(0, 1)
    b = np.ascontiguousarray(O.create_noise_schedule(1e-4, 0.02, 10, "linear"), np.float32)
    eng = _engine(max_batch=4)
    good = np.arange(0, 10, 3, dtype=np.int32)
    bad = [
        (b, 10, good, 4, 0, "order"),
        (b, 10, good, 4, 4, "order"),
        (b, 10, good, 4, -1, "order"),
        (b, 1, np.asarray([0, 5], np.int32), 2, 2, "in \\[1, T\\]"),            # K > T
        (b, 10, np.asarray([5, 5], np.int32), 2, 2, "strictly increasing"),
        (b, 10, np.asarray([6, 2], np.int32), 2, 2, "strictly increasing"),
        (b, 10, np.asarray([-1, 2], np.int32), 2, 2, "strictly increasing"),
        (b, 10, np.asarray([2, 10], np.int32), 2, 2, "strictly increasing"),
        (b, 10, good, 0, 2, "in \\[1, T\\]"),
        (b, 0, good, 1, 2, "T out of range"),
        (np.zeros(8193, np.float32) + 1e-3, 8193, good, 4, 2, "T out of range"),
        (np.zeros(10, np.float32), 10, good, 4, 2, "alpha_bar"),               # beta = 0: alpha_bar = 1
    ]
    for bb, T, s, K, order, msg in bad:
        with pytest.raises(ValueError, match=msg):
            L.check(lib.smd_dpm_tables(_fp(bb), T, _ip(s), K, order, key, None, None, None))
        with pytest.raises(ValueError, match=msg):
            L.check(lib.smd_dpm_setup(eng._plan, _fp(bb), T, _ip(s), K, order, key, None))
    for order in (1, 2, 3):
        L.check(lib.smd_dpm_tables(_fp(b), 10, _ip(good), 4, order, key, None, None, None))
    # valid arguments on a plan without a workspace: a call-order error
    with pytest.raises(L.SmdError, match="workspace not bound"):
        L.check(lib.smd_dpm_setup(eng._plan, _fp(b), 10, _ip(good), 4, 2, key, None))
    # more samples than the plan holds and a half infill pair come before the setup check
    with pytest.raises(ValueError, match="n out of range"):
        L.check(lib.smd_dpm_sample(eng._plan, None, None, 5, None, None, None, None, None, 1, None))
    with pytest.raises(ValueError, match="go together"):
        L.check(lib.smd_dpm_sample(eng._plan, None, None, 4, None, None, 1024, None, None, 1, None))
    with pytest.raises(L.SmdError, match="smd_dpm_setup has not been called"):
        L.check(lib.smd_dpm_sample(eng._plan, None, None, 4, None, None, None, None, None, 1, None))
    mdn = _engine("TransformerMDN", max_batch=4)
    with pytest.raises(ValueError, match="TransformerMDN"):
        L.check(lib.smd_dpm_setup(mdn._plan, _fp(b), 10, _ip(good), 4, 2, key, None))
    with pytest.raises(ValueError, match="TransformerMDN"):
        L.check(lib.smd_dpm_sample(mdn._plan, None, None, 4, None, None, None, None, None, 1, None))
    with pytest.raises(ValueError, match="order"):
        ebm_utils.dpm_solver_dynamics((0, 0), None, b, None, None, None, None, order=4)


def test_flags_and_dispatch():
    from absl import flags

    from smd_b200 import train_ncsn
    fl = flags.FLAGS
    assert "dpm" in fl["sampling"].parser.enum_values
    assert fl["dpm_steps"].default == 20 and fl["dpm_order"].default == 2
    assert fl["dpm_schedule"].default == "uniform"
    assert list(fl["dpm_schedule"].parser.enum_values) == list(ebm_utils.DDIM_SCHEDULES)
    for bad in ("0", "4"):
        with pytest.raises(flags.IllegalFlagValueError):
            fl["dpm_order"].parse(bad)
    if not fl.is_parsed():
        fl.mark_as_parsed()
    alg = train_ncsn.dpm_algorithm()
    assert alg.func is ebm_utils.dpm_solver_dynamics
    assert alg.keywords == dict(steps=20, order=2, schedule="uniform")


def test_interpolate_rejects_dpm():
    from absl import flags

    from smd_b200 import sample_ncsn
    fl = flags.FLAGS
    if not fl.is_parsed():
        fl.mark_as_parsed()
    saved = fl.interpolate, fl.sampling
    try:
        fl.interpolate, fl.sampling = True, "dpm"
        with pytest.raises(ValueError, match="--sampling=dpm"):
            sample_ncsn.check_flags()
    finally:
        fl.interpolate, fl.sampling = saved
