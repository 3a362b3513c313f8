"""The DDIM chain's host side on the CPU: the schedules, the coefficient / key / slot tables smd_ddim_setup uploads
against the float64 restatement, the identity with the DDPM ancestral step at K = T and eta = 1, and the rejections
of the new entry points."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import ddpm_oracle as O
from oracle import threefry as tf
from smd_b200 import Engine, ModelConfig, ebm_utils
from smd_b200 import lib as L
from tests import ddim_reference as R

BETAS = O.create_noise_schedule(1e-6, 0.01, 1000, "linear")


def _fp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))


def _ip(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_int))


def _tables(betas, steps, eta, key=(0, 7)):
    lib = L.load_library()
    b = np.ascontiguousarray(betas, np.float32)
    s = np.ascontiguousarray(steps, np.int32)
    K = len(s)
    coef = np.zeros((K, 8), np.float32)
    keys = np.zeros((K, 4), np.uint32)
    slots = np.zeros((K,), np.int32)
    k = (ctypes.c_uint32 * 2)(*key)
    L.check(lib.smd_ddim_tables(_fp(b), len(b), _ip(s), K, float(eta), k, _fp(coef),
                                keys.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)), _ip(slots)))
    return coef, keys, slots


# ------------------------------------------------------------------------------------------------------ schedules
def test_uniform_schedule():
    tau = ebm_utils.ddim_schedule(1000, 50, "uniform")
    assert tau.dtype == np.int32 and len(tau) == 50 and tau[0] == 0 and tau[-1] == 999
    np.testing.assert_array_equal(tau, [round(i * 999 / 49) for i in range(50)])
    np.testing.assert_array_equal(ebm_utils.ddim_schedule(1000, 1000), np.arange(1000))
    np.testing.assert_array_equal(ebm_utils.ddim_schedule(1000, 1), [999])
    np.testing.assert_array_equal(ebm_utils.ddim_schedule(4, 3), [0, 2, 3])     # 1.5 rounds half to even
    for T, K in [(7, 7), (10, 3), (1000, 999), (8192, 37)]:
        assert (np.diff(ebm_utils.ddim_schedule(T, K)) > 0).all()


def test_quadratic_schedule():
    tau = ebm_utils.ddim_schedule(1000, 20, "quadratic")
    np.testing.assert_array_equal(tau, [round(999 * (i / 19) ** 2) for i in range(20)])
    assert tau[0] == 0 and tau[-1] == 999 and (np.diff(tau) > 0).all()
    np.testing.assert_array_equal(ebm_utils.ddim_schedule(10, 1, "quadratic"), [9])
    with pytest.raises(ValueError, match="repeats"):
        ebm_utils.ddim_schedule(10, 10, "quadratic")          # round(9 (1/9)^2) = 0 = tau_0
    with pytest.raises(ValueError, match="repeats"):
        ebm_utils.ddim_schedule(1000, 100, "quadratic")


@pytest.mark.parametrize("T,K,schedule", [(10, 0, "uniform"), (10, 11, "uniform"), (10, -1, "quadratic"),
                                          (10, 5, "cosine")])
def test_schedule_rejections(T, K, schedule):
    with pytest.raises(ValueError):
        ebm_utils.ddim_schedule(T, K, schedule)


# --------------------------------------------------------------------------------------------------------- tables
@pytest.mark.parametrize("steps,eta", [(np.arange(1000), 1.0), (ebm_utils.ddim_schedule(1000, 50), 0.0),
                                       (ebm_utils.ddim_schedule(1000, 20, "quadratic"), 0.5), ([999], 1.0),
                                       ([3, 17, 500, 501], 2.0)])
def test_coefficient_table_matches_float64(lib, steps, eta):
    coef, _, _ = _tables(BETAS, steps, eta)
    tab = R.tables(BETAS, steps, eta)
    names = ["sqrt_recip", "sqrt_m1", "c_x0", "c_dir", "sig", "sqrt_a", "sqrt_1m", "a"]
    for j, name in enumerate(names):
        np.testing.assert_allclose(coef[:, j], tab[name], rtol=1e-6, atol=1e-12, err_msg=name)
    assert coef[0, 2] == 1 and coef[0, 4] == 0          # the last step: a' = 1, no noise
    np.testing.assert_array_equal(coef[:, 7], R.alpha_bar(BETAS)[np.asarray(steps)])   # alpha_bar as the ddpm chain
    if eta == 0:
        assert (coef[:, 4] == 0).all()


def test_eta_one_full_schedule_is_the_posterior_variance(lib):
    coef, _, _ = _tables(BETAS, np.arange(1000), 1.0)
    # sig^2 = beta_tilde_t = beta_t (1 - alpha_bar_{t-1}) / (1 - alpha_bar_t), in float64 from the float32 alpha_bar
    ab = R.alpha_bar(BETAS).astype(np.float64)
    beta = 1 - ab[1:] / ab[:-1]
    tilde = beta * (1 - ab[:-1]) / (1 - ab[1:])
    np.testing.assert_allclose(coef[1:, 4].astype(np.float64) ** 2, tilde, rtol=1e-6)
    # the DDPM chain's float32 sigma loses up to ~1e-3 to the cancellation in 1 - alpha_bar near t = 0
    c = O.reverse_coefficients(BETAS)
    np.testing.assert_allclose(coef[1:, 4], c["sigma"][1:], rtol=5e-3)


def test_key_and_slot_tables_equal_the_ddpm_chain_at_k_equal_t(lib):
    T = 1000
    key = (3, 11)
    _, keys, slots = _tables(BETAS, np.arange(T), 1.0, key)
    # the ddpm chain's keys (test_gpu_sampler's restatement of ebm_utils.py:329, 342, 360), by t
    rkey = np.array(key, np.uint32)
    for t in range(T - 1, -1, -1):
        rkey, _ = tf.split(rkey, 2)
        rkey, infill_k = tf.split(rkey, 2)
        rkey, noise_k = tf.split(rkey, 2)
        np.testing.assert_array_equal(keys[t], np.concatenate([noise_k, infill_k]), err_msg=str(t))
    want = O.collection_slots(T)
    want[want >= 41] = -1
    np.testing.assert_array_equal(slots, want)
    # K < T: the same rules over K steps
    _, keys20, slots20 = _tables(BETAS, ebm_utils.ddim_schedule(T, 20), 0.0, key)
    ref = R.step_keys(key, 20)
    for i in range(20):
        np.testing.assert_array_equal(keys20[i], np.concatenate(ref[i]))
    want = O.collection_slots(20)
    want[want >= 41] = -1
    np.testing.assert_array_equal(slots20, want)


# ------------------------------------------------------------------------------------------------------- identity
@pytest.mark.parametrize("t", [999, 640, 200, 1, 0])
@pytest.mark.parametrize("infill", [False, True])
def test_full_schedule_eta_one_is_the_ancestral_step(t, infill):
    """K = T, eta = 1: sqrt(a') x0 + sqrt(1 - a' - sig^2) eps' = mu1 x0 + mu2 x for the clipped x0, so one DDIM step is
    the reference's reverse step for any network output."""
    g = np.random.default_rng(t)
    shape = (3, 32, 42)
    x = torch.from_numpy(g.standard_normal(shape) * 1.3)
    eps = torch.from_numpy(g.standard_normal(shape) * 2.0)       # arbitrary: many x0 entries clip
    z, iz = torch.from_numpy(g.standard_normal(shape)), torch.from_numpy(g.standard_normal(shape))
    ix = torch.from_numpy(g.uniform(-1, 1, shape))
    im = torch.from_numpy((g.uniform(size=shape) < 0.3).astype(np.float64))
    seen = []

    def apply_fn(a, cond):
        seen.append(float(cond.flatten()[0]))
        return eps

    tab = R.tables(BETAS, np.arange(1000), 1.0)
    kw = dict(infill_samples=ix, infill_masks=im, infill_z=iz) if infill else {}
    got, _, m = R.ddim_step(apply_fn, x, t, tab, z, **kw)
    infill_args = (ix, im, iz) if infill else ()
    # the oracle's ancestral step with its coefficients in float64 from the same float32 alpha_bar: equal to rounding
    ab = R.alpha_bar(BETAS).astype(np.float64)
    abp = np.concatenate([[1.0], ab[:-1]])
    alpha = ab / abp
    beta = 1 - alpha
    coef64 = dict(sqrt_recip_alpha_prod=np.sqrt(1 / ab), sqrt_alpha_prod_m1=np.sqrt(1 - ab) * np.sqrt(1 / ab),
                  mu1=beta * np.sqrt(abp) / (1 - ab), mu2=(1 - abp) * np.sqrt(alpha) / (1 - ab),
                  sigma=np.sqrt(beta * (1 - abp) / (1 - ab)), sqrt_alpha_prod=np.sqrt(ab),
                  sqrt_one_minus_alpha_prod=np.sqrt(1 - ab), alpha_prod=ab)
    ref, _, rm = O.reverse_step(apply_fn, x, t, coef64, z, *infill_args)
    err = float((got - ref).abs().max() / ref.abs().max())
    assert err < 1e-10, err
    np.testing.assert_allclose([float(v) for v in m], [float(v) for v in rm], rtol=1e-10)
    # and the float32 coefficients of smd_sampler_setup, which lose up to ~1e-2 to cancellation near t = 0
    ref32, _, _ = O.reverse_step(apply_fn, x, t, O.reverse_coefficients(BETAS), z, *infill_args)
    assert abs(seen[0] - seen[2]) < 1e-7 * seen[2]             # the same conditioning value sqrt(alpha_bar_t)
    err = float((got - ref32).abs().max() / ref32.abs().max())
    assert err < (2e-2 if t < 10 else 1e-5), err


# --------------------------------------------------------------------------------------------------- rejections
def _engine(arch="TransformerDDPM", **kw):
    cfg = dict(channels=42)
    if arch == "TransformerMDN":
        cfg.update(num_layers=1, num_mlp_layers=1)
    if arch == "DenseDDPM":
        cfg = dict(channels=512, num_layers=2)
    return Engine(ModelConfig(arch=arch, **cfg), **kw)


def test_rejections(lib):
    key = (ctypes.c_uint32 * 2)(0, 1)
    b = np.ascontiguousarray(O.create_noise_schedule(1e-4, 0.02, 10, "linear"), np.float32)
    eng = _engine(max_batch=4)
    good = np.arange(0, 10, 3, dtype=np.int32)
    bad = [
        (b, 1, np.asarray([0, 5], np.int32), 2, 0.0, "in \\[1, T\\]"),            # K > T
        (b, 10, np.asarray([5, 5], np.int32), 2, 0.0, "strictly increasing"),
        (b, 10, np.asarray([6, 2], np.int32), 2, 0.0, "strictly increasing"),
        (b, 10, np.asarray([-1, 2], np.int32), 2, 0.0, "strictly increasing"),
        (b, 10, np.asarray([2, 10], np.int32), 2, 0.0, "strictly increasing"),
        (b, 10, good, 4, -0.1, "eta"),
        (b, 10, good, 4, float("nan"), "eta"),
        (b, 10, good, 4, float("inf"), "eta"),
        (b, 10, good, 0, 0.0, "in \\[1, T\\]"),
        (b, 0, good, 1, 0.0, "T out of range"),
        (np.zeros(8193, np.float32) + 1e-3, 8193, good, 4, 0.0, "T out of range"),
        (np.zeros(10, np.float32), 10, good, 4, 0.0, "alpha_bar"),               # beta = 0: alpha_bar = 1
    ]
    for bb, T, s, K, eta, msg in bad:
        with pytest.raises(ValueError, match=msg):
            L.check(lib.smd_ddim_tables(_fp(bb), T, _ip(s), K, eta, key, None, None, None))
        with pytest.raises(ValueError, match=msg):
            L.check(lib.smd_ddim_setup(eng._plan, _fp(bb), T, _ip(s), K, eta, key, None))
    L.check(lib.smd_ddim_tables(_fp(b), 10, _ip(good), 4, 1.0, key, None, None, None))
    # valid arguments on a plan without a workspace: a call-order error
    with pytest.raises(L.SmdError, match="workspace not bound"):
        L.check(lib.smd_ddim_setup(eng._plan, _fp(b), 10, _ip(good), 4, 0.0, key, None))
    # more samples than the plan holds comes before the setup check
    with pytest.raises(ValueError, match="n out of range"):
        L.check(lib.smd_ddim_sample(eng._plan, None, None, 5, None, None, None, None, 1, None))
    with pytest.raises(ValueError, match="go together"):
        L.check(lib.smd_ddim_sample(eng._plan, None, None, 4, None, 1024, None, None, 1, None))
    with pytest.raises(L.SmdError, match="smd_ddim_setup has not been called"):
        L.check(lib.smd_ddim_sample(eng._plan, None, None, 4, None, None, None, None, 1, None))
    mdn = _engine("TransformerMDN", max_batch=4)
    with pytest.raises(ValueError, match="TransformerMDN"):
        L.check(lib.smd_ddim_setup(mdn._plan, _fp(b), 10, _ip(good), 4, 0.0, key, None))
    with pytest.raises(ValueError, match="TransformerMDN"):
        L.check(lib.smd_ddim_sample(mdn._plan, None, None, 4, None, None, None, None, 1, None))


def test_flags_and_dispatch():
    from absl import flags

    from smd_b200 import train_ncsn
    fl = flags.FLAGS
    assert "ddim" in fl["sampling"].parser.enum_values
    assert fl["ddim_steps"].default == 50 and fl["ddim_eta"].default == 0.0
    assert fl["ddim_schedule"].default == "uniform"
    if not fl.is_parsed():
        fl.mark_as_parsed()
    alg = train_ncsn.ddim_algorithm()
    assert alg.func is ebm_utils.ddim_dynamics
    assert alg.keywords == dict(steps=50, eta=0.0, schedule="uniform")
