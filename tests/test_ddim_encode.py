"""The DDIM encoder's host side on the CPU: the coefficient table smd_ddim_encode_setup uploads against the float64
restatement, its mirror relation with the DDIM chain's table, the rejections of the new entry points, ebm_utils.slerp,
and the argument errors of sample_ncsn --interpolate_encoder."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import ddpm_oracle as O
from smd_b200 import Engine, ModelConfig, ebm_utils
from smd_b200 import lib as L
from tests import ddim_encode_reference as RE
from tests import ddim_reference as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BETAS = O.create_noise_schedule(1e-6, 0.01, 1000, "linear")


def _fp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))


def _ip(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_int))


def encode_table(betas, steps):
    lib = L.load_library()
    b = np.ascontiguousarray(betas, np.float32)
    s = np.ascontiguousarray(steps, np.int32)
    coef = np.full((len(s), 8), np.nan, np.float32)
    L.check(lib.smd_ddim_encode_tables(_fp(b), len(b), _ip(s), len(s), _fp(coef)))
    return coef


# --------------------------------------------------------------------------------------------------------- tables
@pytest.mark.parametrize("steps", [np.arange(1000), ebm_utils.ddim_schedule(1000, 50),
                                   ebm_utils.ddim_schedule(1000, 20, "quadratic"), [999], [0], [3, 17, 500, 501]])
def test_coefficient_table_matches_float64(lib, steps):
    coef = encode_table(BETAS, steps)
    tab = RE.tables(BETAS, steps)
    for j, name in enumerate(RE.COLUMNS):
        np.testing.assert_allclose(coef[:, j], tab[name], rtol=1e-6, atol=1e-12, err_msg=name)
        # rounded once from float64
        np.testing.assert_array_equal(coef[:, j], tab[name].astype(np.float32), err_msg=name)
    assert (coef[:, 5:] == 0).all()
    # the first step starts at the data, a = 1: x0 = 1 x - 0 eps, conditioned on sqrt(1) = 1
    assert coef[0, 0] == 1 and coef[0, 1] == 0 and coef[0, 4] == 1
    ab = R.alpha_bar(BETAS).astype(np.float64)[np.asarray(steps)]
    assert coef[0, 2] == np.float32(np.sqrt(ab[0])) and coef[0, 3] == np.float32(np.sqrt(1 - ab[0]))


@pytest.mark.parametrize("steps", [ebm_utils.ddim_schedule(1000, 50), [999], [3, 17, 500, 501]])
def test_table_mirrors_the_ddim_chain(lib, steps):
    """Encoder step i runs the DDIM chain's step i backwards: it lands on the level the chain's step i starts from,
    and it leaves the level the chain's step i-1 starts from."""
    K = len(steps)
    b = np.ascontiguousarray(BETAS, np.float32)
    s = np.ascontiguousarray(steps, np.int32)
    dec = np.zeros((K, 8), np.float32)
    L.check(L.load_library().smd_ddim_tables(_fp(b), len(b), _ip(s), K, 0.0, None, _fp(dec), None, None))
    enc = encode_table(BETAS, steps)
    np.testing.assert_array_equal(enc[:, 2], dec[:, 5])          # sqrt(a_i)
    np.testing.assert_array_equal(enc[:, 3], dec[:, 6])          # sqrt(1 - a_i)
    np.testing.assert_array_equal(enc[1:, 0], dec[:-1, 0])       # sqrt(1 / a_{i-1})
    np.testing.assert_array_equal(enc[1:, 1], dec[:-1, 1])
    np.testing.assert_array_equal(enc[1:, 4], dec[:-1, 5])       # the conditioning value sqrt(a_{i-1})


def test_constant_network_round_trip_in_float64():
    """With eps = c the encoder's code is sqrt(a_{K-1}) x0 + sqrt(1 - a_{K-1}) c, and the DDIM chain at eta = 0 on it
    returns x0 (the restatements, in float64)."""
    g = np.random.default_rng(4)
    x0 = torch.from_numpy(g.uniform(-0.9, 0.9, (3, 32, 6)))
    c = torch.from_numpy(g.uniform(-0.5, 0.5, (6,)))
    apply_fn = lambda x, cond: c.expand_as(x)                 # noqa: E731
    steps = ebm_utils.ddim_schedule(1000, 10)
    code = RE.encode_chain(apply_fn, BETAS, steps, x0)
    a = float(R.alpha_bar(BETAS)[steps[-1]])
    want = np.sqrt(a) * x0 + np.sqrt(1 - a) * c
    assert float((code - want).abs().max()) < 1e-12
    back, _, _ = R.ddim_chain(apply_fn, BETAS, steps, 0.0, code, (0, 1))
    assert float((back - x0).abs().max()) < 1e-12


# --------------------------------------------------------------------------------------------------- rejections
def _engine(arch="TransformerDDPM", **kw):
    cfg = dict(channels=42)
    if arch == "TransformerMDN":
        cfg.update(num_layers=1, num_mlp_layers=1)
    return Engine(ModelConfig(arch=arch, **cfg), **kw)


def test_rejections(lib):
    b = np.ascontiguousarray(O.create_noise_schedule(1e-4, 0.02, 10, "linear"), np.float32)
    eng = _engine(max_batch=4)
    good = np.arange(0, 10, 3, dtype=np.int32)
    bad = [
        (b, 1, np.asarray([0, 5], np.int32), 2, "in \\[1, T\\]"),            # K > T
        (b, 10, np.asarray([5, 5], np.int32), 2, "strictly increasing"),
        (b, 10, np.asarray([6, 2], np.int32), 2, "strictly increasing"),
        (b, 10, np.asarray([-1, 2], np.int32), 2, "strictly increasing"),
        (b, 10, np.asarray([2, 10], np.int32), 2, "strictly increasing"),
        (b, 10, good, 0, "in \\[1, T\\]"),
        (b, 0, good, 1, "T out of range"),
        (np.zeros(8193, np.float32) + 1e-3, 8193, good, 4, "T out of range"),
        (np.zeros(10, np.float32), 10, good, 4, "alpha_bar"),               # beta = 0: alpha_bar = 1
    ]
    for bb, T, s, K, msg in bad:
        with pytest.raises(ValueError, match=msg):
            L.check(lib.smd_ddim_encode_tables(_fp(bb), T, _ip(s), K, None))
        with pytest.raises(ValueError, match=msg):
            L.check(lib.smd_ddim_encode_setup(eng._plan, _fp(bb), T, _ip(s), K, None))
    with pytest.raises(ValueError, match="null betas"):
        L.check(lib.smd_ddim_encode_tables(None, 10, _ip(good), 4, None))
    L.check(lib.smd_ddim_encode_tables(_fp(b), 10, _ip(good), 4, None))
    # valid arguments on a plan without a workspace: a call-order error
    with pytest.raises(L.SmdError, match="workspace not bound"):
        L.check(lib.smd_ddim_encode_setup(eng._plan, _fp(b), 10, _ip(good), 4, None))
    for n in (0, 5):
        with pytest.raises(ValueError, match="n out of range"):
            L.check(lib.smd_ddim_encode(eng._plan, None, None, n, 1, None))
    with pytest.raises(L.SmdError, match="smd_ddim_encode_setup has not been called"):
        L.check(lib.smd_ddim_encode(eng._plan, None, None, 4, 1, None))
    mdn = _engine("TransformerMDN", max_batch=4)
    with pytest.raises(ValueError, match="TransformerMDN"):
        L.check(lib.smd_ddim_encode_setup(mdn._plan, _fp(b), 10, _ip(good), 4, None))
    with pytest.raises(ValueError, match="TransformerMDN"):
        L.check(lib.smd_ddim_encode(mdn._plan, None, None, 4, 1, None))


# -------------------------------------------------------------------------------------------------------- slerp
def test_slerp_endpoints_are_exact():
    g = np.random.default_rng(1)
    z0 = torch.from_numpy(g.standard_normal((5, 32, 42)).astype(np.float32))
    z1 = torch.from_numpy(g.standard_normal((5, 32, 42)).astype(np.float32))
    a = ebm_utils.slerp(z0, z1, 0.0)
    b = ebm_utils.slerp(z0, z1, 1.0)
    assert a.dtype == torch.float64 and a.shape == z0.shape
    assert torch.equal(a.float(), z0) and torch.equal(b.float(), z1)
    # numpy endpoints too, and the 9 points sample_ncsn decodes
    pts = [ebm_utils.slerp(z0.numpy(), z1.numpy(), al) for al in np.linspace(0.0, 1.0, 9)]
    assert torch.equal(pts[0].float(), z0) and torch.equal(pts[-1].float(), z1)


def test_slerp_matches_the_closed_form_and_keeps_the_norm():
    g = np.random.default_rng(2)
    z0 = g.standard_normal((6, 300))
    z1 = g.standard_normal((6, 300))
    z1 *= np.linalg.norm(z0, axis=1, keepdims=True) / np.linalg.norm(z1, axis=1, keepdims=True)
    theta = np.arccos(np.sum(z0 * z1, 1) / (np.linalg.norm(z0, axis=1) * np.linalg.norm(z1, axis=1)))
    for alpha in (0.1, 0.5, 0.77):
        got = ebm_utils.slerp(z0, z1, alpha).numpy()
        want = (np.sin((1 - alpha) * theta)[:, None] * z0 + np.sin(alpha * theta)[:, None] * z1) / np.sin(theta)[:, None]
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(np.linalg.norm(got, axis=1), np.linalg.norm(z0, axis=1), rtol=1e-12)
    # a linear mix of the same rows shrinks (near-orthogonal Gaussian rows: about 0.71 of the norm at alpha = 0.5)
    lin = np.linalg.norm(0.5 * z0 + 0.5 * z1, axis=1) / np.linalg.norm(z0, axis=1)
    assert (lin < 0.8).all()


def test_slerp_falls_back_to_linear_for_tiny_angles():
    g = np.random.default_rng(3)
    z0 = g.standard_normal((4, 50))
    z1 = z0.copy()
    z1[0] *= 1.5                                # angle 0, different norm
    z1[1] += 1e-9 * g.standard_normal(50)       # angle far below 1e-6
    z1[2] = 0.0                                 # a zero row has no angle
    z1[3] = g.standard_normal(50)               # a proper angle, slerp
    for alpha in (0.25, 0.5):
        got = ebm_utils.slerp(z0, z1, alpha).numpy()
        assert np.isfinite(got).all()
        np.testing.assert_allclose(got[:3], (1 - alpha) * z0[:3] + alpha * z1[:3], rtol=1e-12, atol=1e-15)
        th = np.arccos(z0[3] @ z1[3] / (np.linalg.norm(z0[3]) * np.linalg.norm(z1[3])))
        want = (np.sin((1 - alpha) * th) * z0[3] + np.sin(alpha * th) * z1[3]) / np.sin(th)
        np.testing.assert_allclose(got[3], want, rtol=1e-12, atol=1e-12)
    with pytest.raises(ValueError, match="equally shaped"):
        ebm_utils.slerp(z0, z1[:2], 0.5)


# ------------------------------------------------------------------------------------------------- command line
@pytest.mark.parametrize("extra,msg", [
    ([], "--interpolate_encoder=ddim needs --interpolate"),
    (["--interpolate"], "--interpolate_encoder=ddim needs --sampling=ddim"),
    (["--interpolate", "--sampling=ddpm"], "--interpolate_encoder=ddim needs --sampling=ddim"),
    (["--interpolate", "--sampling=ddim", "--ddim_eta=0.5"], "--interpolate_encoder=ddim needs --ddim_eta=0"),
])
def test_interpolate_encoder_flag_errors(tmp_path, extra, msg):
    r = subprocess.run([sys.executable, "-m", "smd_b200.sample_ncsn", "--interpolate_encoder=ddim", *extra,
                        f"--model_dir={tmp_path}"], capture_output=True, text=True, timeout=300, cwd=ROOT,
                       env=dict(os.environ, PYTHONPATH=ROOT))
    assert r.returncode != 0 and f"ValueError: {msg}" in r.stderr, r.stderr[-2000:]
    assert not os.listdir(tmp_path)


def test_reconstruction_errors():
    from smd_b200 import sample_ncsn
    g = np.random.default_rng(5)
    starts = g.uniform(-1, 1, (4, 3, 2)).astype(np.float32)
    goals = np.roll(starts, 1, axis=0)
    gen = np.stack([starts + 0.1] + [starts] * 7 + [goals - 0.2 * (np.arange(2) == 1)]).astype(np.float32)
    r = sample_ncsn.reconstruction_errors(gen, starts, goals)
    assert r["start_mse"] == pytest.approx(0.01, rel=1e-5) and r["start_max_abs"] == pytest.approx(0.1, rel=1e-5)
    assert r["goal_mse"] == pytest.approx(0.02, rel=1e-5) and r["goal_max_abs"] == pytest.approx(0.2, rel=1e-5)
