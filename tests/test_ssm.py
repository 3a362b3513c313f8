"""Sliced score matching on the CPU: the Rademacher draw, the fp64 restatement of the objective (reverse over reverse,
as the reference) against a forward-mode restatement and finite differences, and the plan-level contract of the new
entry points (DenseNCSN only, other architectures' workspaces untouched)."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import ddpm_oracle as O
from oracle import threefry as tf
from tests import ssm_reference as R

KW = dict(num_layers=2, mlp_dims=16)
C = 8


@pytest.mark.parametrize("seed,shape", [(0, (4, 8)), (7, (3, 5)), (123, (64, 512)), (2 ** 33 + 5, (17,))])
def test_rademacher_is_the_sign_of_uniform_below_half(seed, shape):
    key = tf.prng_key(seed)
    v = R.rademacher(key, shape)
    assert v.shape == shape and v.dtype == np.float32
    assert set(np.unique(v).tolist()) <= {-1.0, 1.0}
    np.testing.assert_array_equal(v == 1.0, tf.uniform01(key, shape) < 0.5)


def _setup(seed=0, B=4):
    p = {k: v.requires_grad_(True) for k, v in R.dense_ncsn_params(C, KW["mlp_dims"], KW["num_layers"], seed).items()}
    g = torch.Generator().manual_seed(seed + 1)
    x0 = torch.rand(B, C, generator=g, dtype=torch.float64) * 2 - 1
    eps = torch.randn(B, C, generator=g, dtype=torch.float64)
    v = torch.where(torch.rand(B, C, generator=g) < 0.5, 1.0, -1.0).double()
    sig = torch.tensor([0.05, 0.3, 1.0, 0.7][:B], dtype=torch.float64)
    return p, x0, eps, v, sig


def test_reverse_over_reverse_equals_reverse_over_forward_fp64():
    p, x0, eps, v, sig = _setup()
    model = lambda a, s: O.dense_ncsn(p, a, s, **KW)
    per, _, _ = R.ssm_loss_tensors(model, x0, sig, eps, v, "none")
    g_rr = torch.autograd.grad(per.mean(), list(p.values()))
    # restatement: the Hessian term as a forward-mode JVP along v, then reverse mode for the parameters
    us = sig.reshape(-1, 1)
    x = x0 + eps * us
    s, s_dot = torch.func.jvp(lambda a: model(a, us), (x,), (v,))
    per2 = (0.5 * (s ** 2).sum(-1) + (v * s_dot).sum(-1)) * sig ** 2
    g_rf = torch.autograd.grad(per2.mean(), list(p.values()))
    assert float(((per - per2).abs().max() / per2.abs().max()).detach()) <= 1e-10
    for name, a, b in zip(p, g_rr, g_rf):
        assert float((a - b).norm() / (b.norm() + 1e-300)) <= 1e-10, name


def test_hessian_term_matches_central_difference():
    p, x0, eps, v, sig = _setup(seed=3)
    model = lambda a, s: O.dense_ncsn(p, a, s, **KW)
    per, score_loss, hess = R.ssm_loss_tensors(model, x0, sig, eps, v, "none")
    us = sig.reshape(-1, 1)
    x = (x0 + eps * us).detach()
    h = 1e-5
    with torch.no_grad():
        fd = ((model(x + h * v, us) * v).sum(-1) - (model(x - h * v, us) * v).sum(-1)) / (2 * h)
    torch.testing.assert_close(hess.detach(), fd, rtol=1e-6, atol=1e-8)
    with torch.no_grad():
        torch.testing.assert_close(score_loss, 0.5 * (model(x, us) ** 2).sum(-1))


def _engine(arch, **kw):
    from smd_b200 import Engine, ModelConfig
    cfg = dict(channels=512, mlp_dims=2048, num_layers=3) if arch != "TransformerDDPM" else dict(channels=42)
    return Engine(ModelConfig(arch=arch, **cfg), **kw)


@pytest.mark.parametrize("training,precision", [(False, "bf16"), (True, "bf16"), (False, "bf16x3")])
def test_dense_ncsn_plans_build_with_tangent_regions(lib, training, precision):
    eng = _engine("DenseNCSN", max_batch=128, training=training, precision=precision)
    ddpm = _engine("DenseDDPM", max_batch=128, training=training, precision=precision)
    # same parameters and primal regions; the tangent regions come on top
    assert eng.layout == ddpm.layout and eng.workspace_bytes > ddpm.workspace_bytes


# smd_workspace_bytes of the architectures without a tangent pass, recorded at the commit before sliced score matching
PARENT_WORKSPACE_BYTES = {
    ("TransformerDDPM", 8, False, "bf16"): 95706112,
    ("TransformerDDPM", 128, True, "bf16"): 868057088,
    ("TransformerDDPM", 8, False, "bf16x3"): 197703680,
    ("DenseDDPM", 128, False, "bf16"): 137525248,
    ("DenseDDPM", 128, True, "bf16"): 119809024,
    ("DenseDDPM", 128, False, "bf16x3"): 281341952,
}


def test_other_architectures_keep_their_workspace_size(lib):
    for (arch, mb, training, precision), want in PARENT_WORKSPACE_BYTES.items():
        assert _engine(arch, max_batch=mb, training=training, precision=precision).workspace_bytes == want


@pytest.mark.parametrize("arch", ["TransformerDDPM", "DenseDDPM"])
def test_ssm_entry_points_reject_other_architectures(lib, arch):
    from smd_b200 import lib as L
    eng = _engine(arch, max_batch=4)
    key = (ctypes.c_uint32 * 2)(0, 0)
    with pytest.raises(ValueError, match="DENSE_NCSN"):
        L.check(lib.smd_ssm_draws(eng._plan, key, 4, 0, 4, 0, None, None, None, None, None))
    with pytest.raises(ValueError, match="DENSE_NCSN"):
        L.check(lib.smd_ssm_loss(eng._plan, None, None, None, None, None, 4, None, None, None, None))
    with pytest.raises(ValueError, match="DENSE_NCSN"):
        L.check(lib.smd_ssm_grads(eng._plan, None, None, None, None, None, 4, 4, None, None, None))
