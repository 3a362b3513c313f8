"""Objectives with the reference signatures (utils/losses.py): the DDPM objective (the hot path) and denoising / sliced
score matching for the NCSN family (SURVEY 8(f4))."""
from __future__ import annotations

import numpy as np
import torch


def reduce_fn(x, mode):
    """utils/losses.py:22-30."""
    if mode == "none" or mode is None:
        return x
    if mode == "sum":
        return x.sum()
    if mode == "mean":
        return x.mean()
    raise ValueError("Unsupported reduction option.")


def diffusion_loss(batch, model, betas, rng, continuous_noise=False, reduction="mean"):
    """utils/losses.py:250-308: draws (labels, alpha-bar, eps) from `rng` on device with jax threefry semantics,
    forms x_t, evaluates the network and reduces the per-example mean-squared error.  `model` is an nn.Model."""
    from .nn import _as_device_f32
    x0 = _as_device_f32(batch)
    eng = model.engine(x0.shape[0])
    betas = np.asarray(betas, np.float32)
    if getattr(eng, "_obj_betas", None) is None or not np.array_equal(eng._obj_betas, betas):
        eng.objective_setup(betas)
        eng._obj_betas = betas.copy()
    # continuous_noise only changes the label range (losses.py:272-275: minval = int(continuous_noise)); the discrete
    # branch is commented out upstream (losses.py:287-288, 301-302), so label 0 reads alphas_prod[-1] (wraps) as there
    used, eps = eng.draws((int(rng[0]), int(rng[1])), x0.shape[0], continuous_noise=bool(continuous_noise))
    loss = eng.ddpm_loss(x0, used, eps)
    return reduce_fn(loss, reduction)


def denoising_score_matching_loss(batch, model, sigmas, rng, continuous_noise=False, reduction="mean"):
    """utils/losses.py:129-179: sigma labels / noise from `rng` (jax threefry semantics, on device), x~ = x + sigma eps,
    scores = model(x~, sigma), 0.5 * sum((scores + eps / sigma)^2) * sigma^2 per example.  `model` must be a score
    network (ncsn.DenseNCSN)."""
    from .nn import _as_device_f32
    x0 = _as_device_f32(batch)
    eng = model.engine(x0.shape[0])
    sig = np.asarray(sigmas, np.float32)
    if getattr(eng, "_dsm_sigmas", None) is None or not np.array_equal(eng._dsm_sigmas, sig):
        eng.dsm_setup(sig)
        eng._dsm_sigmas = sig.copy()
    used, eps = eng.dsm_draws((int(rng[0]), int(rng[1])), x0.shape[0], continuous_noise=bool(continuous_noise))
    return reduce_fn(eng.dsm_loss(x0, used, eps), reduction)


def _score_engine(batch, model, sigmas):
    from .nn import _as_device_f32
    x0 = _as_device_f32(batch)
    eng = model.engine(x0.shape[0])
    sig = np.asarray(sigmas, np.float32)
    if getattr(eng, "_dsm_sigmas", None) is None or not np.array_equal(eng._dsm_sigmas, sig):
        eng.dsm_setup(sig)
        eng._dsm_sigmas = sig.copy()
    return x0, eng


def sliced_score_matching_loss(batch, model, sigmas, rng, continuous_noise=False, reduction="mean"):
    """utils/losses.py:182-247 (one particle): sigma labels, noise and Rademacher vectors v from `rng` (jax threefry
    semantics, on device), x~ = x + sigma eps, s = model(x~, sigma), (0.5 |s|^2 + v.J_s v) sigma^2 per example.  The
    Hessian term v.J_s v is a Jacobian-vector product through the network.  `model` must be ncsn.DenseNCSN."""
    x0, eng = _score_engine(batch, model, sigmas)
    used, eps, v = eng.ssm_draws((int(rng[0]), int(rng[1])), x0.shape[0], continuous_noise=bool(continuous_noise))
    return reduce_fn(eng.ssm_loss(x0, used, eps, v), reduction)
