"""Float64 restatement of the DDIM chain (smd_ddim_setup / smd_ddim_sample, include/smd.h) for any network callable
apply_fn(x, cond) -> eps, with the noise drawn by the numpy threefry restatement (oracle/threefry.py).

alpha_bar is the float32 cumulative product smd_sampler_setup forms; every later operation is float64.  Step i of the
chain (i = K-1 .. 0) sits at t = tau_i with a = alpha_bar(tau_i), a' = alpha_bar(tau_{i-1}) (1 at i = 0):
  eps = model(x, sqrt(a)),  x0 = clip(sqrt(1/a) x - sqrt(1-a) sqrt(1/a) eps, -1, 1),  eps' = (x - sqrt(a) x0) / sqrt(1-a),
  sig = eta sqrt((1-a')/(1-a)) sqrt(1 - a/a'),  x <- sqrt(a') x0 + sqrt(max(1-a'-sig^2, 0)) eps' + sig z,
then the infill blend of diffusion_dynamics at t = tau_i."""
from __future__ import annotations

import numpy as np
import torch

from oracle import ddpm_oracle as O
from oracle import threefry as tf


def alpha_bar(betas):
    """cumprod(1 - betas) in float32, sequentially, as smd_sampler_setup."""
    return np.cumprod((np.float32(1) - np.asarray(betas, np.float32)).astype(np.float32), dtype=np.float32)


def tables(betas, steps, eta):
    """Per-step float64 scalars of the K selected levels, indexed by i."""
    ab = alpha_bar(betas).astype(np.float64)
    steps = np.asarray(steps, np.int64)
    a = ab[steps]
    ap = np.concatenate([[1.0], a[:-1]])
    sig = float(eta) * np.sqrt((1 - ap) / (1 - a)) * np.sqrt(np.maximum(1 - a / ap, 0.0))
    return dict(t=steps, a=a, a_prev=ap, sig=sig, sqrt_recip=np.sqrt(1 / a), sqrt_m1=np.sqrt(1 - a) * np.sqrt(1 / a),
                c_x0=np.sqrt(ap), c_dir=np.sqrt(np.maximum(1 - ap - sig * sig, 0.0)), sqrt_a=np.sqrt(a),
                sqrt_1m=np.sqrt(1 - a))


def step_keys(key, K):
    """(noise key, infill key) of step i: diffusion_dynamics' scan carry over K steps, consumed for i = K-1 .. 0."""
    rng = np.asarray(key, np.uint32)
    out = [None] * K
    for i in range(K - 1, -1, -1):
        rng, _ = tf.split(rng, 2)
        rng, infill = tf.split(rng, 2)
        rng, noise = tf.split(rng, 2)
        out[i] = (noise, infill)
    return out


def _nrm(a):   # utils/ebm_utils.py:381-383: sqrt(sum(a^2, axis=1) + 1e-10).mean()
    return torch.sqrt((a * a).sum(dim=1) + 1e-10).mean()


def ddim_step(apply_fn, x, i, tab, z, infill_samples=None, infill_masks=None, infill_z=None):
    """One step at index i with supplied noise z (and infill noise); returns next, eps, (grad, step, alpha_bar, noise)."""
    dt = torch.float64
    c = {k: float(v[i]) for k, v in tab.items()}
    cond = torch.full((x.shape[0],) + (1,) * (x.dim() - 1), c["sqrt_a"], dtype=dt)
    eps = apply_fn(x, cond).to(dt)
    x0 = torch.clamp(c["sqrt_recip"] * x - c["sqrt_m1"] * eps, -1.0, 1.0)
    direction = (x - c["sqrt_a"] * x0) / c["sqrt_1m"]
    noise = c["sig"] * z if c["sig"] != 0 else torch.zeros_like(x)
    nxt = c["c_x0"] * x0 + c["c_dir"] * direction + noise
    if infill_masks is not None:
        y = c["sqrt_a"] * infill_samples + c["sqrt_1m"] * infill_z if c["t"] > 0 else infill_samples
        nxt = nxt * (1 - infill_masks) + y * infill_masks
    return nxt, eps, (_nrm(eps), _nrm(x - nxt), c["a"], _nrm(noise))


def ddim_chain(apply_fn, betas, steps, eta, init, key, infill_samples=None, infill_masks=None):
    """The whole chain from `init` (float64).  Returns state, collection (41, *init.shape), metrics (4, K)."""
    dt = torch.float64
    K = len(steps)
    tab = tables(betas, steps, eta)
    keys = step_keys(key, K)
    slots = O.collection_slots(K)
    x = init.to(dt)
    infill = infill_masks is not None
    if infill:
        infill_samples, infill_masks = infill_samples.to(dt), infill_masks.to(dt)
    collection = torch.zeros((41,) + tuple(init.shape), dtype=dt)
    collection[0] = x * (1 - infill_masks) + infill_samples * infill_masks if infill else x
    mets = torch.zeros((4, K), dtype=dt)
    shape = tuple(init.shape)
    for j, i in enumerate(range(K - 1, -1, -1)):
        nk, ik = keys[i]
        z = torch.from_numpy(tf.normal(nk, shape).astype(np.float64)) if tab["sig"][i] != 0 else None
        iz = torch.from_numpy(tf.normal(ik, shape).astype(np.float64)) if infill and tab["t"][i] > 0 else None
        x, _, m = ddim_step(apply_fn, x, i, tab, z, infill_samples if infill else None,
                            infill_masks if infill else None, iz)
        for r in range(4):
            mets[r, j] = m[r]
        if 0 <= slots[i] < 41:
            collection[slots[i]] = x
    return x, collection, mets
