"""Float64 restatement of the DPM-Solver++ multistep chain (smd_dpm_setup / smd_dpm_sample, include/smd.h; Lu et al.
2022, Algorithm 2 and its third-order form) for any network callable apply_fn(x, cond) -> eps.

The levels are the DDIM chain's: a_i = alpha_bar(tau_i) (the float32 cumulative product, tests/ddim_reference.py) for
i = K-1 .. 0 and a_{-1} = 1, with alpha = sqrt(a), sigma = sqrt(1-a), lambda = log(alpha / sigma).  Step i goes from
level i to level i-1 with the data estimate m0 = clip(sqrt(1/a) x - sqrt(1-a) sqrt(1/a) eps, -1, 1) and those of the
two steps before, m1 and m2.  `update` states the solver as the paper writes it; `tables` reads the per-step
coefficients (c_x, c_0, c_1, c_2) off it, as its responses to unit inputs, which makes them independent of the
library's gathered closed forms."""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle import ddpm_oracle as O
from oracle import threefry as tf
from tests import ddim_reference as D


def levels(betas, steps):
    """The float64 alpha_bar of the K selected indices (from the float32 product), indexed by i."""
    return D.alpha_bar(betas).astype(np.float64)[np.asarray(steps, np.int64)]


def step_order(i, K, order):
    """The order of step i: min(order, j + 1) for the step j = K-1-i from the noisiest, and 1 at the last step."""
    return 1 if i == 0 else min(int(order), K - i)


def update(x, m0, m1, m2, a, i, order):
    """The step from level i to level i-1 of the given order on the levels a (a[i] = alpha_bar(tau_i)), as the paper
    writes it.  x, m0, m1, m2 may be scalars or tensors (m1 / m2 unused below order 2 / 3)."""
    if i == 0:
        return m0                                       # into a = 1: sigma = 0, alpha = 1
    lam = lambda k: math.log(math.sqrt(a[k]) / math.sqrt(1.0 - a[k]))  # noqa: E731
    alpha_t, sigma_t, sigma_s = math.sqrt(a[i - 1]), math.sqrt(1.0 - a[i - 1]), math.sqrt(1.0 - a[i])
    h = lam(i - 1) - lam(i)
    if order == 1:
        return sigma_t / sigma_s * x + alpha_t * (1.0 - math.exp(-h)) * m0
    r0 = (lam(i) - lam(i + 1)) / h
    if order == 2:
        d = (1.0 + 1.0 / (2.0 * r0)) * m0 - 1.0 / (2.0 * r0) * m1
        return sigma_t / sigma_s * x + alpha_t * (1.0 - math.exp(-h)) * d
    r1 = (lam(i + 1) - lam(i + 2)) / h
    phi1 = math.expm1(-h)
    phi2 = phi1 / h + 1.0
    phi3 = phi2 / h - 0.5
    d1_0 = (m0 - m1) / r0
    d1_1 = (m1 - m2) / r1
    d1 = d1_0 + r0 / (r0 + r1) * (d1_0 - d1_1)
    d2 = (d1_0 - d1_1) / (r0 + r1)
    return sigma_t / sigma_s * x - alpha_t * phi1 * m0 + alpha_t * phi2 * d1 - alpha_t * phi3 * d2


def tables(betas, steps, order):
    """Per-step float64 scalars of the chain, indexed by i: the coefficients of x, m0, m1, m2 (the update's
    responses to unit inputs) and the x0-estimate and conditioning values."""
    a = levels(betas, steps)
    K = len(a)
    c = np.zeros((K, 4))
    for i in range(K):
        o = step_order(i, K, order)
        for j in range(4):
            e = [0.0] * 4
            e[j] = 1.0
            c[i, j] = update(*e, a, i, o)
    return dict(t=np.asarray(steps, np.int64), a=a, c_x=c[:, 0], c_0=c[:, 1], c_1=c[:, 2], c_2=c[:, 3],
                sqrt_recip=np.sqrt(1 / a), sqrt_m1=np.sqrt(1 - a) * np.sqrt(1 / a), sqrt_a=np.sqrt(a),
                sqrt_1m=np.sqrt(1 - a))


def library_tables(coef):
    """The dict of `tables` from the (K, 8) float32 table smd_dpm_tables returns, in float64."""
    c = np.asarray(coef, np.float64)
    return dict(a=c[:, 7], c_x=c[:, 2], c_0=c[:, 3], c_1=c[:, 4], c_2=c[:, 6], sqrt_recip=c[:, 0], sqrt_m1=c[:, 1],
                sqrt_a=c[:, 5], sqrt_1m=np.sqrt(1 - c[:, 7]))


def _nrm(a):   # utils/ebm_utils.py:381-383: sqrt(sum(a^2, axis=1) + 1e-10).mean()
    return torch.sqrt((a * a).sum(dim=1) + 1e-10).mean()


def dpm_chain(apply_fn, betas, steps, order, init, key, infill_samples=None, infill_masks=None, tab=None, clip=True,
              stop_before_last=False):
    """The whole chain from `init` (float64) with the coefficients `tab` (default: tables(betas, steps, order)).
    clip=False drops the clipping of the x0 estimate; stop_before_last returns the state at level tau_0, before the
    final step.  Returns state, collection (41, *init.shape), metrics (4, K)."""
    dt = torch.float64
    tau = np.asarray(steps, np.int64)
    K = len(tau)
    tab = tables(betas, steps, order) if tab is None else tab
    keys = D.step_keys(key, K)
    slots = O.collection_slots(K)
    x = init.to(dt)
    infill = infill_masks is not None
    if infill:
        infill_samples, infill_masks = infill_samples.to(dt), infill_masks.to(dt)
    collection = torch.zeros((41,) + tuple(init.shape), dtype=dt)
    collection[0] = x * (1 - infill_masks) + infill_samples * infill_masks if infill else x
    mets = torch.zeros((4, K), dtype=dt)
    shape = tuple(init.shape)
    hist = []                                           # data estimates of the steps before, newest first
    for j, i in enumerate(range(K - 1, -1, -1)):
        if stop_before_last and i == 0:
            break
        c = {k: float(v[i]) for k, v in tab.items()}
        cond = torch.full((x.shape[0],) + (1,) * (x.dim() - 1), c["sqrt_a"], dtype=dt)
        eps = apply_fn(x, cond).to(dt)
        m0 = c["sqrt_recip"] * x - c["sqrt_m1"] * eps
        if clip:
            m0 = torch.clamp(m0, -1.0, 1.0)
        nxt = c["c_x"] * x + c["c_0"] * m0
        if c["c_1"] != 0:
            nxt = nxt + c["c_1"] * hist[0]
        if c["c_2"] != 0:
            nxt = nxt + c["c_2"] * hist[1]
        hist = [m0] + hist[:1]
        if infill:
            if tau[i] > 0:
                iz = torch.from_numpy(tf.normal(keys[i][1], shape).astype(np.float64))
                y = c["sqrt_a"] * infill_samples + c["sqrt_1m"] * iz
            else:
                y = infill_samples
            nxt = nxt * (1 - infill_masks) + y * infill_masks
        for r, v in enumerate((_nrm(eps), _nrm(x - nxt), c["a"], _nrm(torch.zeros_like(x)))):
            mets[r, j] = v
        x = nxt
        if 0 <= slots[i] < 41:
            collection[slots[i]] = x
    return x, collection, mets
