"""Float64 restatement of the DDIM encoder (smd_ddim_encode_setup / smd_ddim_encode, include/smd.h) for any network
callable apply_fn(x, cond) -> eps.

alpha_bar is the float32 cumulative product smd_sampler_setup forms (ddim_reference.alpha_bar); every later operation
is float64.  The levels are a_{-1} = 1 (the data) and a_i = alpha_bar(tau_i); step i = 0 .. K-1 goes from
a = a_{i-1} to a' = a_i:
  eps = model(x, sqrt(a)),  x0 = sqrt(1/a) x - sqrt(1-a) sqrt(1/a) eps  (not clipped),  x <- sqrt(a') x0 + sqrt(1-a') eps."""
from __future__ import annotations

import numpy as np
import torch

from tests.ddim_reference import alpha_bar


def tables(betas, steps):
    """Per-step float64 scalars of the K steps, indexed by i, in the column order of smd_ddim_encode_tables."""
    ab = alpha_bar(betas).astype(np.float64)
    a_next = ab[np.asarray(steps, np.int64)]
    a = np.concatenate([[1.0], a_next[:-1]])
    return dict(a=a, a_next=a_next, sqrt_recip=np.sqrt(1 / a), sqrt_m1=np.sqrt(1 - a) * np.sqrt(1 / a),
                c_x0=np.sqrt(a_next), c_eps=np.sqrt(1 - a_next), sqrt_a=np.sqrt(a))


COLUMNS = ("sqrt_recip", "sqrt_m1", "c_x0", "c_eps", "sqrt_a")


def encode_step(apply_fn, x, i, tab):
    """One encoder step at index i (float64)."""
    dt = torch.float64
    c = {k: float(v[i]) for k, v in tab.items()}
    cond = torch.full((x.shape[0],) + (1,) * (x.dim() - 1), c["sqrt_a"], dtype=dt)
    eps = apply_fn(x, cond).to(dt)
    x0 = c["sqrt_recip"] * x - c["sqrt_m1"] * eps
    return c["c_x0"] * x0 + c["c_eps"] * eps


def encode_chain(apply_fn, betas, steps, x0):
    """The whole encoder from the data x0: returns the codes (float64)."""
    tab = tables(betas, steps)
    x = x0.to(torch.float64)
    for i in range(len(steps)):
        x = encode_step(apply_fn, x, i, tab)
    return x
