"""CPU restatement of sliced score matching (utils/losses.py:182-247), next to the oracle it builds on.

Test infrastructure only.  ``rademacher`` restates jax.random.rademacher as of jax 0.2.8 from memory of that version
(not checkable offline, the same status as SURVEY D8): ``2 * bernoulli(key, 0.5) - 1`` with ``bernoulli`` =
``uniform(key, shape, float32) < 0.5``.  With the uniform01 bit recipe (bits >> 9 as the mantissa) that is +1 exactly
when the threefry word is < 2^31.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import ddpm_oracle as O
from oracle import threefry as tf


def rademacher(key, shape) -> np.ndarray:
    bits = tf.random_bits(key, shape)
    return np.where(bits < np.uint32(1 << 31), 1.0, -1.0).astype(np.float32)


def ssm_draws(rng_key, batch_shape, sigmas, continuous_noise=False):
    """losses.py:203-223.  Returns labels, used_sigmas (B,), eps (unit normal), v (+-1)."""
    sig = np.asarray(sigmas, np.float32)
    rng, label_rng, sample_rng, score_rng = tf.split(rng_key, 4)
    B = batch_shape[0]
    labels = tf.randint(label_rng, (B,), int(continuous_noise), len(sig))
    if continuous_noise:
        rng, noise_rng = tf.split(rng, 2)
        used = O.uniform_minmax(tf.uniform01(noise_rng, (B,)), sig[labels - 1], sig[labels])
    else:
        used = sig[labels]
    eps = tf.normal(sample_rng, tuple(batch_shape))
    v = rademacher(score_rng, tuple(batch_shape))
    return labels, used.astype(np.float32), eps, v


def ssm_loss_tensors(apply_fn, batch, used, eps, v, reduction="mean"):
    """losses.py:224-247 given the draws, in the reference's order: first_grad = model(x~), then
    second_grad = grad_x sum(model(x~) * v) with create_graph, so .backward() gives reverse-over-reverse parameter
    gradients.  Returns (loss, score_loss (B,), hessian_loss (B,))."""
    B = batch.shape[0]
    us = used.reshape(B, *([1] * (batch.dim() - 1)))
    x = (batch + eps * us).detach().requires_grad_(True)
    first_grad = apply_fn(x, us)
    second_grad, = torch.autograd.grad((apply_fn(x, us) * v).sum(), x, create_graph=True)
    score_loss = 0.5 * (first_grad.reshape(B, -1) ** 2).sum(dim=-1)
    hessian_loss = (v * second_grad).reshape(B, -1).sum(dim=-1)
    loss = (score_loss + hessian_loss) * used.reshape(B) ** 2
    return O.reduce_fn(loss, reduction), score_loss, hessian_loss


def dense_ncsn_params(C, mlp_dims, num_layers, seed=0, dtype=torch.float64):
    """Named DenseNCSN parameters (the arena names) with lecun-normal-like kernels and perturbed norms / biases."""
    g = torch.Generator().manual_seed(seed)
    p = {}

    def dense(pre, i, o):
        p[pre + "kernel"] = torch.randn(i, o, generator=g, dtype=dtype) / i ** 0.5
        p[pre + "bias"] = 0.05 * torch.randn(o, generator=g, dtype=dtype)

    def norm(pre, n):
        p[pre + "scale"] = 1 + 0.1 * torch.randn(n, generator=g, dtype=dtype)
        p[pre + "bias"] = 0.1 * torch.randn(n, generator=g, dtype=dtype)

    dense("in.", C, mlp_dims)
    for k in range(num_layers):
        dense(f"k{k}.film.d1.", 128, 512)
        dense(f"k{k}.film.d2.", 512, 512)
        dense(f"k{k}.film.ss.", 512, 2 * mlp_dims)
        norm(f"k{k}.res.ln_a.", mlp_dims)
        dense(f"k{k}.res.a.", mlp_dims, mlp_dims)
        norm(f"k{k}.res.ln_b.", mlp_dims)
        dense(f"k{k}.res.b.", mlp_dims, mlp_dims)
    norm("out_ln.", mlp_dims)
    dense("out.", mlp_dims, C)
    return p
