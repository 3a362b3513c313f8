"""Latent-space evaluation metrics with the reference's names and semantics (utils/metrics.py:24-77): Frechet
distance between Gaussian fits and kernel (MMD) distances between two sample sets.

frechet_distance / mmd_rbf / mmd_polynomial evaluate them on host arrays, as the reference does with scipy and
scikit-learn.  latent_metrics computes all three on the GPU (smd_latent_stats) from one Gram product of the centred
sets, which scales to the flattened sequence shapes (d = S * C) the host route cannot hold.  The MIDI framewise
statistics of utils/metrics.py:80-244 need note_seq and are out of scope."""
from __future__ import annotations

import math

import numpy as np
import scipy.linalg
import torch

from . import lib as _lib
from . import nn


def frechet_distance(real, fake, eps: float = 1e-6) -> float:
    """|mu1 - mu2|^2 + tr(S1) + tr(S2) - 2 tr(sqrtm(S1 S2))   (utils/metrics.py:24-55).  Lower is better.

    (Upstream's singular-product fallback references an undefined `eps`; 1e-6 -- the value of the FID code it was
    taken from -- is used here.)"""
    real, fake = np.asarray(real, np.float64), np.asarray(fake, np.float64)
    mu1, sigma1 = real.mean(axis=0), np.cov(real, rowvar=False)
    mu2, sigma2 = fake.mean(axis=0), np.cov(fake, rowvar=False)
    diff = mu1 - mu2
    covmean = scipy.linalg.sqrtm(sigma1.dot(sigma2))
    if not np.isfinite(covmean).all():
        offset = np.eye(sigma1.shape[0]) * eps
        covmean = scipy.linalg.sqrtm((sigma1 + offset).dot(sigma2 + offset))
    if np.iscomplexobj(covmean):       # numerical error may leave a slight imaginary component
        if not np.allclose(np.diagonal(covmean).imag, 0, atol=1e-3):
            raise ValueError("Imaginary component {}".format(np.max(np.abs(covmean.imag))))
        covmean = covmean.real
    return float(diff.dot(diff) + np.trace(sigma1) + np.trace(sigma2) - 2.0 * np.trace(covmean))


def _sq_dists(x, y):
    xx = (x * x).sum(axis=1)[:, None]
    yy = (y * y).sum(axis=1)[None, :]
    return np.maximum(xx + yy - 2.0 * x.dot(y.T), 0.0)


def _mmd(real, fake, kernel) -> float:
    real, fake = np.asarray(real, np.float64), np.asarray(fake, np.float64)
    return float(kernel(real, real).mean() + kernel(fake, fake).mean() - 2.0 * kernel(real, fake).mean())


def mmd_rbf(real, fake, gamma: float = 1.0) -> float:
    """Biased MMD^2 estimate with k(x, y) = exp(-gamma |x - y|^2)   (utils/metrics.py:58-66)."""
    return _mmd(real, fake, lambda a, b: np.exp(-gamma * _sq_dists(a, b)))


def mmd_polynomial(real, fake, degree: int = 2, gamma: float = 1, coef0: float = 0) -> float:
    """Biased MMD^2 estimate with k(x, y) = (gamma <x, y> + coef0)^degree   (utils/metrics.py:69-77)."""
    return _mmd(real, fake, lambda a, b: (gamma * a.dot(b.T) + coef0) ** degree)


def combine_latent_stats(stats, cross_nuclear_norm: float, n: int, m: int) -> dict:
    """The three metrics from smd_latent_stats' nine statistics (include/smd.h) and the nuclear norm of its centred
    cross block C = (x - mean x)(y - mean y)^T.  The nonzero eigenvalues of S1 S2 are the squared singular values of
    C / sqrt((n - 1)(m - 1)), so tr sqrtm(S1 S2) = |C|_* / sqrt((n - 1)(m - 1)) at any rank (n < d included)."""
    s = [float(v) for v in stats]
    trace_sqrt = float(cross_nuclear_norm) / math.sqrt((n - 1) * (m - 1))
    return {"frechet_distance": s[0] + s[1] + s[2] - 2.0 * trace_sqrt,
            "mmd_rbf": s[3] + s[4] - 2.0 * s[5],
            "mmd_polynomial": s[6] + s[7] - 2.0 * s[8]}


def latent_metrics(real, fake, gamma: float = 1.0, degree: int = 2, poly_gamma: float = 1.0,
                   coef0: float = 0.0) -> dict:
    """frechet_distance, mmd_rbf(gamma) and mmd_polynomial(degree, poly_gamma, coef0) of real (N, ...) and fake
    (M, ...) on the GPU, each example flattened to one vector.  NumPy arrays or CUDA tensors; returns Python floats.
    Raises ValueError for what smd_latent_stats rejects (fewer than 2 examples, N + M > 16384, degree < 1)."""
    x, y = nn._as_device_f32(real), nn._as_device_f32(fake)
    if x.dim() < 1 or y.dim() < 1:
        raise ValueError("real and fake need a leading example axis")
    x, y = x.reshape(x.shape[0], -1), y.reshape(y.shape[0], -1)
    if x.shape[1] != y.shape[1]:
        raise ValueError(f"real and fake examples differ in size: {tuple(x.shape)} vs {tuple(y.shape)}")
    (n, d), m = x.shape, y.shape[0]
    lib = _lib.load_library()
    ws = torch.empty(lib.smd_latent_stats_workspace_bytes(n, m, d), dtype=torch.uint8, device=x.device)
    stats = torch.empty(9, dtype=torch.float64, device=x.device)
    cross = torch.empty((n, m), dtype=torch.float32, device=x.device)
    _lib.check(lib.smd_latent_stats(x.data_ptr(), n, y.data_ptr(), m, d, float(gamma), int(degree),
                                    float(poly_gamma), float(coef0), ws.data_ptr(), ws.numel(), stats.data_ptr(),
                                    cross.data_ptr(), torch.cuda.current_stream(x.device).cuda_stream))
    nuclear = torch.linalg.svdvals(cross.double()).sum()
    return combine_latent_stats(stats.cpu().numpy(), float(nuclear), n, m)
