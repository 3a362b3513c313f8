"""Latent-space evaluation metrics with the reference's names and semantics (utils/metrics.py:24-77): Frechet
distance between Gaussian fits and kernel (MMD) distances between two sample sets.

frechet_distance / mmd_rbf / mmd_polynomial evaluate them on host arrays, as the reference does with scipy and
scikit-learn.  latent_metrics computes all three on the GPU (smd_latent_stats) from one Gram product of the centred
sets, which scales to the flattened sequence shapes (d = S * C) the host route cannot hold.  The MIDI framewise
statistics of utils/metrics.py:80-244 need note_seq and are out of scope.

Coverage metrics.  sample_ncsn.py:132-159 also calls precision_recall_distribution, prd_f_beta_score, f1_score,
precision_recall, realism_scores and ndb_score, which the reference never defines.  They are defined here after the
published metrics their names refer to:
  - precision_recall / realism_scores: improved precision and recall and the realism score of Kynkaanniemi et al.
    2019 (k-NN radii in the real and the fake set; realism with the real radii above their median pruned);
  - precision_recall_distribution / prd_f_beta_score: PRD of Sajjadi et al. 2018 (k-means histograms of the union,
    averaged over runs; F_8 and F_1/8; equal set sizes, as the published enforce_balance);
  - ndb_score: NDB of Richardson & Weiss 2018 (k-means bins of the real set, two-proportion z-test at 0.05) over k.
The host functions are numpy fp64 restatements and serve as the test reference.  k-means is Lloyd's algorithm on a
squared-distance matrix with k-means++ seeding from given uniforms (kmeans_distance); the uniforms come from
np.random.default_rng(seed) in the layout coverage_uniforms describes, so host and device use the same seeds.
coverage_metrics computes all eight values on the GPU (smd_latent_coverage) from the same Gram product as
latent_metrics."""
from __future__ import annotations

import math

import numpy as np
import scipy.linalg
import scipy.stats
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


# ---- coverage metrics (sample_ncsn.py:132-159) ------------------------------------------------------------------
COVERAGE_DEFAULTS = dict(neighbors=3, prd_clusters=20, prd_runs=10, ndb_bins=50, restarts=10, max_iter=300)


def _flat64(a):
    a = np.asarray(a, np.float64)
    return a.reshape(len(a), -1)


def _union_sq_dists(real, fake):
    z = np.concatenate([_flat64(real), _flat64(fake)])
    return _sq_dists(z, z)


def coverage_uniforms(seed, prd_clusters=20, prd_runs=10, ndb_bins=50, restarts=10):
    """The k-means++ uniforms of one evaluation: (prd_runs * prd_clusters + ndb_bins) * restarts draws of
    np.random.default_rng(seed).random, PRD run r / restart s at [(r * restarts + s) * prd_clusters], then NDB restart
    s at [prd_runs * restarts * prd_clusters + s * ndb_bins] (include/smd.h, smd_latent_coverage).  Returns
    (prd (prd_runs, restarts, prd_clusters), ndb (restarts, ndb_bins))."""
    u = np.random.default_rng(seed).random((prd_runs * prd_clusters + ndb_bins) * restarts)
    cut = prd_runs * restarts * prd_clusters
    return u[:cut].reshape(prd_runs, restarts, prd_clusters), u[cut:].reshape(restarts, ndb_bins)


def knn_radii(dist, k):
    """k-th smallest entry of each row of the square distance matrix dist, the diagonal (self) excluded by index."""
    d = np.array(dist, np.float64)
    np.fill_diagonal(d, np.inf)
    return np.partition(d, k - 1, axis=1)[:, k - 1]


def coverage_from_dists(dist, n, k=3):
    """(counts, realism) of smd_latent_coverage from the (n + m)^2 squared distances of x (first n rows) and y:
    counts[0] = y rows within r_a of some x row a, counts[1] = the reverse; realism of each y row from the x radii
    with those above their median set to 0."""
    dxx, dyy, dxy = dist[:n, :n], dist[n:, n:], dist[:n, n:]
    rx, ry = knn_radii(dxx, k), knn_radii(dyy, k)
    counts = np.array([(dxy <= rx[:, None]).any(axis=0).sum(), (dxy <= ry[None, :]).any(axis=1).sum()])
    pruned = np.where(rx > np.percentile(rx, 50), 0.0, rx)
    realism = (np.sqrt(pruned)[:, None] / (np.sqrt(dxy) + 1e-5)).max(axis=0)
    return counts, realism


def _cluster_sums(dist, labels, k):
    """S(p, C) = sum of dist[p, b] over the columns b with labels[b] = C."""
    return dist @ np.eye(k)[labels]


def _within(S, labels, k):
    size = np.bincount(labels, minlength=k).astype(np.float64)
    W = np.array([S[labels == c, c].sum() for c in range(k)])
    return W, size


def _nearest(S, W, size):
    """argmin_C S(p, C) / |C| - W_C / (2 |C|^2) over the nonempty clusters, lowest index on ties."""
    with np.errstate(divide="ignore", invalid="ignore"):
        v = S / size - W / (2.0 * size * size)
    v[:, size == 0] = np.inf
    return v.argmin(axis=1)


def kmeans_distance(dist, k, uniforms, max_iter=300):
    """Lloyd's k-means on the points of the square squared-distance matrix dist, without centroid vectors: every
    distance to a cluster mean is S(p, C) / |C| - W_C / (2 |C|^2) (S(p, C) = sum_{b in C} dist[p, b], W_C = sum_{p in C}
    S(p, C)).  One restart per row of uniforms (restarts, k): k-means++ seeding (seed 0 = floor(u_0 N); seed j = the
    smallest index whose prefix sum of the min distance to the seeds exceeds u_j times the total, floor(u_j N) if the
    total is 0), then reassignment to the nearest cluster (lowest index on ties, empty clusters stay empty) until no
    label changes or max_iter iterations.  Returns (labels, inertia, iterations) of the restart with the lowest inertia
    sum_C W_C / (2 |C|) (lowest restart on ties); iterations is the most any restart ran."""
    dist = np.asarray(dist, np.float64)
    N = len(dist)
    best, most = None, 0
    for u in np.asarray(uniforms, np.float64).reshape(-1, k):
        s = min(int(u[0] * N), N - 1)
        mind, labels = dist[s].copy(), np.zeros(N, np.int64)
        for j in range(1, k):
            cum = np.cumsum(mind)
            total = cum[-1]
            s = min(int(np.searchsorted(cum, u[j] * total, side="right")), N - 1) if total > 0 else \
                min(int(u[j] * N), N - 1)
            closer = dist[s] < mind
            mind[closer], labels[closer] = dist[s][closer], j
        it = 0
        for it in range(1, max_iter + 1):
            S = _cluster_sums(dist, labels, k)
            W, size = _within(S, labels, k)
            new = _nearest(S, W, size)
            if np.array_equal(new, labels):
                break
            labels = new
        else:
            S = _cluster_sums(dist, labels, k)
            W, size = _within(S, labels, k)
        most = max(most, it)
        inertia = 0.0
        for c in range(k):
            if size[c]:
                inertia += W[c] / (2.0 * size[c])
        if best is None or inertia < best[1]:
            best = (labels, inertia, W, size)
    return best[0], best[1], most


def _prd_curve(ref_hist, eval_hist, num_angles=1001, epsilon=1e-10):
    """Sajjadi et al.: precision(l) = sum min(l p_ref, p_eval), recall = precision / l, l = tan of num_angles angles
    in (0, pi/2), clipped to [0, 1] against rounding."""
    slopes = np.tan(np.linspace(epsilon, np.pi / 2 - epsilon, num_angles))
    ref = np.asarray(ref_hist, np.float64) / np.sum(ref_hist)
    ev = np.asarray(eval_hist, np.float64) / np.sum(eval_hist)
    precision = np.minimum(ref[None, :] * slopes[:, None], ev[None, :]).sum(axis=1)
    recall = precision / slopes
    return np.clip(precision, 0, 1), np.clip(recall, 0, 1)


def prd_from_histograms(hists, num_angles=1001):
    """PRD curve (precision, recall) averaged over runs of (runs, 2, clusters) histograms, [:, 0] the reference
    (real) counts and [:, 1] the evaluated (fake) counts."""
    curves = [_prd_curve(h[0], h[1], num_angles) for h in np.asarray(hists)]
    return np.mean([c[0] for c in curves], axis=0), np.mean([c[1] for c in curves], axis=0)


def precision_recall_distribution(real, fake, num_clusters=20, num_angles=1001, num_runs=10, seed=0, restarts=10,
                                  max_iter=300):
    """PRD (Sajjadi et al. 2018) of fake (the evaluated set) against real (the reference set): num_runs k-means fits
    of both sets together, their histograms turned into precision / recall curves and averaged.  Raises ValueError
    for sets of different sizes (the published enforce_balance)."""
    real, fake = _flat64(real), _flat64(fake)
    if len(real) != len(fake):
        raise ValueError(f"PRD needs sets of equal size: {len(real)} real vs {len(fake)} fake examples")
    n = len(real)
    dist = _union_sq_dists(real, fake)
    u, _ = coverage_uniforms(seed, num_clusters, num_runs, 1, restarts)
    hists = []
    for r in range(num_runs):
        labels = kmeans_distance(dist, num_clusters, u[r], max_iter)[0]
        hists.append([np.bincount(labels[:n], minlength=num_clusters), np.bincount(labels[n:], minlength=num_clusters)])
    return prd_from_histograms(hists, num_angles)


def _f_beta(precision, recall, beta):
    return (1 + beta ** 2) * (precision * recall) / ((beta ** 2 * precision) + recall + 1e-10)


def prd_f_beta_score(prd, beta=8):
    """(max F_beta, max F_1/beta) over a PRD curve (precision, recall); the reference unpacks them as recall,
    precision."""
    precision, recall = (np.asarray(a, np.float64) for a in prd)
    return float(np.max(_f_beta(precision, recall, beta))), float(np.max(_f_beta(precision, recall, 1.0 / beta)))


def f1_score(precision, recall):
    """2PR / (P + R), 0 when P + R = 0."""
    s = precision + recall
    return float(2.0 * precision * recall / s) if s > 0 else 0.0


def precision_recall(real, fake, k=3):
    """Improved precision (share of fake examples inside the real k-NN manifold) and recall (share of real examples
    inside the fake one), Kynkaenniemi et al. 2019."""
    n, m = len(real), len(fake)
    counts, _ = coverage_from_dists(_union_sq_dists(real, fake), n, k)
    return float(counts[0] / m), float(counts[1] / n)


def realism_scores(real, fake, k=3):
    """Realism score of every fake example (Kynkaenniemi et al. 2019): max over real a of r_a / |a - b|, with the real
    k-NN radii r_a above their median set to 0 (and 1e-5 added to the distance)."""
    return coverage_from_dists(_union_sq_dists(real, fake), len(real), k)[1]


def ndb_from_histogram(hist, n, m, alpha=0.05):
    """Share of bins whose real (hist[0], n examples) and fake (hist[1], m) proportions differ in a two-proportion
    z-test at level alpha; bins with a pooled proportion of 0 or 1 do not count."""
    P, Q = np.asarray(hist[0], np.float64) / n, np.asarray(hist[1], np.float64) / m
    pooled = (np.asarray(hist[0], np.float64) + np.asarray(hist[1], np.float64)) / (n + m)
    ok = (pooled > 0) & (pooled < 1)
    se = np.sqrt(np.where(ok, pooled * (1 - pooled), 1.0) * (1.0 / n + 1.0 / m))
    z = (P - Q) / se
    return float(np.sum(ok & (np.abs(z) > scipy.stats.norm.ppf(1 - alpha / 2))) / len(P))


def ndb_histogram(dist, n, k, uniforms, max_iter=300):
    """NDB bins: k-means of the first n points of the square distance matrix dist (the real set), then every other
    point to its nearest bin.  Returns the (2, k) real and fake counts."""
    labels = kmeans_distance(dist[:n, :n], k, uniforms, max_iter)[0]
    S = _cluster_sums(dist[:n, :n], labels, k)
    W, size = _within(S, labels, k)
    y_labels = _nearest(_cluster_sums(dist[n:, :n], labels, k), W, size)
    return np.array([np.bincount(labels, minlength=k), np.bincount(y_labels, minlength=k)])


def ndb_score(real, fake, k=50, seed=0, restarts=10, max_iter=300):
    """NDB / k (Richardson & Weiss 2018): k-means bins of real, each fake example to its nearest bin, and the share of
    bins whose proportions differ significantly."""
    n, m = len(real), len(fake)
    _, u = coverage_uniforms(seed, ndb_bins=k, restarts=restarts)
    return ndb_from_histogram(ndb_histogram(_union_sq_dists(real, fake), n, k, u, max_iter), n, m)


def combine_coverage(counts, realism, prd_hist, ndb_hist, n: int, m: int) -> dict:
    """The eight coverage values (sample_ncsn.py:142-159) from smd_latent_coverage's outputs for real x (n) and fake
    y (m)."""
    if n != m:
        raise ValueError(f"PRD needs sets of equal size: {n} real vs {m} fake examples")
    counts = [int(c) for c in counts]
    recall, precision = prd_f_beta_score(prd_from_histograms(np.asarray(prd_hist)))
    improved_p, improved_r = counts[0] / m, counts[1] / n
    return {"precision": precision, "recall": recall, "f1": f1_score(precision, recall),
            "improved_precision": improved_p, "improved_recall": improved_r,
            "improved_f1": f1_score(improved_p, improved_r),
            "ipr_realism": float(np.mean(np.asarray(realism, np.float64))),
            "ndb": ndb_from_histogram(np.asarray(ndb_hist), n, m)}


def latent_coverage(real, fake, seed=0, neighbors=3, prd_clusters=20, prd_runs=10, ndb_bins=50, restarts=10,
                    max_iter=300):
    """Raw smd_latent_coverage outputs (counts, realism, prd_hist, ndb_hist, iterations) as CUDA tensors, with the
    uniforms of coverage_uniforms(seed, ...).  Raises ValueError for what the call rejects."""
    x, y = nn._as_device_f32(real), nn._as_device_f32(fake)
    if x.dim() < 1 or y.dim() < 1:
        raise ValueError("real and fake need a leading example axis")
    x, y = x.reshape(x.shape[0], -1), y.reshape(y.shape[0], -1)
    if x.shape[1] != y.shape[1]:
        raise ValueError(f"real and fake examples differ in size: {tuple(x.shape)} vs {tuple(y.shape)}")
    (n, d), m = x.shape, y.shape[0]
    cfg = _lib.SmdCoverageConfig(neighbors, prd_clusters, prd_runs, ndb_bins, restarts, max_iter)
    lib = _lib.load_library()
    nbytes = lib.smd_latent_coverage_workspace_bytes(n, m, d, cfg)
    if nbytes == 0:      # the call below reports why
        nbytes = 256
    u_prd, u_ndb = coverage_uniforms(seed, max(prd_clusters, 1), max(prd_runs, 1), max(ndb_bins, 1), max(restarts, 1))
    u = torch.from_numpy(np.concatenate([u_prd.ravel(), u_ndb.ravel()])).to(x.device)
    dev = dict(device=x.device)
    ws = torch.empty(nbytes, dtype=torch.uint8, **dev)
    counts = torch.empty(2, dtype=torch.int32, **dev)
    realism = torch.empty(m, dtype=torch.float64, **dev)
    prd_hist = torch.empty((max(prd_runs, 1), 2, max(prd_clusters, 1)), dtype=torch.int32, **dev)
    ndb_hist = torch.empty((2, max(ndb_bins, 1)), dtype=torch.int32, **dev)
    iterations = torch.empty(2, dtype=torch.int32, **dev)
    _lib.check(lib.smd_latent_coverage(x.data_ptr(), n, y.data_ptr(), m, d, cfg, u.data_ptr(), ws.data_ptr(),
                                       ws.numel(), counts.data_ptr(), realism.data_ptr(), prd_hist.data_ptr(),
                                       ndb_hist.data_ptr(), iterations.data_ptr(),
                                       torch.cuda.current_stream(x.device).cuda_stream))
    return counts, realism, prd_hist, ndb_hist, iterations


def coverage_metrics(real, fake, seed=0, neighbors=3, prd_clusters=20, prd_runs=10, ndb_bins=50, restarts=10,
                     max_iter=300) -> dict:
    """precision, recall, f1 (PRD), improved_precision, improved_recall, improved_f1, ipr_realism and ndb of real
    (N, ...) and fake (N, ...) on the GPU, each example flattened to one vector; Python floats.  Raises ValueError for
    what smd_latent_coverage rejects and for sets of different sizes (PRD)."""
    if len(real) != len(fake):
        raise ValueError(f"PRD needs sets of equal size: {len(real)} real vs {len(fake)} fake examples")
    counts, realism, prd_hist, ndb_hist, _ = latent_coverage(real, fake, seed, neighbors, prd_clusters, prd_runs,
                                                             ndb_bins, restarts, max_iter)
    return combine_coverage(counts.cpu().numpy(), realism.cpu().numpy(), prd_hist.cpu().numpy(),
                            ndb_hist.cpu().numpy(), len(real), len(fake))
