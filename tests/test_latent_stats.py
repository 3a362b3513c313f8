"""Host side of the GPU latent metrics, without a GPU: the combination of smd_latent_stats' outputs into Frechet
distance and MMDs (fed with an fp64 NumPy restatement of those outputs), and sample_ncsn's --compute_metrics
evaluation layout."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from smd_b200 import metrics

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def latent_stats_np(x, y, gamma=1.0, degree=2, poly_gamma=1.0, coef0=0.0):
    """fp64 restatement of smd_latent_stats: the nine statistics and the centred cross block."""
    x = np.asarray(x, np.float64).reshape(len(x), -1)
    y = np.asarray(y, np.float64).reshape(len(y), -1)
    n, m = len(x), len(y)
    xc, yc = x - x.mean(0), y - y.mean(0)
    delta = x.mean(0) - y.mean(0)
    rbf = lambda a, b: np.exp(-gamma * metrics._sq_dists(a, b)).mean()  # noqa: E731
    pol = lambda a, b: ((poly_gamma * a.dot(b.T) + coef0) ** degree).mean()  # noqa: E731
    stats = [delta @ delta, (xc * xc).sum() / (n - 1), (yc * yc).sum() / (m - 1),
             rbf(x, x), rbf(y, y), rbf(x, y), pol(x, x), pol(y, y), pol(x, y)]
    return np.array(stats), xc @ yc.T


def combine_np(x, y, **kw):
    stats, cross = latent_stats_np(x, y, **kw)
    return metrics.combine_latent_stats(stats, np.linalg.svd(cross, compute_uv=False).sum(), len(x), len(y))


# n > d, and n < d where both covariances are singular
@pytest.mark.parametrize("n,m,d", [(400, 300, 64), (120, 90, 700)])
def test_combination_reproduces_the_host_metrics(n, m, d):
    rng = np.random.default_rng(n + d)
    x = rng.uniform(-1, 1, (n, d))
    y = 0.7 * rng.uniform(-1, 1, (m, d)) + 0.05 * rng.standard_normal(d)
    for gamma in (1.0, 1.0 / d):
        got = combine_np(x, y, gamma=gamma, degree=3, poly_gamma=0.5, coef0=1.0)
        want_rbf = metrics.mmd_rbf(x, y, gamma=gamma)
        assert abs(got["mmd_rbf"] - want_rbf) <= 1e-9 * abs(want_rbf)
    want_pol = metrics.mmd_polynomial(x, y, degree=3, gamma=0.5, coef0=1.0)
    assert abs(got["mmd_polynomial"] - want_pol) <= 1e-9 * abs(want_pol)
    want_fd = metrics.frechet_distance(x, y)
    # for n < d, scipy's sqrtm of the singular product S1 S2 is itself only good to ~1e-7 relative; the nuclear norm
    # of the n x m cross block has no such loss, so there the bound is the reference's own accuracy
    tol = 1e-9 if n > d else 1e-6
    assert abs(got["frechet_distance"] - want_fd) <= tol * abs(want_fd), (got["frechet_distance"], want_fd)


def test_combination_of_identical_sets_is_zero():
    x = np.random.default_rng(2).uniform(-1, 1, (200, 30))
    got = combine_np(x, x)
    assert abs(got["frechet_distance"]) < 1e-9 and abs(got["mmd_rbf"]) < 1e-12 and abs(got["mmd_polynomial"]) < 1e-9


def test_evaluation_points():
    from smd_b200 import sample_ncsn
    coll = np.arange(41)[:, None, None] * np.ones((1, 3, 2))
    pts = sample_ncsn.evaluation_points(coll)
    idx = [int(p[0, 0]) for p in pts]
    assert idx == list(np.linspace(0, 40, 20).astype(np.uint32)) and idx[0] == 0 and idx[-1] == 40
    last = sample_ncsn.evaluation_points(coll, final_only=True)
    assert len(last) == 1 and int(last[0][0, 0]) == 40


def _host_metrics(real, fake):
    real, fake = real.reshape(len(real), -1), fake.reshape(len(fake), -1)
    return {"frechet_distance": metrics.frechet_distance(real, fake), "mmd_rbf": metrics.mmd_rbf(real, fake),
            "mmd_polynomial": metrics.mmd_polynomial(real, fake)}


@pytest.mark.parametrize("final_only", [False, True])
def test_metrics_json_layout(tmp_path, final_only):
    from smd_b200 import sample_ncsn
    rng = np.random.default_rng(3)
    real = rng.uniform(-1, 1, (24, 4, 3)).astype(np.float32)
    coll = np.stack([real * (0.5 + 0.5 * k / 29) for k in range(30)]).astype(np.float32)
    results = sample_ncsn.evaluate(real, coll, seed=5, final_only=final_only, metric_fn=_host_metrics)
    path = sample_ncsn.save_metrics(results, str(tmp_path / "ncsn"))
    assert path == str(tmp_path / "ncsn" / "metrics.json")
    back = json.load(open(path))
    assert sorted(back) == ["ncsn", "random", "real"]
    npts = 1 if final_only else 20
    assert sorted(back["ncsn"], key=int) == [str(i) for i in range(npts)]
    assert list(back["random"]) == ["0"] and list(back["real"]) == ["0"]
    for model in back.values():
        for vals in model.values():
            assert sorted(vals) == ["frechet_distance", "mmd_polynomial", "mmd_rbf"]
            assert all(np.isfinite(v) for v in vals.values())
    assert abs(back["real"]["0"]["frechet_distance"]) < 1e-9
    # the last point is the collection's last entry; the random baseline is seeded
    assert back["ncsn"][str(npts - 1)] == pytest.approx(_host_metrics(real, coll[-1]))
    again = sample_ncsn.evaluate(real, coll, seed=5, final_only=final_only, metric_fn=_host_metrics)
    assert again["random"] == results["random"]
    with pytest.raises(ValueError):
        sample_ncsn.evaluate(real[:10], coll, seed=5, metric_fn=_host_metrics)
    with pytest.warns(UserWarning, match="Normalize"):      # samples outside [-1, 1]
        sample_ncsn.evaluate(real, 2 * coll, seed=5, final_only=True, metric_fn=_host_metrics)


def test_interpolate_with_compute_metrics_raises(tmp_path):
    r = subprocess.run([sys.executable, "-m", "smd_b200.sample_ncsn", "--interpolate", "--compute_metrics",
                        f"--model_dir={tmp_path}"], capture_output=True, text=True, timeout=300, cwd=ROOT,
                       env=dict(os.environ, PYTHONPATH=ROOT))
    assert r.returncode != 0 and "ValueError: --compute_metrics does not apply to --interpolate" in r.stderr, \
        r.stderr[-2000:]
    assert not os.listdir(tmp_path)
