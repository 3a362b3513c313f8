"""Host side of the coverage metrics (metrics.py: improved precision / recall, realism, PRD, NDB), without a GPU:
the numpy restatements against scikit-learn where it has the same algorithm, hand-computed cases, the combination
of smd_latent_coverage's outputs, and sample_ncsn --full_metrics."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.stats

from smd_b200 import metrics

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ["f1", "improved_f1", "improved_precision", "improved_recall", "ipr_realism", "ndb", "precision", "recall"]


def blobs(n_per, centers, d, seed, spread=0.05):
    rng = np.random.default_rng(seed)
    c = rng.uniform(-10, 10, (centers, d))
    pts = np.concatenate([c[i] + spread * rng.standard_normal((n_per, d)) for i in range(centers)])
    return pts, np.repeat(np.arange(centers), n_per)


def same_partition(a, b):
    """a and b label the points identically up to a relabelling."""
    pairs = set(zip(np.asarray(a).tolist(), np.asarray(b).tolist()))
    return len(pairs) == len(set(a.tolist())) == len(set(b.tolist()))


def test_knn_radii_and_membership_match_sklearn():
    NearestNeighbors = pytest.importorskip("sklearn.neighbors").NearestNeighbors
    rng = np.random.default_rng(1)
    x, y = rng.standard_normal((150, 12)), 0.8 * rng.standard_normal((120, 12)) + 0.2
    for k in (1, 3, 5):
        rx = NearestNeighbors(n_neighbors=k + 1).fit(x).kneighbors(x)[0][:, k] ** 2
        ry = NearestNeighbors(n_neighbors=k + 1).fit(y).kneighbors(y)[0][:, k] ** 2
        np.testing.assert_allclose(metrics.knn_radii(metrics._sq_dists(x, x), k), rx, rtol=1e-10, atol=1e-12)
        dxy = ((x[:, None, :] - y[None, :, :]) ** 2).sum(-1)
        want_p = np.mean([(dxy[:, b] <= rx).any() for b in range(len(y))])
        want_r = np.mean([(dxy[a] <= ry).any() for a in range(len(x))])
        p, r = metrics.precision_recall(x, y, k=k)
        assert (p, r) == (pytest.approx(want_p, abs=1e-12), pytest.approx(want_r, abs=1e-12))
        med = np.percentile(rx, 50)
        keep = np.where(rx <= med, rx, 0.0)
        want_real = (np.sqrt(keep)[:, None] / (np.sqrt(dxy) + 1e-5)).max(axis=0)
        np.testing.assert_allclose(metrics.realism_scores(x, y, k=k), want_real, rtol=1e-9)


def test_duplicates_count_as_neighbours():
    x = np.array([[0.0], [0.0], [3.0], [7.0]])
    assert metrics.knn_radii(metrics._sq_dists(x, x), 1).tolist() == [0.0, 0.0, 9.0, 16.0]


def test_kmeans_matches_sklearn_on_separated_blobs():
    KMeans = pytest.importorskip("sklearn.cluster").KMeans
    pts, truth = blobs(30, 6, 5, seed=2)
    u = np.random.default_rng(0).random((4, 6))
    labels, inertia, iters = metrics.kmeans_distance(metrics._sq_dists(pts, pts), 6, u)
    sk = KMeans(n_clusters=6, n_init=10, random_state=0).fit(pts)
    assert same_partition(labels, sk.labels_) and same_partition(labels, truth)
    assert inertia == pytest.approx(sk.inertia_, rel=1e-9) and 1 <= iters <= 300


def test_kmeans_seeding_and_ties():
    # four points on a line, two clusters: seed 0 = floor(u0 * 4) = point 1; the prefix sums of the min distances
    # (1, 0, 1, 16) exceed 0.5 * 18 first at point 3
    pts = np.array([[0.0], [1.0], [2.0], [5.0]])
    labels, inertia, _ = metrics.kmeans_distance(metrics._sq_dists(pts, pts), 2, [[0.3, 0.5]])
    assert labels.tolist() == [0, 0, 0, 1] and inertia == pytest.approx(2.0)
    # all points equal: the total is 0, seeds fall back to floor(u N); the second cluster ends empty
    labels, inertia, _ = metrics.kmeans_distance(np.zeros((5, 5)), 2, [[0.1, 0.9]])
    assert labels.tolist() == [0] * 5 and inertia == 0.0


def test_prd_of_identical_and_disjoint_histograms():
    h = np.array([[[5, 3, 0, 2], [5, 3, 0, 2]]] * 3)
    f8, f18 = metrics.prd_f_beta_score(metrics.prd_from_histograms(h))
    assert abs(f8 - 1) < 1e-6 and abs(f18 - 1) < 1e-6
    h = np.array([[[5, 5, 0, 0], [0, 0, 4, 6]]])
    assert metrics.prd_f_beta_score(metrics.prd_from_histograms(h)) == (0.0, 0.0)
    with pytest.raises(ValueError):
        metrics.precision_recall_distribution(np.zeros((5, 2)), np.zeros((6, 2)))


def test_ndb_two_bins_by_hand():
    # bin 0: 30 of 50 real vs 10 of 50 fake -> pooled 0.4, z = 0.4 / sqrt(0.24 * 0.04) = 4.08 (different);
    # bin 1: 20 / 50 vs 40 / 50 -> z = -4.08 (different)
    assert metrics.ndb_from_histogram([[30, 20], [10, 40]], 50, 50) == 1.0
    # 26 / 50 vs 24 / 50: pooled 0.5, z = 0.04 / 0.1 = 0.4 (same); an empty bin does not count
    assert metrics.ndb_from_histogram([[26, 24, 0], [24, 26, 0]], 50, 50) == 0.0
    z = 0.2 / np.sqrt(0.4 * 0.6 * 0.04)
    assert z > scipy.stats.norm.ppf(0.975)
    x, _ = blobs(40, 3, 4, seed=3)
    assert metrics.ndb_score(x, x, k=3) == 0.0


def test_combine_coverage():
    prd = np.array([[[4, 4, 2], [4, 4, 2]], [[5, 5, 0], [5, 5, 0]]])
    got = metrics.combine_coverage([6, 8], np.array([0.5, 1.0, 1.5, 0.0, 2.0, 1.0, 0.5, 0.5, 1.0, 2.0]), prd,
                                   [[5, 5], [10, 0]], 10, 10)
    assert sorted(got) == KEYS and all(isinstance(v, float) for v in got.values())
    assert got["improved_precision"] == 0.6 and got["improved_recall"] == 0.8
    assert got["improved_f1"] == pytest.approx(2 * 0.6 * 0.8 / 1.4)
    assert got["ipr_realism"] == pytest.approx(1.0)
    assert abs(got["precision"] - 1) < 1e-6 and abs(got["recall"] - 1) < 1e-6 and abs(got["f1"] - 1) < 1e-6
    assert got["ndb"] == 1.0           # 5 / 10 vs 10 / 10 and 5 / 10 vs 0 / 10
    with pytest.raises(ValueError):
        metrics.combine_coverage([0, 0], np.zeros(9), prd, [[5, 5], [9, 0]], 10, 9)


def test_host_functions_agree_with_the_device_restatement():
    """precision_recall_distribution / ndb_score consume the same uniforms as smd_latent_coverage
    (coverage_uniforms) and the same k-means as kmeans_distance."""
    rng = np.random.default_rng(4)
    x, y = rng.uniform(-1, 1, (40, 6)), rng.uniform(-1, 1, (40, 6))
    dist = metrics._union_sq_dists(x, y)
    u_prd, u_ndb = metrics.coverage_uniforms(7, prd_clusters=5, prd_runs=2, ndb_bins=4, restarts=3)
    hists = []
    for r in range(2):
        lab = metrics.kmeans_distance(dist, 5, u_prd[r])[0]
        hists.append([np.bincount(lab[:40], minlength=5), np.bincount(lab[40:], minlength=5)])
    want = metrics.prd_from_histograms(hists)
    got = metrics.precision_recall_distribution(x, y, num_clusters=5, num_runs=2, seed=7, restarts=3)
    np.testing.assert_array_equal(got[0], want[0])
    # ndb_score takes the NDB slice of the draw with the default PRD sizes
    _, u_ndb_default = metrics.coverage_uniforms(7, ndb_bins=4, restarts=3)
    hist = metrics.ndb_histogram(dist, 40, 4, u_ndb_default)
    assert metrics.ndb_score(x, y, k=4, seed=7, restarts=3) == metrics.ndb_from_histogram(hist, 40, 40)
    assert hist.sum(axis=1).tolist() == [40, 40]


def _host_full(real, fake):
    real, fake = real.reshape(len(real), -1), fake.reshape(len(fake), -1)
    recall, precision = metrics.prd_f_beta_score(
        metrics.precision_recall_distribution(real, fake, num_clusters=4, num_runs=2, restarts=2))
    ip, ir = metrics.precision_recall(real, fake)
    return {"frechet_distance": metrics.frechet_distance(real, fake), "mmd_rbf": metrics.mmd_rbf(real, fake),
            "mmd_polynomial": metrics.mmd_polynomial(real, fake), "precision": precision, "recall": recall,
            "f1": metrics.f1_score(precision, recall), "improved_precision": ip, "improved_recall": ir,
            "improved_f1": metrics.f1_score(ip, ir), "ipr_realism": float(metrics.realism_scores(real, fake).mean()),
            "ndb": metrics.ndb_score(real, fake, k=3, restarts=2)}


def test_full_metrics_json_layout(tmp_path):
    from smd_b200 import sample_ncsn
    rng = np.random.default_rng(3)
    real = rng.uniform(-1, 1, (16, 4, 3)).astype(np.float32)
    coll = np.stack([real * (0.5 + 0.5 * k / 29) for k in range(30)]).astype(np.float32)
    results = sample_ncsn.evaluate(real, coll, seed=5, final_only=True, metric_fn=_host_full)
    back = json.load(open(sample_ncsn.save_metrics(results, str(tmp_path / "ncsn"))))
    assert sorted(back) == ["ncsn", "random", "real"]
    for model in back.values():
        for vals in model.values():
            assert sorted(vals) == sorted(KEYS + ["frechet_distance", "mmd_polynomial", "mmd_rbf"])
            assert all(np.isfinite(v) for v in vals.values())
    real_vals = back["real"]["0"]
    assert real_vals["improved_precision"] == real_vals["improved_recall"] == 1.0 and real_vals["ndb"] == 0.0


def test_full_metrics_without_compute_metrics_raises(tmp_path):
    r = subprocess.run([sys.executable, "-m", "smd_b200.sample_ncsn", "--full_metrics", f"--model_dir={tmp_path}"],
                       capture_output=True, text=True, timeout=300, cwd=ROOT, env=dict(os.environ, PYTHONPATH=ROOT))
    assert r.returncode != 0 and "ValueError: --full_metrics needs --compute_metrics" in r.stderr, r.stderr[-2000:]
    assert not os.listdir(tmp_path)
