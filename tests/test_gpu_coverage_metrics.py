"""smd_latent_coverage / metrics.coverage_metrics on the GPU against the numpy restatements of metrics.py (improved
precision / recall, realism, PRD and NDB k-means in distance form), and sample_ncsn --full_metrics end to end."""
import json
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from smd_b200 import metrics
from tests.test_coverage_metrics import KEYS

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMALL = dict(neighbors=3, prd_clusters=5, prd_runs=3, ndb_bins=4, restarts=3, max_iter=300)


def _exact_sets(n, m, d, seed):
    """Small integers in +/- pairs around an integer mean: every centred entry, Gram entry and fp64 distance is
    exact, so the device and the host see the same distances."""
    rng = np.random.default_rng(seed)

    def one(rows):
        c = rng.integers(-3, 4, d)
        v = rng.integers(-4, 5, (rows // 2, d))
        return np.concatenate([c + v, c - v]).astype(np.float32)
    return one(n), one(m)


def _host(x, y, cfg, seed):
    """fp64 restatement of every device output from the raw rows."""
    n = len(x)
    dist = metrics._union_sq_dists(x, y)
    counts, realism = metrics.coverage_from_dists(dist, n, cfg["neighbors"])
    u_prd, u_ndb = metrics.coverage_uniforms(seed, cfg["prd_clusters"], cfg["prd_runs"], cfg["ndb_bins"],
                                             cfg["restarts"])
    K = cfg["prd_clusters"]
    prd = []
    for r in range(cfg["prd_runs"]):
        lab = metrics.kmeans_distance(dist, K, u_prd[r], cfg["max_iter"])[0]
        prd.append([np.bincount(lab[:n], minlength=K), np.bincount(lab[n:], minlength=K)])
    ndb = metrics.ndb_histogram(dist, n, cfg["ndb_bins"], u_ndb, cfg["max_iter"])
    return counts, realism, np.array(prd), ndb


def _device(x, y, cfg, seed):
    out = metrics.latent_coverage(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), seed, **cfg)
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in out]


@pytest.mark.parametrize("n,m,d,cfg", [(40, 40, 64, SMALL), (60, 36, 70, SMALL), (96, 128, 200, SMALL),
                                       (64, 64, 33, dict(SMALL, neighbors=1, prd_clusters=12, ndb_bins=9)),
                                       (60, 60, 70, metrics.COVERAGE_DEFAULTS)])
def test_exact_inputs_give_the_host_results(lib, n, m, d, cfg):
    x, y = _exact_sets(n, m, d, seed=n + d)
    counts, realism, prd, ndb, iters = _device(x, y, cfg, seed=3)
    want = _host(x, y, cfg, seed=3)
    np.testing.assert_array_equal(counts, want[0])
    np.testing.assert_allclose(realism, want[1], rtol=1e-12)
    np.testing.assert_array_equal(prd, want[2])
    np.testing.assert_array_equal(ndb, want[3])
    assert prd.sum(axis=2).tolist() == [[n, m]] * cfg["prd_runs"] and ndb.sum(axis=1).tolist() == [n, m]
    assert 1 <= iters[0] <= cfg["max_iter"] and 1 <= iters[1] <= cfg["max_iter"]


def _sets(n, m, d, seed):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-1, 1, (n, d)).astype(np.float32)
    y = (0.8 * rng.uniform(-1, 1, (m, d)) + 0.1 * rng.standard_normal(d)).astype(np.float32)
    return x, y


@pytest.mark.parametrize("n,m,d", [(300, 200, 42), (600, 600, 512), (1000, 1000, 1344), (257, 129, 4100)])
def test_float_inputs_match_the_host_within_the_rounding_margin(lib, n, m, d):
    x, y = _sets(n, m, d, seed=n + d)
    counts, realism, _, _, _ = _device(x, y, metrics.COVERAGE_DEFAULTS, seed=0)
    dist = metrics._union_sq_dists(x, y)
    want_counts, want_realism = metrics.coverage_from_dists(dist, n, 3)
    rx, ry = metrics.knn_radii(dist[:n, :n], 3), metrics.knn_radii(dist[n:, n:], 3)
    dxy = dist[:n, n:]
    # rows with a pair within 1e-4 (relative) of the radius may go either way under the fp32 Gram product
    near_y = (np.abs(dxy - rx[:, None]) < 1e-4 * rx[:, None]).any(axis=0).sum()
    near_x = (np.abs(dxy - ry[None, :]) < 1e-4 * ry[None, :]).any(axis=1).sum()
    assert abs(int(counts[0]) - int(want_counts[0])) <= near_y, (counts, want_counts, near_y)
    assert abs(int(counts[1]) - int(want_counts[1])) <= near_x, (counts, want_counts, near_x)
    assert abs(realism.mean() - want_realism.mean()) <= 1e-4 * want_realism.mean()


def _blob_sets(seed):
    rng = np.random.default_rng(seed)
    centers = rng.uniform(-10, 10, (5, 64))
    sizes_x, sizes_y = [10, 20, 30, 40, 50], [50, 35, 30, 20, 15]
    x = np.concatenate([c + 0.1 * rng.standard_normal((k, 64)) for c, k in zip(centers, sizes_x)])
    y = np.concatenate([c + 0.1 * rng.standard_normal((k, 64)) for c, k in zip(centers, sizes_y)])
    return x.astype(np.float32), y.astype(np.float32)


def test_blobs_partition_as_sklearn(lib):
    KMeans = pytest.importorskip("sklearn.cluster").KMeans
    x, y = _blob_sets(5)
    n = len(x)
    cfg = dict(metrics.COVERAGE_DEFAULTS, prd_clusters=5, ndb_bins=5)
    _, _, prd, ndb, _ = _device(x, y, cfg, seed=1)
    both = np.concatenate([x, y]).astype(np.float64)
    sk = KMeans(n_clusters=5, n_init=10, random_state=0).fit(both).labels_
    want = sorted(zip(np.bincount(sk[:n], minlength=5), np.bincount(sk[n:], minlength=5)))
    for run in prd:
        assert sorted(zip(run[0], run[1])) == want
    km = KMeans(n_clusters=5, n_init=10, random_state=0).fit(x.astype(np.float64))
    want = sorted(zip(np.bincount(km.labels_, minlength=5), np.bincount(km.predict(y.astype(np.float64)), minlength=5)))
    assert sorted(zip(ndb[0], ndb[1])) == want


@pytest.mark.parametrize("n,d", [(200, 42), (1000, 1344)])
def test_real_against_itself(lib, n, d):
    x, _ = _sets(n, 2, d, seed=9)
    got = metrics.coverage_metrics(x, x, seed=2)
    assert sorted(got) == KEYS and all(isinstance(v, float) for v in got.values())
    assert got["improved_precision"] == got["improved_recall"] == 1.0 and got["ndb"] == 0.0
    assert abs(got["precision"] - 1) < 1e-6 and abs(got["recall"] - 1) < 1e-6


def _raw(lib, x, y, cfg, u, ws):
    from smd_b200 import lib as L
    n, d = x.shape
    m = y.shape[0]
    counts = torch.empty(2, dtype=torch.int32, device="cuda")
    realism = torch.empty(m, dtype=torch.float64, device="cuda")
    prd = torch.empty((cfg.prd_runs, 2, cfg.prd_clusters), dtype=torch.int32, device="cuda")
    ndb = torch.empty((2, cfg.ndb_bins), dtype=torch.int32, device="cuda")
    L.check(lib.smd_latent_coverage(x.data_ptr(), n, y.data_ptr(), m, d, cfg, u.data_ptr(), ws.data_ptr(),
                                    ws.numel(), counts.data_ptr(), realism.data_ptr(), prd.data_ptr(), ndb.data_ptr(),
                                    None, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return counts, realism, prd, ndb


def test_repeated_calls_are_bitwise_equal(lib):
    from smd_b200 import lib as L
    x, y = (torch.from_numpy(a).cuda() for a in _sets(1000, 700, 1344, seed=11))
    cfg = L.SmdCoverageConfig(**metrics.COVERAGE_DEFAULTS)
    u_prd, u_ndb = metrics.coverage_uniforms(4)
    u = torch.from_numpy(np.concatenate([u_prd.ravel(), u_ndb.ravel()])).cuda()
    nbytes = lib.smd_latent_coverage_workspace_bytes(1000, 700, 1344, cfg)
    first = _raw(lib, x, y, cfg, u, torch.zeros(nbytes, dtype=torch.uint8, device="cuda"))
    second = _raw(lib, x, y, cfg, u, torch.full((nbytes,), 255, dtype=torch.uint8, device="cuda"))
    assert all(torch.equal(a, b) for a, b in zip(first, second))


def test_rejected_arguments_raise_value_error(lib):
    from smd_b200 import lib as L
    x = torch.zeros((64, 40), device="cuda")
    good = dict(metrics.COVERAGE_DEFAULTS, prd_clusters=4, ndb_bins=4, prd_runs=2, restarts=2)
    cfg = L.SmdCoverageConfig(**good)
    nbytes = lib.smd_latent_coverage_workspace_bytes(64, 64, 40, cfg)
    ws = torch.empty(nbytes + 256, dtype=torch.uint8, device="cuda")
    u = torch.zeros(1000, dtype=torch.float64, device="cuda")
    i32 = torch.zeros(1000, dtype=torch.int32, device="cuda")
    f64 = torch.zeros(1000, dtype=torch.float64, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def call(n=64, m=64, d=40, xp=x.data_ptr(), yp=x.data_ptr(), up=u.data_ptr(), wsp=ws.data_ptr(), nb=nbytes,
             cp=i32.data_ptr(), rp=f64.data_ptr(), pp=i32.data_ptr(), np_=i32.data_ptr(), conf=cfg):
        L.check(lib.smd_latent_coverage(xp, n, yp, m, d, conf, up, wsp, nb, cp, rp, pp, np_, None, st))

    call()
    torch.cuda.synchronize()
    bad_cfgs = [dict(neighbors=0), dict(neighbors=33), dict(prd_clusters=0), dict(prd_clusters=65),
                dict(ndb_bins=0), dict(ndb_bins=65), dict(restarts=0), dict(prd_runs=0), dict(max_iter=0)]
    for kw in bad_cfgs:
        bad = L.SmdCoverageConfig(**dict(good, **kw))
        with pytest.raises(ValueError):
            call(conf=bad)
        assert lib.smd_latent_coverage_workspace_bytes(64, 64, 40, bad) == 0
    # more bins than x rows, more PRD clusters than rows in both sets
    for shape, kw in (((50, 64), dict(ndb_bins=60)), ((4, 4), dict(prd_clusters=10))):
        bad = L.SmdCoverageConfig(**dict(good, **kw))
        with pytest.raises(ValueError):
            call(*shape, conf=bad)
        assert lib.smd_latent_coverage_workspace_bytes(*shape, 40, bad) == 0
    for kw in (dict(n=3), dict(m=3), dict(d=0), dict(n=8192, m=8193), dict(xp=None), dict(yp=None), dict(up=None),
               dict(wsp=None), dict(cp=None), dict(rp=None), dict(pp=None), dict(np_=None), dict(conf=None),
               dict(nb=nbytes - 1), dict(wsp=ws.data_ptr() + 128)):
        with pytest.raises(ValueError):
            call(**kw)
    for shape in ((3, 64, 40), (64, 3, 40), (64, 64, 0), (8192, 8193, 40)):
        assert lib.smd_latent_coverage_workspace_bytes(*shape, cfg) == 0
    assert lib.smd_latent_coverage_workspace_bytes(64, 64, 40, None) == 0
    with pytest.raises(ValueError):
        metrics.coverage_metrics(np.zeros((64, 5), np.float32), np.zeros((60, 5), np.float32))
    with pytest.raises(ValueError):
        metrics.coverage_metrics(np.zeros((64, 5), np.float32), np.zeros((64, 6), np.float32))
    with pytest.raises(ValueError):
        metrics.coverage_metrics(np.zeros((40, 5), np.float32), np.zeros((40, 5), np.float32))   # 50 NDB bins


def test_sample_ncsn_full_metrics(tmp_path):
    """A tiny DDPM checkpoint on --synthetic data, then sample_ncsn --compute_metrics --full_metrics over 64 samples."""
    cfg = tmp_path / "ddpm-tiny.cfg"
    cfg.write_text(textwrap.dedent(f"""\
        --loss=ddpm
        --sampling=ddpm
        --schedule_type=linear
        --sigma_begin=1e-6
        --sigma_end=0.01
        --num_sigmas=50
        --continuous_noise
        --problem=vae
        --ema=False
        --nosnapshot_sampling
        --architecture=TransformerDDPM
        --num_layers=1
        --num_mlp_layers=1
        --data_shape=32,42
        --batch_size=8
        --learning_rate=1e-3
        --max_steps=3
        --snapshot_freq=3
        --logging_freq=3
        --synthetic
        --synthetic_examples=64
        --model_dir={tmp_path / 'run'}
        """))
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "smd_b200.train_ncsn", f"--flagfile={cfg}"], capture_output=True,
                       text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([sys.executable, "-m", "smd_b200.sample_ncsn", f"--flagfile={cfg}", "--sample_size=64",
                        "--compute_metrics", "--full_metrics"], capture_output=True, text=True, timeout=600, env=env,
                       cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.load(open(tmp_path / "run" / "samples" / "ncsn" / "metrics.json"))
    assert sorted(res) == ["ncsn", "random", "real"] and len(res["ncsn"]) == 20
    for model in res.values():
        for vals in model.values():
            assert sorted(vals) == sorted(KEYS + ["frechet_distance", "mmd_polynomial", "mmd_rbf"])
            assert all(np.isfinite(v) for v in vals.values())
            assert all(0.0 <= vals[k] <= 1.0 for k in KEYS if k != "ipr_realism") and vals["ipr_realism"] >= 0.0
    real = res["real"]["0"]
    assert real["improved_precision"] == real["improved_recall"] == 1.0 and real["ndb"] == 0.0
    assert "ipr_realism=" in r.stderr and "frechet_distance=" in r.stderr
