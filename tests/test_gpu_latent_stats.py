"""smd_latent_stats / metrics.latent_metrics on the GPU against the host metrics (utils/metrics.py:24-77) on the same
fp32 inputs in fp64, and sample_ncsn --compute_metrics end to end."""
import json
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from smd_b200 import metrics
from tests.test_latent_stats import latent_stats_np

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _sets(n, m, d, seed):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-1, 1, (n, d)).astype(np.float32)
    y = (0.8 * rng.uniform(-1, 1, (m, d)) + 0.1 * rng.standard_normal(d)).astype(np.float32)
    return x, y


def _run(lib, x, y, gamma=1.0, degree=2, poly_gamma=1.0, coef0=0.0, ws=None):
    from smd_b200 import lib as L
    n, d = x.shape
    m = y.shape[0]
    if ws is None:
        ws = torch.empty(lib.smd_latent_stats_workspace_bytes(n, m, d), dtype=torch.uint8, device="cuda")
    stats = torch.empty(9, dtype=torch.float64, device="cuda")
    cross = torch.empty((n, m), dtype=torch.float32, device="cuda")
    L.check(lib.smd_latent_stats(x.data_ptr(), n, y.data_ptr(), m, d, gamma, degree, poly_gamma, coef0, ws.data_ptr(),
                                 ws.numel(), stats.data_ptr(), cross.data_ptr(), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return stats, cross


@pytest.mark.parametrize("n,m,d", [(300, 200, 42), (600, 600, 512), (1000, 1000, 1344), (257, 129, 4100)])
def test_latent_metrics_match_the_host_metrics(lib, n, m, d):
    x, y = _sets(n, m, d, seed=n + d)
    x64, y64 = x.astype(np.float64), y.astype(np.float64)
    want_stats, _ = latent_stats_np(x64, y64)
    tr = want_stats[1] + want_stats[2]
    if d <= 1344:
        want_fd = metrics.frechet_distance(x64, y64)
    else:   # sqrtm of a 4100 x 4100 singular product: the fp64 Gram restatement instead
        want_fd = metrics.combine_latent_stats(*_np_combination_inputs(x64, y64), n, m)["frechet_distance"]
    for gamma in (1.0, 1.0 / d):
        got = metrics.latent_metrics(x, torch.from_numpy(y).cuda(), gamma=gamma)
        assert set(got) == {"frechet_distance", "mmd_rbf", "mmd_polynomial"}
        assert all(isinstance(v, float) for v in got.values())
        assert abs(got["frechet_distance"] - want_fd) <= 1e-4 * tr, (got["frechet_distance"], want_fd, tr)
        want_rbf = metrics.mmd_rbf(x64, y64, gamma=np.float32(gamma))
        assert abs(got["mmd_rbf"] - want_rbf) <= 1e-5, (gamma, got["mmd_rbf"], want_rbf)
    want_pol = metrics.mmd_polynomial(x64, y64)
    assert abs(got["mmd_polynomial"] - want_pol) <= 1e-4 * max(abs(want_stats[6:9])), (got["mmd_polynomial"], want_pol)
    # the raw statistics: |delta|^2 from the fp64 means, the traces from the Gram diagonal (bf16x3 products, fp32
    # accumulation over d: the same 1e-4 budget as the Frechet distance), and (N, S, C) inputs flatten to the same result
    stats = _run(lib, torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda())[0].cpu().numpy()
    assert abs(stats[0] - want_stats[0]) <= 1e-9 * want_stats[0]
    np.testing.assert_allclose(stats[1:3], want_stats[1:3], rtol=1e-4)
    if d % 2 == 0:
        got3 = metrics.latent_metrics(x.reshape(n, 2, d // 2), y.reshape(m, 2, d // 2))
        assert got3 == pytest.approx(metrics.latent_metrics(x, y), rel=1e-12, abs=1e-12)


def _np_combination_inputs(x, y):
    stats, cross = latent_stats_np(x, y)
    return stats, np.linalg.svd(cross, compute_uv=False).sum()


@pytest.mark.parametrize("n,d", [(300, 42), (1000, 1344)])
def test_identical_sets_are_at_zero(lib, n, d):
    x, _ = _sets(n, 2, d, seed=7)
    want_stats, _ = latent_stats_np(x, x)
    for gamma in (1.0, 1.0 / d):
        got = metrics.latent_metrics(x, x, gamma=gamma)
        assert abs(got["frechet_distance"]) <= 1e-4 * (want_stats[1] + want_stats[2])
        assert abs(got["mmd_rbf"]) <= 1e-5
        assert abs(got["mmd_polynomial"]) <= 1e-4 * max(abs(want_stats[6:9]))


def test_repeated_calls_are_bitwise_equal(lib):
    x, y = (torch.from_numpy(a).cuda() for a in _sets(1000, 700, 1344, seed=11))
    s1, c1 = _run(lib, x, y, gamma=1.0 / 1344, degree=3, poly_gamma=0.5, coef0=1.0)
    ws = torch.full((lib.smd_latent_stats_workspace_bytes(1000, 700, 1344),), 255, dtype=torch.uint8, device="cuda")
    s2, c2 = _run(lib, x, y, gamma=1.0 / 1344, degree=3, poly_gamma=0.5, coef0=1.0, ws=ws)
    assert torch.equal(s1, s2) and torch.equal(c1, c2)


def test_rejected_arguments_raise_value_error(lib):
    from smd_b200 import lib as L
    x = torch.zeros((8, 64), device="cuda")
    stats = torch.empty(9, dtype=torch.float64, device="cuda")
    ws = torch.empty(lib.smd_latent_stats_workspace_bytes(8, 8, 64), dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def call(n=8, m=8, d=64, degree=2, xp=x.data_ptr(), yp=x.data_ptr(), wsp=ws.data_ptr(), nbytes=ws.numel(),
             sp=stats.data_ptr()):
        L.check(lib.smd_latent_stats(xp, n, yp, m, d, 1.0, degree, 1.0, 0.0, wsp, nbytes, sp, None, st))

    call()
    for kw in (dict(n=1), dict(m=1), dict(d=0), dict(degree=0), dict(n=8192, m=8193), dict(xp=None), dict(yp=None),
               dict(wsp=None), dict(sp=None), dict(nbytes=ws.numel() - 1)):
        with pytest.raises(ValueError):
            call(**kw)
    assert lib.smd_latent_stats_workspace_bytes(8192, 8193, 64) == 0
    with pytest.raises(ValueError):
        metrics.latent_metrics(np.zeros((1, 5), np.float32), np.zeros((4, 5), np.float32))
    with pytest.raises(ValueError):
        metrics.latent_metrics(np.zeros((4, 5), np.float32), np.zeros((4, 6), np.float32))


def test_sample_ncsn_compute_metrics(tmp_path):
    """A tiny DDPM checkpoint on --synthetic data, then sample_ncsn --compute_metrics over 64 samples."""
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
                        "--compute_metrics"], capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.load(open(tmp_path / "run" / "samples" / "ncsn" / "metrics.json"))
    assert sorted(res) == ["ncsn", "random", "real"] and len(res["ncsn"]) == 20
    for model in res.values():
        for vals in model.values():
            assert sorted(vals) == ["frechet_distance", "mmd_polynomial", "mmd_rbf"]
            assert all(np.isfinite(v) for v in vals.values())
    # real against itself is zero up to rounding, far below the distance to the standard-normal baseline
    assert abs(res["real"]["0"]["frechet_distance"]) < 1e-4 * res["random"]["0"]["frechet_distance"]
    assert "frechet_distance=" in r.stderr      # train_utils.log_metrics of the last point
