"""Sliced score matching on DenseNCSN (utils/losses.py:182-247): draws, the tangent (Jacobian-vector product) pass and
its second-order backward through the C ABI, against the CPU restatement on the same seeded inputs.

Tolerances are about twice the errors measured on an H100 with bf16 tensor-core operands (the strict test: bf16x3)."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from oracle import ddpm_oracle as O
from oracle import threefry as tf
from tests import ssm_reference as R
from tests.util import params_torch, rel_l2

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KW = dict(num_layers=2, mlp_dims=2048)
C = 64
SIGMAS = O.create_noise_schedule(1.0, 0.01, 15, "geometric")


def _engine(batch, training=False, precision=None):
    from smd_b200 import Engine, ModelConfig
    eng = Engine(ModelConfig(arch="DenseNCSN", channels=C, **KW), max_batch=batch, cta_group=2, training=training,
                 precision=precision)
    flat = eng.init_params(seed=4, perturb=0.02)
    eng.set_params(flat)
    return eng, flat


def _inputs(B, seed):
    rng = np.random.default_rng(seed)
    x0 = rng.uniform(-1, 1, (B, C)).astype(np.float32)
    eps = rng.standard_normal((B, C)).astype(np.float32)
    v = np.where(rng.random((B, C)) < 0.5, 1.0, -1.0).astype(np.float32)
    sig = SIGMAS[rng.integers(0, 15, B)].astype(np.float32)
    return x0, sig, eps, v


def _dev(*arrs):
    return [torch.from_numpy(a).cuda() for a in arrs]


def _oracle(p, x0, sig, eps, v):
    """fp64 per-example loss, score and Hessian term v.J_s v of the reference's reverse-over-reverse formulation."""
    t = lambda a: torch.from_numpy(a).double()
    model = lambda a, s: O.dense_ncsn(p, a, s, **KW)
    per, _, hess = R.ssm_loss_tensors(model, t(x0), t(sig), t(eps), t(v), "none")
    us = t(sig).reshape(-1, 1)
    score = model(t(x0) + t(eps) * us, us)
    return per, score, hess


@pytest.mark.parametrize("continuous", [False, True])
def test_ssm_draws_match_jax_restatement(lib, continuous):
    eng, _ = _engine(64)
    eng.dsm_setup(SIGMAS)
    key = tf.prng_key(3)
    used, eps, v, lab = eng.ssm_draws((int(key[0]), int(key[1])), 64, want_labels=True, continuous_noise=continuous)
    rl, ru, re, rv = R.ssm_draws(key, (64, C), SIGMAS, continuous)
    np.testing.assert_array_equal(lab.cpu().numpy(), rl)
    np.testing.assert_array_equal(used.cpu().numpy(), ru)
    np.testing.assert_array_equal(v.cpu().numpy(), rv)
    np.testing.assert_allclose(eps.cpu().numpy(), re, rtol=2e-5, atol=2e-6)
    u2, e2, v2 = eng.ssm_draws((int(key[0]), int(key[1])), 16, global_batch=64, first_row=16, continuous_noise=continuous)
    assert torch.equal(u2, used[16:32]) and torch.equal(e2, eps[16:32]) and torch.equal(v2, v[16:32])


def test_strict_jvp_matches_fp64_oracle(lib):
    x0, sig, eps, v = _inputs(8, 0)
    errs = {}
    for precision in ("bf16x3", "bf16"):
        eng, flat = _engine(8, precision=precision)
        loss, score, hvp = eng.ssm_loss(*_dev(x0, sig, eps, v), want_terms=True)
        p = params_torch(eng, flat, torch.float64)
        per, ref_score, ref_hess = _oracle(p, x0, sig, eps, v)
        errs[precision] = (rel_l2(score, ref_score), rel_l2(hvp, ref_hess), rel_l2(loss, per))
    print("ssm strict rel-L2 (score, hessian, loss):", errs)
    # measured on an H100: bf16x3 7.0e-6 / 3.3e-6 / 6.1e-6; bf16 3.9e-3 / 2.0e-3 / 1.1e-3
    s3, h3, l3 = errs["bf16x3"]
    s1, h1, _ = errs["bf16"]
    assert s3 <= 1e-4 and h3 <= 1e-4 and l3 <= 1e-4
    assert s1 >= 10 * s3 and h1 >= 10 * h3


def test_ssm_loss_and_gradients(lib):
    eng, flat = _engine(8, training=True)
    eng.init_train_state()
    x0, sig, eps, v = _inputs(8, 1)
    loss, score, hvp = eng.ssm_loss(*_dev(x0, sig, eps, v), want_terms=True)
    eng.compute_ssm_grads(*_dev(x0, sig, eps, v))
    torch.cuda.synchronize()
    p = {k: t.requires_grad_(True) for k, t in params_torch(eng, flat, torch.float64).items()}
    per, ref_score, ref_hess = _oracle(p, x0, sig, eps, v)
    per.mean().backward()
    e_score, e_hess, e_loss = rel_l2(score, ref_score), rel_l2(hvp, ref_hess), rel_l2(loss, per)
    e_mean = abs(float(eng.loss_mean) - float(per.mean())) / abs(float(per.mean()))
    got = eng.flat_to_dict(eng.grads)
    tot = sum(float((t.grad ** 2).sum()) for t in p.values())
    dot = sum(float((torch.from_numpy(got[k]).double() * t.grad).sum()) for k, t in p.items())
    nn_ = sum(float((torch.from_numpy(got[k]).double() ** 2).sum()) for k in p)
    cos, ratio = dot / np.sqrt(nn_ * tot), np.sqrt(nn_ / tot)
    per_tensor = {k: rel_l2(torch.from_numpy(got[k]), t.grad) for k, t in p.items()
                  if float((t.grad ** 2).sum()) >= 1e-4 * tot}
    worst = max(per_tensor.items(), key=lambda kv: kv[1])
    print(f"ssm bf16: score {e_score:.3e} hessian {e_hess:.3e} loss {e_loss:.3e} mean-loss {e_mean:.3e} "
          f"grad cos {cos:.6f} norm ratio {ratio:.5f} worst tensor {worst}")
    # measured on an H100: 3.6e-3, 5.6e-4, 5.9e-4, 6.5e-5; cos 0.999986, norm ratio 1.00004, worst tensor 6.7e-3
    assert e_score < 8e-3 and e_hess < 1.2e-3 and e_loss < 1.2e-3 and e_mean < 2e-4
    assert cos > 0.99997 and abs(ratio - 1) < 1e-4
    assert worst[1] < 1.4e-2, worst


def test_ssm_grads_graph_replay(lib):
    eng, _ = _engine(16, training=True)
    eng.init_train_state()
    a = _dev(*_inputs(16, 2))
    b = _dev(*_inputs(16, 3))
    stream = torch.cuda.Stream()
    outs = []
    with torch.cuda.stream(stream):
        for inp in (a, a, a, b):        # eager (first use), capture + replay, replay, replay with new tensors
            eng.compute_ssm_grads(*inp)
            outs.append((eng.grads.clone(), eng.loss_sum.clone()))
    stream.synchronize()
    for g, l in outs[1:3]:
        torch.testing.assert_close(g, outs[0][0], rtol=1e-4, atol=1e-7)   # atomics ordering only
        assert torch.equal(l, outs[0][1])
    eng.compute_ssm_grads(*b)            # legacy default stream: not capturable, eager
    torch.cuda.synchronize()
    torch.testing.assert_close(outs[3][0], eng.grads, rtol=1e-4, atol=1e-7)
    assert torch.equal(outs[3][1], eng.loss_sum)


def test_ssm_training_lowers_the_loss(lib):
    eng, _ = _engine(32, training=True)
    eng.init_train_state()
    inp = _dev(*_inputs(32, 4))
    before = float(eng.ssm_loss(*inp).mean())
    for _ in range(10):
        eng.compute_ssm_grads(*inp)
        eng.apply_grads(1e-3)
    after = float(eng.ssm_loss(*inp).mean())
    assert np.isfinite(before) and np.isfinite(after) and np.isfinite(float(eng.grad_norm))
    assert after < before, (before, after)


def test_sliced_score_matching_loss_matches_oracle(lib):
    from smd_b200 import ncsn, nn
    from smd_b200.losses import sliced_score_matching_loss
    eng, flat = _engine(16)
    module = ncsn.DenseNCSN.partial(**KW)
    model = nn.Model(module, nn.ParamArena(module, (C,), flat))
    x0 = np.random.default_rng(5).uniform(-1, 1, (16, C)).astype(np.float32)
    key = tf.prng_key(9)
    for continuous in (False, True):
        got = float(sliced_score_matching_loss(x0, model, SIGMAS, key, continuous, "mean"))
        _, used, eps, v = R.ssm_draws(key, (16, C), SIGMAS, continuous)
        per, _, _ = _oracle(params_torch(eng, flat, torch.float64), x0, used, eps, v)
        err = abs(got - float(per.mean())) / float(per.abs().mean())
        print(f"ssm objective (continuous={continuous}): rel err {err:.3e}")
        assert err < 1e-3, (continuous, got, float(per.mean()))   # measured on an H100: 3.9e-4 / 1.5e-4
    with pytest.raises(ValueError):
        sliced_score_matching_loss(x0, model, SIGMAS, key, False, "median")


def test_train_ssm_and_sample_cli(tmp_path):
    cfg = tmp_path / "ncsn-ssm.cfg"
    cfg.write_text(textwrap.dedent(f"""\
        --loss=ssm
        --sampling=ald
        --architecture=DenseNCSN
        --num_layers=2
        --mlp_dims=512
        --num_sigmas=4
        --ld_steps=2
        --ld_epsilon=2e-6
        --problem=vae
        --ema=True
        --nosnapshot_sampling
        --data_shape=512
        --batch_size=16
        --learning_rate=1e-3
        --max_steps=4
        --snapshot_freq=2
        --logging_freq=1
        --synthetic
        --synthetic_examples=64
        --model_dir={tmp_path / 'run'}
        """))
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "smd_b200.train_ncsn", f"--flagfile={cfg}"], capture_output=True,
                       text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    from smd_b200 import checkpoints
    assert checkpoints.list_checkpoints(str(tmp_path / "run")) == ["checkpoint_0", "checkpoint_1"]
    r = subprocess.run([sys.executable, "-m", "smd_b200.sample_ncsn", f"--flagfile={cfg}", "--sample_size=8"],
                       capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    import pickle
    gen = pickle.load(open(tmp_path / "run" / "samples" / "ncsn" / "generated.pkl", "rb"))
    assert gen.shape == (8, 512) and np.isfinite(gen).all()
