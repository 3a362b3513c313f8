"""The DDIM chain on the device (smd_ddim_setup / smd_ddim_sample): short chains against the float64 restatement on
the bf16-emulating oracle networks (and the strict mode against the float64 networks), the full schedule at eta = 1
against smd_ddpm_sample, determinism at eta = 0, graph replay, sharding, launch counts, the chain-invalidation rules
and the command lines."""
import json
import os
import pickle
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from oracle import ddpm_oracle as O
from oracle import threefry as tf
from tests import ddim_reference as R
from tests.util import oracle_kwargs, params_torch, rel_l2

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CASES = {
    "t32": (dict(arch="TransformerDDPM", num_layers=1, num_mlp_layers=1, seq_len=32, channels=42), (32, 42)),
    "t64": (dict(arch="TransformerDDPM", num_layers=1, num_mlp_layers=1, seq_len=64, channels=42), (64, 42)),
    "t128": (dict(arch="TransformerDDPM", num_layers=1, num_mlp_layers=1, seq_len=128, channels=42), (128, 42)),
    "dense": (dict(arch="DenseDDPM", channels=512, num_layers=2), (512,)),
}
BETAS = O.create_noise_schedule(1e-4, 0.02, 1000, "linear")


def _engine(case, batch=4, seed=3, **kw):
    from smd_b200 import Engine, ModelConfig
    cfg, shape = CASES[case]
    eng = Engine(ModelConfig(**cfg), max_batch=batch, **kw)
    flat = eng.init_params(seed=seed, perturb=0.02)
    eng.set_params(flat)
    return eng, flat, shape


def _apply(eng, flat, dtype=torch.float32, emulate_bf16=True):
    p = params_torch(eng, flat, dtype)
    kw = oracle_kwargs(eng.cfg)
    return lambda a, c: O.model_apply(eng.cfg.arch, p, a.to(dtype), c.to(dtype), emulate_bf16=emulate_bf16, **kw)


def _inputs(shape, n, seed=0):
    g = np.random.default_rng(seed)
    init = torch.from_numpy(g.standard_normal((n,) + shape).astype(np.float32)).cuda()
    samples = torch.from_numpy(g.uniform(-1, 1, (n,) + shape).astype(np.float32)).cuda()
    masks = torch.zeros((n,) + shape, device="cuda")
    masks.view(n, -1)[:, : masks[0].numel() // 4] = 1
    return init, samples, masks


def device_chain(eng, steps, eta, key, init, ix=None, im=None, use_graph=True, shard=(0, 0), betas=BETAS):
    x = init.clone()
    coll = torch.zeros((41,) + tuple(x.shape), device="cuda")
    coll[0] = x * (1 - im) + ix * im if ix is not None else x
    mets = torch.zeros((4, len(steps)), device="cuda")
    eng.ddim_setup(betas, steps, eta, key=(int(key[0]), int(key[1])))
    eng.set_sampler_shard(*shard)
    eng.ddim_sample(x, infill_x=ix, infill_mask=im, collection=coll, metrics=mets, use_graph=use_graph)
    eng.set_sampler_shard(0, 0)
    torch.cuda.synchronize()
    return x, coll, mets


# --------------------------------------------------------------------------------------------- against the oracle
SHORT = [
    # case, steps, eta, infill
    ("t32", [999], 1.0, False),                 # one step: a' = 1
    ("t32", [0, 400, 999], 1.0, True),
    ("t64", [120, 530, 870], 0.0, False),
    ("t64", [0, 250, 999], 0.5, True),
    ("t128", [0, 333, 666, 999], 1.0, False),
    ("dense", [0, 400, 999], 1.0, True),
    ("dense", [10, 20, 995], 0.3, False),
]


@pytest.mark.parametrize("case,steps,eta,infill", SHORT)
def test_short_chain_matches_bf16_oracle(lib, case, steps, eta, infill):
    eng, flat, shape = _engine(case)
    init, samples, masks = _inputs(shape, 4, seed=len(steps))
    ix, im = (samples, masks) if infill else (None, None)
    key = tf.prng_key(11)
    x, coll, mets = device_chain(eng, steps, eta, key, init, ix, im)
    apply_fn = _apply(eng, flat)
    rx, rc, rm = R.ddim_chain(apply_fn, BETAS, steps, eta, init.cpu(), key,
                              None if ix is None else ix.cpu(), None if im is None else im.cpu())
    # the x0 estimate multiplies the network's bf16 error by sqrt((1-a)/a), about 160 at t = 999 of this schedule:
    # measured up to 1.6e-2 on an H100; the strict test below pins the chain's own arithmetic
    assert rel_l2(x, rx) < 3e-2
    for r in range(1, 41):
        if rc[r].abs().sum() > 0:
            assert rel_l2(coll[r], rc[r]) < 3e-2, r
    np.testing.assert_allclose(mets.cpu().numpy(), rm.numpy(), rtol=2e-2, atol=1e-6)
    if infill:   # the held entries end at the template of the last step
        t0 = steps[0]
        if t0 == 0:
            assert torch.equal(x[masks > 0], samples[masks > 0])


def test_strict_chain_matches_float64(lib):
    eng, flat, shape = _engine("t32", precision="bf16x3")
    init, samples, masks = _inputs(shape, 4, seed=5)
    key = tf.prng_key(2)
    steps = [0, 300, 700, 999]
    x, _, mets = device_chain(eng, steps, 1.0, key, init, samples, masks)
    rx, _, rm = R.ddim_chain(_apply(eng, flat, torch.float64, emulate_bf16=False), BETAS, steps, 1.0, init.cpu(), key,
                             samples.cpu(), masks.cpu())
    assert rel_l2(x, rx) < 1e-4           # measured 1.9e-5 on an H100
    np.testing.assert_allclose(mets.cpu().numpy(), rm.numpy(), rtol=1e-3, atol=1e-7)


# ----------------------------------------------------------------------------------- the full schedule at eta = 1
@pytest.mark.parametrize("infill", [False, True])
def test_full_schedule_eta_one_equals_ddpm_sample(lib, infill):
    """tau = 0..T-1, eta = 1 is diffusion_dynamics: the same keys, the same collection rows, the same step in exact
    arithmetic.  The two chains round differently (the DDPM coefficients mu1, mu2 against sqrt(a'), eps'), and a
    one-ulp change of x can flip the network's bf16 input rounding, so agreement is measured, not bitwise."""
    eng, _, shape = _engine("t32", batch=8)
    init, samples, masks = _inputs(shape, 8, seed=21)
    ix, im = (samples, masks) if infill else (None, None)
    key = tf.prng_key(7)
    x1 = init.clone()
    c1 = torch.zeros((41,) + tuple(x1.shape), device="cuda")
    c1[0] = x1 * (1 - im) + ix * im if infill else x1
    m1 = torch.zeros((4, 1000), device="cuda")
    eng.sampler_setup(BETAS, key=(int(key[0]), int(key[1])))
    eng.sample(x1, steps=1000, infill_x=ix, infill_mask=im, collection=c1, metrics=m1)
    x2, c2, m2 = device_chain(eng, np.arange(1000), 1.0, key, init, ix, im)
    state_err = rel_l2(x2, x1)
    coll_err = max(rel_l2(c2[r], c1[r]) for r in range(41))
    met_err = float(((m2 - m1).abs() / (m1.abs() + 1e-6)).max())
    # measured on an H100: state 3.9e-4 / 3.4e-4, collection 3.5e-4 / 3.0e-4, metrics 8.2e-4 / 2.4e-4 (without /
    # with infill)
    assert state_err < 8e-4 and coll_err < 7e-4, (state_err, coll_err)
    assert met_err < 1.6e-3, met_err
    assert torch.equal(m2[2], m1[2])                  # alpha_bar rows: the same float32 cumulative product
    if infill:
        assert torch.equal(x2[masks > 0], x1[masks > 0])


# ----------------------------------------------------------------------------------------------- device behaviour
def test_eta_zero_is_deterministic_across_keys(lib):
    eng, _, shape = _engine("t32")
    init = _inputs(shape, 4, seed=3)[0]
    steps = [0, 100, 300, 600, 999]
    a = device_chain(eng, steps, 0.0, (0, 1), init)
    b = device_chain(eng, steps, 0.0, (5, 99), init)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert (a[2][3] < 1e-4).all()                     # noise_norm: sqrt(0 + 1e-10)
    c = device_chain(eng, steps, 1.0, (0, 1), init)
    assert not torch.equal(a[0], c[0])


@pytest.mark.parametrize("case", ["t32", "dense"])
def test_graph_replay_equals_eager_and_repeats(lib, case):
    eng, _, shape = _engine(case)
    init, samples, masks = _inputs(shape, 4, seed=8)
    steps = [0, 200, 450, 700, 999]
    key = tf.prng_key(4)
    e = device_chain(eng, steps, 1.0, key, init, samples, masks, use_graph=False)
    g1 = device_chain(eng, steps, 1.0, key, init, samples, masks)
    x = init.clone()                                   # same buffers twice: the captured graph is replayed
    coll = torch.zeros_like(g1[1])
    mets = torch.zeros_like(g1[2])
    for _ in range(2):
        x.copy_(init)
        coll.zero_()
        coll[0] = x * (1 - masks) + samples * masks
        eng.ddim_sample(x, infill_x=samples, infill_mask=masks, collection=coll, metrics=mets)
        torch.cuda.synchronize()
        assert torch.equal(x, e[0]) and torch.equal(coll, e[1])
    assert torch.equal(g1[0], e[0]) and torch.equal(g1[1], e[1])
    # the metrics are batch means summed with atomics across blocks: equal up to the order of the sum
    torch.testing.assert_close(g1[2], e[2], rtol=1e-6, atol=0)
    torch.testing.assert_close(mets, e[2], rtol=1e-6, atol=0)


def test_more_levels_than_film_rows_runs_the_generator(lib):
    eng, flat, shape = _engine("t32")
    from smd_b200 import Engine, ModelConfig
    small = Engine(ModelConfig(**CASES["t32"][0]), max_batch=4, sampler_T=3)
    small.set_params(flat)
    init = _inputs(shape, 4, seed=1)[0]
    steps = [0, 200, 450, 700, 999]
    a = device_chain(eng, steps, 1.0, (0, 3), init)
    b = device_chain(small, steps, 1.0, (0, 3), init)
    c = device_chain(small, steps, 1.0, (0, 3), init, use_graph=False)
    assert torch.equal(b[0], c[0])
    assert rel_l2(b[0], a[0]) < 1e-3


@pytest.mark.parametrize("case", ["t32", "dense"])
def test_two_shards_gather_the_whole_batch(lib, case):
    eng, _, shape = _engine(case, batch=8)
    init, samples, masks = _inputs(shape, 8, seed=9)
    steps = [0, 250, 500, 999]
    key = tf.prng_key(5)
    fx, fc, fm = device_chain(eng, steps, 1.0, key, init, samples, masks)
    xs, cs, ms = [], [], []
    for r in range(2):
        sl = slice(4 * r, 4 * r + 4)
        x, c, m = device_chain(eng, steps, 1.0, key, init[sl].contiguous(), samples[sl].contiguous(),
                               masks[sl].contiguous(), shard=(4 * r, 8))
        xs.append(x)
        cs.append(c)
        ms.append(m)
    assert torch.equal(torch.cat(xs), fx)
    assert torch.equal(torch.cat(cs, dim=1), fc)
    w = ms[0] * 0.5 + ms[1] * 0.5
    w[2] = ms[0][2]
    torch.testing.assert_close(w, fm, rtol=1e-5, atol=0)


def test_launches_per_step_equal_the_ddpm_chain(lib):
    eng, _, shape = _engine("t32")
    init = _inputs(shape, 4)[0]
    key = (0, 1)
    per = {}
    for name in ("ddpm", "ddim"):
        for _ in range(2):                             # the second call replays the captured step
            x = init.clone()
            if name == "ddpm":
                eng.sampler_setup(BETAS, key=key)
                before = eng.launch_count()
                eng.sample(x, steps=20)
            else:
                eng.ddim_setup(BETAS, np.arange(0, 1000, 50), 1.0, key=key)
                before = eng.launch_count()
                eng.ddim_sample(x)
            torch.cuda.synchronize()
            per[name] = (eng.launch_count() - before) / 20
    assert per["ddim"] == per["ddpm"], per


def test_setups_invalidate_each_other(lib):
    from smd_b200 import lib as L
    eng, _, shape = _engine("t32")
    x = _inputs(shape, 4)[0]
    steps = [0, 500, 999]
    eng.ddim_setup(BETAS, steps, 0.0)
    eng.ddim_sample(x.clone())
    eng.sampler_setup(BETAS, key=(0, 1))
    with pytest.raises(L.SmdError, match="smd_ddim_setup"):
        eng.ddim_sample(x.clone())
    eng.ddim_setup(BETAS, steps, 0.0)
    with pytest.raises(L.SmdError, match="smd_sampler_setup"):
        eng.sample(x.clone(), steps=3)
    with pytest.raises(L.SmdError, match="smd_sampler_setup"):
        eng.reverse_step(x.clone(), 2)
    with pytest.raises(L.SmdError, match="smd_langevin_setup"):
        eng.langevin_sample(x.clone())
    eng.langevin_setup(np.asarray([1.0, 0.1], np.float32), 2, 1e-5, "ald")
    with pytest.raises(L.SmdError, match="smd_ddim_setup"):
        eng.ddim_sample(x.clone())
    eng.langevin_sample(x.clone())
    eng.ddim_setup(BETAS, steps, 0.0)
    with pytest.raises(ValueError, match="n out of range"):
        eng.ddim_sample(torch.zeros((16,) + shape, device="cuda"))
    with pytest.raises(ValueError, match="strictly increasing"):
        eng.ddim_setup(BETAS, [5, 5], 0.0)
    eng.ddim_sample(x.clone())                         # a rejected setup leaves the previous chain in place
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------- command lines
FLAGS = """\
    --loss=ddpm
    --sampling=ddim
    --ddim_steps=10
    --ddim_eta=0.5
    --schedule_type=linear
    --sigma_begin=1e-4
    --sigma_end=0.02
    --num_sigmas=100
    --problem=vae
    --ema=False
    --architecture=TransformerDDPM
    --num_layers=1
    --num_mlp_layers=1
    --data_shape=32,42
    --batch_size=8
    --learning_rate=1e-3
    --max_steps=2
    --snapshot_freq=2
    --eval_samples=16
    --synthetic
    --synthetic_examples=64
    --model_dir={run}
    """


def _run(module, cfg, *extra):
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", module, f"--flagfile={cfg}", *extra], capture_output=True, text=True,
                       timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]


def _load(path):
    with open(path, "rb") as f:
        return pickle.load(f)


def test_command_lines(lib, tmp_path):
    cfg = tmp_path / "ddim.cfg"
    cfg.write_text(textwrap.dedent(FLAGS).format(run=tmp_path / "run"))
    run = tmp_path / "run"
    _run("smd_b200.train_ncsn", cfg)                      # --snapshot_sampling (the default) with the ddim chain
    fake = _load(run / "samples" / "fake" / "2.pkl")
    assert fake.shape == (16, 32, 42) and np.isfinite(fake).all()
    ld = np.load(run / "sampling_epoch0" / "ld_metrics.npz")
    assert ld["slope"].shape == (10, 1) and np.isfinite(ld["slope"]).all()
    assert json.loads(open(run / "samples" / "metrics.jsonl").readline())["global_step"] == 2

    _run("smd_b200.sample_ncsn", cfg, "--sample_size=16", "--compute_metrics")
    out = run / "samples" / "ncsn"
    gen, coll = _load(out / "generated.pkl"), _load(out / "collection.pkl")
    assert gen.shape == (16, 32, 42) and coll.shape == (41, 16, 32, 42) and np.isfinite(gen).all()
    res = json.load(open(out / "metrics.json"))
    assert np.isfinite(res["ncsn"]["19"]["frechet_distance"])

    # infill: the last step sits at t = 0, whose template is the held latents themselves
    _run("smd_b200.sample_ncsn", cfg, "--sample_size=8", "--infill", "--sampling_dir=infill", "--ddim_steps=10",
         "--ddim_schedule=quadratic")
    out = run / "infill" / "ncsn"
    gen, real = _load(out / "generated.pkl"), _load(out / "real.pkl")
    np.testing.assert_allclose(gen[:, :8], real[:, :8], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(gen[:, -8:], real[:, -8:], rtol=1e-5, atol=1e-5)
    assert np.abs(gen[:, 8:-8] - real[:, 8:-8]).mean() > 1e-2

    # the stochastic encoder of --interpolate is the ddpm chain's
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "smd_b200.sample_ncsn", f"--flagfile={cfg}", "--sample_size=8",
                        "--interpolate", "--sampling_dir=interp"], capture_output=True, text=True, timeout=600,
                       env=env, cwd=ROOT)
    assert r.returncode != 0 and "AssertionError" in r.stderr
