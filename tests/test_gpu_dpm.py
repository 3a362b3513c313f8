"""The DPM-Solver++ chain on the device (smd_dpm_setup / smd_dpm_sample): short chains of orders 1-3 against the
float64 restatement on the bf16-emulating oracle networks (and the strict mode against the float64 networks), order 1
against the DDIM eta = 0 chain, graph replay, sharding, launch counts, the chain-invalidation rules and the command
lines."""
import json
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from oracle import threefry as tf
from tests import dpm_reference as R
from tests.test_gpu_ddim import BETAS, FLAGS, _apply, _engine, _inputs, _load, _run
from tests.util import rel_l2

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def device_chain(eng, steps, order, key, init, ix=None, im=None, use_graph=True, shard=(0, 0)):
    x = init.clone()
    coll = torch.zeros((41,) + tuple(x.shape), device="cuda")
    coll[0] = x * (1 - im) + ix * im if ix is not None else x
    mets = torch.zeros((4, len(steps)), device="cuda")
    eng.dpm_setup(BETAS, steps, order, key=(int(key[0]), int(key[1])))
    eng.set_sampler_shard(*shard)
    eng.dpm_sample(x, infill_x=ix, infill_mask=im, collection=coll, metrics=mets, use_graph=use_graph)
    eng.set_sampler_shard(0, 0)
    torch.cuda.synchronize()
    return x, coll, mets


# --------------------------------------------------------------------------------------------- against the oracle
SHORT = [
    # case, steps, order, infill
    ("t32", [999], 2, False),                   # one step: first order, x' = m0
    ("t32", [0, 400, 700, 999], 1, True),
    ("t32", [0, 250, 500, 750, 999], 2, False),
    ("t64", [120, 400, 650, 870, 990], 3, False),
    ("t64", [0, 250, 600, 999], 2, True),
    ("t128", [0, 200, 450, 700, 999], 3, True),
    ("dense", [0, 300, 600, 999], 3, True),
    ("dense", [10, 20, 500, 995], 2, False),
]


@pytest.mark.parametrize("case,steps,order,infill", SHORT)
def test_short_chain_matches_bf16_oracle(lib, case, steps, order, infill):
    eng, flat, shape = _engine(case)
    init, samples, masks = _inputs(shape, 4, seed=len(steps) + order)
    ix, im = (samples, masks) if infill else (None, None)
    key = tf.prng_key(11)
    x, coll, mets = device_chain(eng, steps, order, key, init, ix, im)
    rx, rc, rm = R.dpm_chain(_apply(eng, flat), BETAS, steps, order, init.cpu(), key,
                             None if ix is None else ix.cpu(), None if im is None else im.cpu())
    # the x0 estimate multiplies the network's bf16 error by sqrt((1-a)/a), as in the DDIM chain's test
    assert rel_l2(x, rx) < 3e-2
    for r in range(1, 41):
        if rc[r].abs().sum() > 0:
            assert rel_l2(coll[r], rc[r]) < 3e-2, r
    np.testing.assert_allclose(mets.cpu().numpy(), rm.numpy(), rtol=2e-2, atol=1e-6)
    if infill and steps[0] == 0:   # the held entries end at the template of the last step
        assert torch.equal(x[masks > 0], samples[masks > 0])


@pytest.mark.parametrize("order", [2, 3])
def test_strict_chain_matches_float64(lib, order):
    eng, flat, shape = _engine("t32", precision="bf16x3")
    init, samples, masks = _inputs(shape, 4, seed=5)
    key = tf.prng_key(2)
    steps = [0, 200, 450, 700, 999]
    x, _, mets = device_chain(eng, steps, order, key, init, samples, masks)
    rx, _, rm = R.dpm_chain(_apply(eng, flat, torch.float64, emulate_bf16=False), BETAS, steps, order, init.cpu(),
                            key, samples.cpu(), masks.cpu())
    err = rel_l2(x, rx)
    assert err < 1e-4, err
    np.testing.assert_allclose(mets.cpu().numpy(), rm.numpy(), rtol=1e-3, atol=1e-7)


# ------------------------------------------------------------------------------------ order 1 is DDIM at eta = 0
@pytest.mark.parametrize("infill", [False, True])
def test_order_one_equals_the_ddim_eta_zero_chain(lib, infill):
    """Order 1 is the DDIM eta = 0 step in exact arithmetic; the two kernels round differently (c_x x + c_0 m0
    against sqrt(a') x0 + c_dir eps'), so agreement is measured on a strict plan, where a last-bit difference
    cannot flip a bf16 rounding of the network input."""
    eng, _, shape = _engine("t32", batch=8, precision="bf16x3")
    init, samples, masks = _inputs(shape, 8, seed=21)
    ix, im = (samples, masks) if infill else (None, None)
    key = tf.prng_key(7)
    steps = np.arange(0, 1000, 50)
    x1, c1, m1 = device_chain(eng, steps, 1, key, init, ix, im)
    x2 = init.clone()
    c2 = torch.zeros_like(c1)
    c2[0] = c1[0]
    m2 = torch.zeros_like(m1)
    eng.ddim_setup(BETAS, steps, 0.0, key=(int(key[0]), int(key[1])))
    eng.ddim_sample(x2, infill_x=ix, infill_mask=im, collection=c2, metrics=m2)
    torch.cuda.synchronize()
    state_err = rel_l2(x1, x2)
    coll_err = max(rel_l2(c1[r], c2[r]) for r in range(41))
    print(f"order 1 vs DDIM eta = 0: state {state_err:.3e}, collection {coll_err:.3e}")
    # measured on an H100: state 4.0e-6 / 3.6e-6, collection 4.0e-6 / 3.6e-6 (without / with infill)
    assert state_err < 8e-6 and coll_err < 8e-6, (state_err, coll_err)
    torch.testing.assert_close(m1, m2, rtol=1e-4, atol=1e-6)
    assert torch.equal(m1[2], m2[2])
    if infill:
        assert torch.equal(x1[masks > 0], x2[masks > 0])


# ----------------------------------------------------------------------------------------------- device behaviour
@pytest.mark.parametrize("case,order", [("t32", 3), ("dense", 2)])
def test_graph_replay_equals_eager_and_repeats(lib, case, order):
    eng, _, shape = _engine(case)
    init, samples, masks = _inputs(shape, 4, seed=8)
    steps = [0, 200, 450, 700, 999]
    key = tf.prng_key(4)
    e = device_chain(eng, steps, order, key, init, samples, masks, use_graph=False)
    g1 = device_chain(eng, steps, order, key, init, samples, masks)
    x = init.clone()                                   # same buffers twice: the captured graph is replayed
    coll = torch.zeros_like(g1[1])
    mets = torch.zeros_like(g1[2])
    for _ in range(2):
        x.copy_(init)
        coll.zero_()
        coll[0] = x * (1 - masks) + samples * masks
        eng.dpm_sample(x, infill_x=samples, infill_mask=masks, collection=coll, metrics=mets)
        torch.cuda.synchronize()
        assert torch.equal(x, e[0]) and torch.equal(coll, e[1])
    assert torch.equal(g1[0], e[0]) and torch.equal(g1[1], e[1])
    # the metrics are batch means summed with atomics across blocks: equal up to the order of the sum
    torch.testing.assert_close(g1[2], e[2], rtol=1e-6, atol=0)
    torch.testing.assert_close(mets, e[2], rtol=1e-6, atol=0)


@pytest.mark.parametrize("case", ["t32", "dense"])
def test_two_shards_gather_the_whole_batch(lib, case):
    eng, _, shape = _engine(case, batch=8)
    init, samples, masks = _inputs(shape, 8, seed=9)
    steps = [0, 250, 500, 750, 999]
    key = tf.prng_key(5)
    fx, fc, fm = device_chain(eng, steps, 3, key, init, samples, masks)
    xs, cs, ms = [], [], []
    for r in range(2):
        sl = slice(4 * r, 4 * r + 4)
        x, c, m = device_chain(eng, steps, 3, key, init[sl].contiguous(), samples[sl].contiguous(),
                               masks[sl].contiguous(), shard=(4 * r, 8))
        xs.append(x)
        cs.append(c)
        ms.append(m)
    assert torch.equal(torch.cat(xs), fx)
    assert torch.equal(torch.cat(cs, dim=1), fc)
    w = ms[0] * 0.5 + ms[1] * 0.5
    w[2] = ms[0][2]
    torch.testing.assert_close(w, fm, rtol=1e-5, atol=0)


def test_launches_per_step_equal_the_ddim_chain(lib):
    eng, _, shape = _engine("t32")
    init = _inputs(shape, 4)[0]
    steps = np.arange(0, 1000, 50)
    per = {}
    for name in ("ddim", "dpm2", "dpm3"):
        for _ in range(2):                             # the second call replays the captured step
            x = init.clone()
            if name == "ddim":
                eng.ddim_setup(BETAS, steps, 0.0)
                before = eng.launch_count()
                eng.ddim_sample(x)
            else:
                eng.dpm_setup(BETAS, steps, int(name[-1]))
                before = eng.launch_count()
                eng.dpm_sample(x)
            torch.cuda.synchronize()
            per[name] = (eng.launch_count() - before) / len(steps)
    assert per["dpm2"] == per["ddim"] and per["dpm3"] == per["ddim"], per


def test_setups_invalidate_each_other(lib):
    from smd_b200 import lib as L
    eng, _, shape = _engine("t32")
    x = _inputs(shape, 4)[0]
    steps = [0, 500, 999]
    others = {
        "smd_sampler_setup": lambda: eng.sampler_setup(BETAS, key=(0, 1)),
        "smd_ddim_setup": lambda: eng.ddim_setup(BETAS, steps, 0.0),
        "smd_ddim_encode_setup": lambda: eng.ddim_encode_setup(BETAS, steps),
        "smd_langevin_setup": lambda: eng.langevin_setup(np.asarray([1.0, 0.1], np.float32), 2, 1e-5, "ald"),
    }
    runs = {
        "smd_sampler_setup": lambda: eng.sample(x.clone(), steps=3),
        "smd_ddim_setup": lambda: eng.ddim_sample(x.clone()),
        "smd_ddim_encode_setup": lambda: eng.ddim_encode(x.clone()),
        "smd_langevin_setup": lambda: eng.langevin_sample(x.clone()),
    }
    for name, setup in others.items():
        eng.dpm_setup(BETAS, steps, 2)
        eng.dpm_sample(x.clone())
        with pytest.raises(L.SmdError, match=name):   # the DPM setup invalidates the other chain
            runs[name]()
        setup()
        runs[name]()
        with pytest.raises(L.SmdError, match="smd_dpm_setup"):
            eng.dpm_sample(x.clone())
    eng.dpm_setup(BETAS, steps, 3)
    with pytest.raises(ValueError, match="n out of range"):
        eng.dpm_sample(torch.zeros((16,) + shape, device="cuda"))
    for half in (dict(infill_x=x), dict(infill_mask=torch.ones_like(x))):
        with pytest.raises(ValueError, match="infill_x and infill_mask go together"):
            eng.dpm_sample(x.clone(), **half)
    with pytest.raises(ValueError, match="order"):
        eng.dpm_setup(BETAS, steps, 4)
    eng.dpm_sample(x.clone())                          # a rejected setup leaves the previous chain in place
    # a null history with order > 1
    with pytest.raises(ValueError, match="history"):
        L.check(eng.lib.smd_dpm_sample(eng._plan, eng.params.data_ptr(), x.data_ptr(), 4, None, None, None, None,
                                       None, 1, eng._stream()))
    eng.dpm_setup(BETAS, steps, 1)                     # order 1 needs none
    L.check(eng.lib.smd_dpm_sample(eng._plan, eng.params.data_ptr(), x.clone().data_ptr(), 4, None, None, None,
                                   None, None, 1, eng._stream()))
    torch.cuda.synchronize()


def test_initial_draw_is_normal():
    from smd_b200 import train_ncsn
    torch.testing.assert_close(train_ncsn.initial_draw((0, 3), (4, 5), "dpm"),
                               train_ncsn.initial_draw((0, 3), (4, 5), "ddpm"), rtol=0, atol=0)


# ---------------------------------------------------------------------------------------------- command lines
def test_command_lines(lib, tmp_path):
    cfg = tmp_path / "dpm.cfg"
    flags = FLAGS.replace("--sampling=ddim", "--sampling=dpm").replace("--ddim_steps=10", "--dpm_steps=10") \
                 .replace("--ddim_eta=0.5", "--dpm_order=3")
    cfg.write_text(textwrap.dedent(flags).format(run=tmp_path / "run"))
    run = tmp_path / "run"
    _run("smd_b200.train_ncsn", cfg)                      # --snapshot_sampling (the default) with the dpm chain
    fake = _load(run / "samples" / "fake" / "2.pkl")
    assert fake.shape == (16, 32, 42) and np.isfinite(fake).all()
    ld = np.load(run / "sampling_epoch0" / "ld_metrics.npz")
    assert ld["slope"].shape == (10, 1) and np.isfinite(ld["slope"]).all()
    assert json.loads(open(run / "samples" / "metrics.jsonl").readline())["global_step"] == 2

    _run("smd_b200.sample_ncsn", cfg, "--sample_size=16", "--compute_metrics", "--dpm_order=2")
    out = run / "samples" / "ncsn"
    gen, coll = _load(out / "generated.pkl"), _load(out / "collection.pkl")
    assert gen.shape == (16, 32, 42) and coll.shape == (41, 16, 32, 42) and np.isfinite(gen).all()
    res = json.load(open(out / "metrics.json"))
    assert np.isfinite(res["ncsn"]["19"]["frechet_distance"])

    # infill: the last step sits at t = 0, whose template is the held latents themselves
    _run("smd_b200.sample_ncsn", cfg, "--sample_size=8", "--infill", "--sampling_dir=infill",
         "--dpm_schedule=quadratic")
    out = run / "infill" / "ncsn"
    gen, real = _load(out / "generated.pkl"), _load(out / "real.pkl")
    np.testing.assert_allclose(gen[:, :8], real[:, :8], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(gen[:, -8:], real[:, -8:], rtol=1e-5, atol=1e-5)
    assert np.abs(gen[:, 8:-8] - real[:, 8:-8]).mean() > 1e-2

    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "smd_b200.sample_ncsn", f"--flagfile={cfg}", "--sample_size=8",
                        "--interpolate", "--sampling_dir=interp"], capture_output=True, text=True, timeout=600,
                       env=env, cwd=ROOT)
    assert r.returncode != 0 and "ValueError" in r.stderr and "--sampling=dpm" in r.stderr
