"""The DDIM encoder on the device (smd_ddim_encode_setup / smd_ddim_encode): short chains against the float64
restatement on the bf16-emulating oracle networks (and the strict mode against the float64 networks), exact
invertibility with a constant network, graph replay, sharding, the generator path, launch counts, the
chain-invalidation rules, the sample_ncsn command line and the kernel's SASS."""
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
from smd_b200 import ebm_utils
from tests import ddim_encode_reference as RE
from tests import ddim_reference as R
from tests.test_sass_evidence import _get, table  # noqa: F401  (module-scoped fixture: one cuobjdump pass)
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
U32 = 2.0 ** -24                                       # unit roundoff of float32


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


def _data(shape, n, seed=0, lim=1.0):
    g = np.random.default_rng(seed)
    return torch.from_numpy(g.uniform(-lim, lim, (n,) + shape).astype(np.float32)).cuda()


def encode(eng, steps, x0, use_graph=True, betas=BETAS):
    x = x0.clone()
    eng.ddim_encode_setup(betas, steps)
    eng.ddim_encode(x, use_graph=use_graph)
    torch.cuda.synchronize()
    return x


# --------------------------------------------------------------------------------------------- against the oracle
SHORT = [
    # case, steps
    ("t32", [999]),                             # one step: a = 1, x0 = x
    ("t32", [0, 400, 999]),
    ("t64", [120, 530, 870]),
    ("t128", [0, 333, 666, 999]),
    ("dense", [0, 400, 999]),
    ("dense", [10, 20, 995]),
]


@pytest.mark.parametrize("case,steps", SHORT)
def test_short_chain_matches_bf16_oracle(lib, case, steps):
    eng, flat, shape = _engine(case)
    x0 = _data(shape, 4, seed=len(steps))
    got = encode(eng, steps, x0)
    want = RE.encode_chain(_apply(eng, flat), BETAS, steps, x0.cpu())
    err = rel_l2(got, want)
    print(f"encode {case} {steps}: rel-L2 {err:.3e}")
    # the network's bf16 error enters each step through eps, with weight sqrt(1-a') - sqrt(a' (1-a) / a): measured up
    # to 4.1e-3 on an H100 (t128), bounded at 3x that; the strict test below pins the chain's own arithmetic
    assert err < 1.2e-2


def test_strict_chain_matches_float64(lib):
    eng, flat, shape = _engine("t32", precision="bf16x3")
    x0 = _data(shape, 4, seed=5)
    steps = [0, 300, 700, 999]
    got = encode(eng, steps, x0)
    want = RE.encode_chain(_apply(eng, flat, torch.float64, emulate_bf16=False), BETAS, steps, x0.cpu())
    err = rel_l2(got, want)
    print(f"encode strict: rel-L2 {err:.3e}")
    assert err < 1e-4                     # measured 1.3e-5 on an H100


# -------------------------------------------------------------------------------------------------- invertibility
def _constant_network(eng, flat, c):
    """Zero output kernel and bias c: the network returns eps = c (per channel) exactly in every precision."""
    d = eng.flat_to_dict(flat)
    d["out.kernel"] = np.zeros_like(d["out.kernel"])
    d["out.bias"] = np.asarray(c, np.float32).reshape(d["out.bias"].shape)
    eng.set_params(eng.dict_to_flat(d))


@pytest.mark.parametrize("K", [1, 10, 1000])
@pytest.mark.parametrize("case", ["t32", "dense"])
def test_constant_network_encodes_and_decodes_exactly(lib, case, K):
    """eps = c: every x0 estimate of the encoder is x0 itself, so the code is sqrt(a_{K-1}) x0 + sqrt(1 - a_{K-1}) c,
    and the DDIM chain at eta = 0 on it returns x0.  Only float32 rounding separates the device from these values."""
    eng, flat, shape = _engine(case)
    C = shape[-1]
    c = np.random.default_rng(K).uniform(-0.5, 0.5, C).astype(np.float32)
    _constant_network(eng, flat, c)
    x0 = _data(shape, 4, seed=K, lim=0.9)
    steps = ebm_utils.ddim_schedule(1000, K)
    code = encode(eng, steps, x0)
    ab = R.alpha_bar(BETAS).astype(np.float64)[steps]
    ct = torch.from_numpy(c.astype(np.float64))
    want = np.sqrt(ab[-1]) * x0.double().cpu() + np.sqrt(1 - ab[-1]) * ct
    # each encoder step rounds a few operations on values below S = max|x0| + max|c| and damps earlier errors by
    # sqrt(a'/a) <= 1: at most 8 u S per step
    S = 0.9 + float(np.abs(c).max())
    enc_tol = 8 * U32 * S * K
    enc_err = float((code.double().cpu() - want).abs().max())
    # the decoder amplifies an error of x at level a_i by sqrt(1/a_i) on its way to a = 1 (sqrt(a'/a) per step)
    dec_tol = enc_tol / np.sqrt(ab[-1]) + 8 * U32 * S * float(np.sum(1 / np.sqrt(ab)))
    x = code.clone()
    eng.ddim_setup(BETAS, steps, 0.0, key=(0, 1))
    eng.ddim_sample(x)
    torch.cuda.synchronize()
    dec_err = float((x - x0).abs().max())
    # measured on an H100: encode 3.9e-8 / 8.1e-8 / 7.1e-7 and decode 1.4e-5 / 1.4e-5 / 1.1e-4 at K = 1 / 10 / 1000
    print(f"invertibility {case} K={K}: encode {enc_err:.3e} (bound {enc_tol:.3e}), decode {dec_err:.3e} "
          f"(bound {dec_tol:.3e})")
    assert enc_err <= enc_tol
    assert dec_err <= dec_tol


# ----------------------------------------------------------------------------------------------- device behaviour
@pytest.mark.parametrize("case", ["t32", "dense"])
def test_graph_replay_equals_eager_and_repeats(lib, case):
    eng, _, shape = _engine(case)
    x0 = _data(shape, 4, seed=8)
    steps = [0, 200, 450, 700, 999]
    e = encode(eng, steps, x0, use_graph=False)
    g = encode(eng, steps, x0)
    assert torch.equal(g, e)
    x = x0.clone()                                     # same buffer twice: the captured graph is replayed
    for _ in range(2):
        x.copy_(x0)
        eng.ddim_encode(x)
        torch.cuda.synchronize()
        assert torch.equal(x, e)
    assert not torch.equal(e, x0)


@pytest.mark.parametrize("case", ["t32", "dense"])
def test_two_halves_equal_the_whole_batch(lib, case):
    eng, _, shape = _engine(case, batch=8)
    x0 = _data(shape, 8, seed=9)
    steps = [0, 250, 500, 999]
    whole = encode(eng, steps, x0)
    halves = [encode(eng, steps, x0[4 * r:4 * r + 4].contiguous()) for r in range(2)]
    assert torch.equal(torch.cat(halves), whole)


def test_more_levels_than_film_rows_runs_the_generator(lib):
    from smd_b200 import Engine, ModelConfig
    eng, flat, shape = _engine("t32")
    small = Engine(ModelConfig(**CASES["t32"][0]), max_batch=4, sampler_T=3)
    small.set_params(flat)
    x0 = _data(shape, 4, seed=1)
    steps = [0, 200, 450, 700, 999]
    a = encode(eng, steps, x0)
    b = encode(small, steps, x0)
    c = encode(small, steps, x0, use_graph=False)
    assert torch.equal(b, c)
    # the table and the generator compute the same FiLM rows in a different launch shape
    assert rel_l2(b, a) < 1e-3


def test_launches_per_step_equal_the_ddim_chain(lib):
    eng, _, shape = _engine("t32")
    x0 = _data(shape, 4)
    steps = np.arange(0, 1000, 50)
    per = {}
    for name in ("ddim", "encode"):
        for _ in range(2):                             # the second call replays the captured step
            x = x0.clone()
            if name == "ddim":
                eng.ddim_setup(BETAS, steps, 0.0, key=(0, 1))
                before = eng.launch_count()
                eng.ddim_sample(x)
            else:
                eng.ddim_encode_setup(BETAS, steps)
                before = eng.launch_count()
                eng.ddim_encode(x)
            torch.cuda.synchronize()
            per[name] = (eng.launch_count() - before) / len(steps)
    assert per["encode"] == per["ddim"], per


def test_setups_invalidate_each_other(lib):
    from smd_b200 import lib as L
    eng, _, shape = _engine("t32")
    x = _data(shape, 4)
    steps = [0, 500, 999]
    eng.ddim_encode_setup(BETAS, steps)
    eng.ddim_encode(x.clone())
    for other in (lambda: eng.sampler_setup(BETAS, key=(0, 1)), lambda: eng.ddim_setup(BETAS, steps, 0.0),
                  lambda: eng.langevin_setup(np.asarray([1.0, 0.1], np.float32), 2, 1e-5, "ald")):
        other()
        with pytest.raises(L.SmdError, match="smd_ddim_encode_setup"):
            eng.ddim_encode(x.clone())
        eng.ddim_encode_setup(BETAS, steps)
        eng.ddim_encode(x.clone())
    with pytest.raises(L.SmdError, match="smd_sampler_setup"):
        eng.sample(x.clone(), steps=3)
    with pytest.raises(L.SmdError, match="smd_sampler_setup"):
        eng.reverse_step(x.clone(), 2)
    with pytest.raises(L.SmdError, match="smd_ddim_setup"):
        eng.ddim_sample(x.clone())
    with pytest.raises(L.SmdError, match="smd_langevin_setup"):
        eng.langevin_sample(x.clone())
    with pytest.raises(ValueError, match="n out of range"):
        eng.ddim_encode(torch.zeros((16,) + shape, device="cuda"))
    with pytest.raises(ValueError, match="strictly increasing"):
        eng.ddim_encode_setup(BETAS, [5, 5])
    eng.ddim_encode(x.clone())                         # a rejected setup leaves the previous chain in place
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------- command line
FLAGS = """\
    --loss=ddpm
    --sampling=ddim
    --ddim_steps=10
    --ddim_eta=0
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
    --nosnapshot_sampling
    --synthetic
    --synthetic_examples=64
    --model_dir={run}
    """


def _run(module, cfg, *extra):
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", module, f"--flagfile={cfg}", *extra], capture_output=True, text=True,
                       timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    return r


def _load(path):
    with open(path, "rb") as f:
        return pickle.load(f)


def test_command_line(lib, tmp_path):
    cfg = tmp_path / "ddim.cfg"
    cfg.write_text(textwrap.dedent(FLAGS).format(run=tmp_path / "run"))
    run = tmp_path / "run"
    _run("smd_b200.train_ncsn", cfg)
    args = ("--sample_size=8", "--interpolate", "--sampling=ddim", "--interpolate_encoder=ddim", "--ddim_steps=10")
    gens = []
    for k in range(2):
        r = _run("smd_b200.sample_ncsn", cfg, *args, f"--sampling_dir=interp{k}")
        out = run / f"interp{k}" / "ncsn"
        gen, coll, real = _load(out / "generated.pkl"), _load(out / "collection.pkl"), _load(out / "real.pkl")
        assert gen.shape == (9, 8, 32, 42) and coll.shape == (9, 41, 8, 32, 42) and real.shape == (8, 32, 42)
        assert np.isfinite(gen).all() and np.isfinite(coll).all()
        rec = json.load(open(out / "reconstruction.json"))
        for key in ("start_mse", "start_max_abs", "goal_mse", "goal_max_abs"):
            assert np.isfinite(rec[key]) and rec[key] >= 0, rec
        assert rec["ddim_steps"] == 10 and "Reconstruction" in r.stderr
        gens.append(gen)
    np.testing.assert_array_equal(gens[0], gens[1])    # deterministic: a rerun writes the same interpolants
    assert gens[0].tobytes() == gens[1].tobytes()


# ---------------------------------------------------------------------------------------------------------- SASS
def test_ddim_encode_step_kernel_does_not_spill(table):  # noqa: F811
    found = _get(table, "ddim_encode_step_kernel")
    assert found
    for c in found:
        assert c.get("STL", 0) == 0 and c.get("LDL", 0) == 0, c
