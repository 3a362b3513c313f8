"""Annealed / consistent Langevin dynamics as one device chain (smd_langevin_setup / smd_langevin_sample): bit-exact
against a host loop of Engine.forward + Engine.langevin_step with the reference's key schedule, close to the bf16
oracle, sharded over simulated ranks, graph re-capture, and the sample_ncsn command lines."""
import os
import pickle
import shutil
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from oracle import ddpm_oracle as O
from oracle import threefry as tf
from tests.util import params_torch, rel_l2

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CASES = {
    "dense": (dict(arch="DenseNCSN", channels=512, num_layers=2, mlp_dims=2048), (512,)),
    "t32": (dict(arch="TransformerDDPM", num_layers=1, num_mlp_layers=1, seq_len=32, channels=42), (32, 42)),
    "t64": (dict(arch="TransformerDDPM", num_layers=1, num_mlp_layers=1, seq_len=64, channels=42), (64, 42)),
}


def _engine(case, batch=8, seed=4, **kw):
    from smd_b200 import Engine, ModelConfig
    cfg, shape = CASES[case]
    eng = Engine(ModelConfig(**cfg), max_batch=batch, **kw)
    flat = eng.init_params(seed=seed, perturb=0.02)
    eng.set_params(flat)
    return eng, flat, shape


def _inputs(shape, n, seed=0):
    g = np.random.default_rng(seed)
    init = torch.from_numpy(g.uniform(-1.7, 1.7, (n,) + shape).astype(np.float32)).cuda()
    samples = torch.from_numpy(g.uniform(-1, 1, (n,) + shape).astype(np.float32)).cuda()
    masks = torch.zeros((n,) + shape, device="cuda")
    masks.view(n, -1)[:, : masks[0].numel() // 4] = 1
    return init, samples, masks


def host_chain(eng, kind, sigmas, T, epsilon, key, init, denoise, ix=None, im=None):
    """The per-step host loop the device chain replaces: Engine.forward + Engine.langevin_step per step, keys from
    the scan carry (split(rng, 3) / split(rng)), coefficients in float32 (utils/ebm_utils.py:89-271)."""
    from smd_b200 import ebm_utils, jrandom as random
    x = init.clone()
    sig = np.asarray(sigmas, np.float32)
    L = len(sig)
    T = T if kind == "ald" else 1
    coll = None
    if kind == "ald":
        coll = torch.zeros((101 + int(denoise),) + tuple(x.shape), device="cuda")
        coll[0] = x * (1 - im) + ix * im if ix is not None else x
    slot_of = ebm_utils._collection_slot_fn(L * T, 100)
    mets = torch.zeros((L, T, 4), device="cuda")
    sigma_dev = torch.empty((1,), device="cuda")
    grad = torch.empty_like(x)
    k = np.asarray(key, np.uint32)
    # squares as products: the reference's jitted `x ** 2` is x * x (numpy's float32 power can be an ulp away)
    r = np.float32(1) - np.float32(epsilon) / (sig[-1] * sig[-1])
    beta = np.sqrt(np.float32(1) - r * r).astype(np.float32)
    for si in range(L):
        s = np.float32(sig[si])
        q = s / np.float32(sig[-1])
        alpha = np.float32(epsilon) * (q * q)
        sigma_dev.copy_(torch.tensor([float(s)]))
        for i in range(T):
            if kind == "ald":
                k, sk, ik = random.split(k, 3)
                noise = float(np.sqrt(np.float32(2) * alpha))
            else:
                k, sk = random.split(k)
                ik = None
                noise = float(beta * (np.float32(sig[si + 1]) if si < L - 1 else np.float32(0)))
            eng.forward(x, sigma_dev, out=grad)
            slot = slot_of(si * T + i + 1) if coll is not None else -1
            if slot >= (coll.shape[0] if coll is not None else 0):
                slot = -1
            eng.langevin_step(x, grad, float(alpha), noise, step_key=sk, infill_x=ix, infill_mask=im,
                              infill_sigma=float(s), infill_key=ik, x_next=x,
                              collection_slot=coll[slot] if slot >= 0 else None, metrics4=mets[si, i])
    if denoise:
        sigma_dev.copy_(torch.tensor([float(sig[-1])]))
        eng.forward(x, sigma_dev, out=grad)
        eng.langevin_step(x, grad, float(np.float32(sig[-1]) * np.float32(sig[-1])), 0.0, x_next=x,
                          collection_slot=coll[-1] if coll is not None else None)
    return x, coll, mets.permute(2, 0, 1).contiguous()


def device_chain(eng, kind, sigmas, T, epsilon, key, init, denoise, ix=None, im=None, use_graph=True, shard=(0, 0)):
    x = init.clone()
    L = len(sigmas)
    T = T if kind == "ald" else 1
    coll = None
    if kind == "ald":
        coll = torch.zeros((101 + int(denoise),) + tuple(x.shape), device="cuda")
        coll[0] = x * (1 - im) + ix * im if ix is not None else x
    mets = torch.zeros((4, L, T), device="cuda")
    eng.langevin_setup(sigmas, T, epsilon, kind, key=(int(key[0]), int(key[1])))
    eng.set_sampler_shard(*shard)
    eng.langevin_sample(x, denoise=denoise, infill_x=ix, infill_mask=im, collection=coll, metrics=mets,
                        use_graph=use_graph)
    eng.set_sampler_shard(0, 0)
    return x, coll, mets


VARIANTS = [
    # case, kind, L, T, infill, denoise  (L*T below and above the 100 collection steps)
    ("dense", "ald", 3, 4, True, True),
    ("dense", "ald", 6, 20, False, False),
    ("dense", "cas", 8, 1, False, True),
    ("t32", "ald", 5, 25, True, False),
    ("t32", "ald", 3, 4, False, True),
    ("t32", "cas", 6, 1, False, False),
    ("t64", "ald", 4, 30, True, True),
    ("t64", "cas", 5, 1, False, True),
]


@pytest.mark.parametrize("case,kind,L,T,infill,denoise", VARIANTS)
def test_device_chain_equals_host_loop_bitwise(lib, case, kind, L, T, infill, denoise):
    eng, _, shape = _engine(case)
    init, samples, masks = _inputs(shape, 8, seed=L * 100 + T)
    ix, im = (samples, masks) if infill else (None, None)
    sigmas = O.create_noise_schedule(1.0, 0.05, L, "geometric")
    key = tf.prng_key(17 + L)
    ref_x, ref_c, ref_m = host_chain(eng, kind, sigmas, T, 2e-5, key, init, denoise, ix, im)
    for use_graph in (True, False):
        x, c, m = device_chain(eng, kind, sigmas, T, 2e-5, key, init, denoise, ix, im, use_graph=use_graph)
        torch.cuda.synchronize()
        assert torch.equal(x, ref_x), (use_graph, float((x - ref_x).abs().max()))
        if kind == "ald":
            assert torch.equal(c, ref_c), use_graph
        else:
            assert c is None
        torch.testing.assert_close(m, ref_m, rtol=1e-6, atol=0)
        assert torch.equal(m[2], ref_m[2])


def test_transformer_chain_matches_bf16_oracle(lib):
    """As test_gpu_ncsn's DenseNCSN chains, for TransformerDDPM (N, 32, 42) through ebm_utils."""
    from smd_b200 import ebm_utils, ncsn, nn
    eng, flat, shape = _engine("t32", batch=4)
    module = ncsn.TransformerDDPM.partial(num_layers=1, num_heads=8, num_mlp_layers=1, mlp_dims=2048)
    model = nn.Model(module, nn.ParamArena(module, shape, flat))
    p = params_torch(eng, flat)
    kw = dict(num_layers=1, num_heads=8, num_mlp_layers=1)
    apply = lambda a, s: O.transformer_ddpm(p, a, s, emulate_bf16=True, **kw)  # noqa: E731
    sigmas = np.asarray([1.0, 0.3, 0.05], np.float32)
    init, samples, masks = (t.cpu() for t in _inputs(shape, 4, seed=3))
    key = tf.prng_key(11)
    state, coll, mets = ebm_utils.annealed_langevin_dynamics(key, model, sigmas, init, 2e-5, 4, True, True, samples,
                                                             masks)
    keys, k = {}, key
    for si in range(3):
        for i in range(4):
            k, sk, ik = tf.split(k, 3)
            keys[(si, i)] = (sk, ik)
    noise_fn = lambda si, i: (torch.from_numpy(tf.normal(keys[(si, i)][0], (4,) + shape)),  # noqa: E731
                              torch.from_numpy(tf.normal(keys[(si, i)][1], (4,) + shape)))
    ref_state, ref_coll, ref_m = O.annealed_langevin_dynamics(apply, sigmas, init, 2e-5, 4, True, noise_fn, True,
                                                              samples, masks)
    assert rel_l2(state, ref_state) < 1e-2
    assert coll.shape == (102, 4) + shape and rel_l2(coll[-1], ref_coll[-1]) < 1e-2
    np.testing.assert_allclose(mets.cpu().numpy(), ref_m.numpy(), rtol=2e-2, atol=1e-7)
    ks, k = [], key
    for _ in range(6):
        k, sk = tf.split(k, 2)
        ks.append(sk)
    sig6 = O.create_noise_schedule(1.0, 0.05, 6, "geometric")
    state, coll, mets = ebm_utils.consistent_langevin_dynamics(key, model, sig6, init, 1e-4, 1, True)
    ref_state, ref_m = O.consistent_langevin_dynamics(apply, sig6, init, 1e-4, True,
                                                      lambda i: torch.from_numpy(tf.normal(ks[i], (4,) + shape)))
    assert coll is None and rel_l2(state, ref_state) < 1e-2
    np.testing.assert_allclose(mets.cpu().numpy(), ref_m.numpy(), rtol=2e-2, atol=1e-7)


@pytest.mark.parametrize("case,kind", [("dense", "ald"), ("t32", "ald"), ("dense", "cas")])
def test_two_ranks_of_four_equal_one_rank_of_eight(lib, case, kind):
    eng, _, shape = _engine(case)
    init, samples, masks = _inputs(shape, 8, seed=9)
    ix, im = (samples, masks) if kind == "ald" else (None, None)
    sigmas = O.create_noise_schedule(1.0, 0.05, 4, "geometric")
    key = tf.prng_key(5)
    full_x, full_c, full_m = device_chain(eng, kind, sigmas, 6, 2e-5, key, init, True, ix, im)
    xs, cs, ms = [], [], []
    for r in range(2):
        sl = slice(4 * r, 4 * r + 4)
        x, c, m = device_chain(eng, kind, sigmas, 6, 2e-5, key, init[sl].contiguous(), True,
                               None if ix is None else ix[sl].contiguous(), None if im is None else im[sl].contiguous(),
                               shard=(4 * r, 8))
        xs.append(x)
        cs.append(c)
        ms.append(m)
    assert torch.equal(torch.cat(xs), full_x)
    if kind == "ald":
        assert torch.equal(torch.cat(cs, dim=1), full_c)
    # the weighted all-reduce of ebm_utils: sum of n_r / N times each rank's batch means; alpha row unweighted
    w = ms[0] * 0.5 + ms[1] * 0.5
    w[2] = ms[0][2]
    torch.testing.assert_close(w, full_m, rtol=1e-6, atol=0)


def test_uniform_rows_are_the_slice_of_the_full_draw(lib):
    from smd_b200 import jrandom as random
    key = random.PRNGKey(42)
    rho = float(np.sqrt(np.float32(12)) / 2)
    full = random.uniform(key, (10, 32, 42), -rho, rho)
    part = random.uniform(key, (10, 32, 42), -rho, rho, rows=(3, 4))
    assert torch.equal(part, full[3:7])


def test_graph_recaptured_on_new_buffers_and_per_step_film(lib):
    eng, flat, shape = _engine("dense")
    init, samples, masks = _inputs(shape, 8, seed=1)
    sigmas = O.create_noise_schedule(1.0, 0.05, 5, "geometric")
    key = tf.prng_key(3)
    ref_x, ref_c, ref_m = host_chain(eng, "ald", sigmas, 4, 2e-5, key, init, True, samples, masks)
    eng.langevin_setup(sigmas, 4, 2e-5, "ald", key=(int(key[0]), int(key[1])))

    def run(x=None, coll=None, mets=None):
        x = init.clone() if x is None else x.copy_(init)
        coll = torch.zeros_like(ref_c) if coll is None else coll.zero_()
        coll[0] = x * (1 - masks) + samples * masks
        mets = torch.zeros_like(ref_m) if mets is None else mets
        eng.langevin_sample(x, denoise=True, infill_x=samples, infill_mask=masks, collection=coll, metrics=mets)
        return x, coll, mets

    x1, c1, m1 = run()
    x2, c2, m2 = run(x1, c1, m1)              # same buffers: the graph is replayed as captured
    assert torch.equal(x2, ref_x) and torch.equal(c2, ref_c)
    x3, c3, m3 = run()                         # new x / collection / metrics: re-captured
    assert torch.equal(x3, ref_x) and torch.equal(c3, ref_c)
    torch.testing.assert_close(m3, ref_m, rtol=1e-6, atol=0)
    # new parameters at a new address: re-captured (and a new FiLM table)
    flat2 = eng.init_params(seed=9, perturb=0.02)
    eng.set_params(flat2)
    ref2 = host_chain(eng, "ald", sigmas, 4, 2e-5, key, init, True, samples, masks)[0]
    assert torch.equal(run(x1, c1, m1)[0], ref2) and not torch.equal(ref2, ref_x)
    # more levels than FiLM-table rows: the per-step generator runs inside the graph
    from smd_b200 import Engine, ModelConfig
    small = Engine(ModelConfig(**CASES["dense"][0]), max_batch=8, sampler_T=4)
    small.set_params(flat)
    sig6 = O.create_noise_schedule(1.0, 0.05, 6, "geometric")
    a = device_chain(small, "ald", sig6, 3, 2e-5, key, init, True, samples, masks)
    b = host_chain(small, "ald", sig6, 3, 2e-5, key, init, True, samples, masks)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_setups_invalidate_each_other(lib):
    from smd_b200 import lib as L
    eng, _, shape = _engine("t32")
    x = _inputs(shape, 4)[0]
    betas = O.create_noise_schedule(1e-6, 0.01, 10, "linear")
    eng.sampler_setup(betas, key=(0, 1))
    eng.langevin_setup(np.asarray([1.0, 0.1], np.float32), 2, 1e-5, "ald")
    with pytest.raises(L.SmdError, match="smd_sampler_setup"):
        eng.sample(x.clone(), steps=10)
    eng.langevin_sample(x.clone())
    eng.sampler_setup(betas, key=(0, 1))
    with pytest.raises(L.SmdError, match="smd_langevin_setup"):
        eng.langevin_sample(x.clone())
    eng.sample(x.clone(), steps=10)
    eng.langevin_setup(np.asarray([1.0, 0.1], np.float32), 1, 1e-5, "cas")
    with pytest.raises(ValueError):
        eng.langevin_sample(x.clone(), infill_x=x, infill_mask=x)
    with pytest.raises(ValueError):
        eng.langevin_sample(x.clone(), collection=torch.zeros((102,) + tuple(x.shape), device="cuda"))
    big = torch.zeros((16,) + shape, device="cuda")
    with pytest.raises(ValueError):
        eng.langevin_sample(big)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------- command lines
def _train(tmp_path, name, flags):
    cfg = tmp_path / f"{name}.cfg"
    cfg.write_text(textwrap.dedent(flags).format(run=tmp_path / name))
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "smd_b200.train_ncsn", f"--flagfile={cfg}"], capture_output=True,
                       text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    return cfg, env


def _sample(cfg, env, *extra, launcher=()):
    cmd = list(launcher) + ([sys.executable, "-m"] if not launcher else ["-m"]) + ["smd_b200.sample_ncsn",
                                                                                f"--flagfile={cfg}", *extra]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]


def _load(d, name):
    with open(os.path.join(d, "ncsn", name), "rb") as f:
        return pickle.load(f)


DENSE_FLAGS = """\
    --loss=dsm
    --sampling=ald
    --architecture=DenseNCSN
    --num_layers=2
    --mlp_dims=512
    --num_sigmas=4
    --ld_steps=30
    --ld_epsilon=2e-6
    --problem=vae
    --ema=False
    --nosnapshot_sampling
    --data_shape=512
    --batch_size=16
    --learning_rate=1e-3
    --max_steps=2
    --snapshot_freq=2
    --synthetic
    --synthetic_examples=64
    --model_dir={run}
    """

TRANSFORMER_FLAGS = """\
    --loss=ddpm
    --sampling=ald
    --schedule_type=geometric
    --sigma_begin=1.0
    --sigma_end=0.001
    --num_sigmas=5
    --ld_steps=25
    --ld_epsilon=2e-6
    --problem=vae
    --ema=False
    --nosnapshot_sampling
    --architecture=TransformerDDPM
    --num_layers=1
    --num_mlp_layers=1
    --data_shape=32,42
    --batch_size=8
    --learning_rate=1e-3
    --max_steps=2
    --snapshot_freq=2
    --synthetic
    --synthetic_examples=64
    --model_dir={run}
    """


def test_sample_ncsn_langevin_command_lines(lib, tmp_path):
    cfg, env = _train(tmp_path, "dense", DENSE_FLAGS)
    _sample(cfg, env, "--sample_size=16")
    out = tmp_path / "dense" / "samples"
    gen, coll = _load(out, "generated.pkl"), _load(out, "collection.pkl")
    assert gen.shape == (16, 512) and coll.shape == (102, 16, 512) and np.isfinite(gen).all()
    # consistent Langevin dynamics: no collection, but generated / real are written
    _sample(cfg, env, "--sample_size=16", "--sampling=cas", "--sampling_dir=cas")
    out = tmp_path / "dense" / "cas"
    assert _load(out, "generated.pkl").shape == (16, 512) and _load(out, "real.pkl").shape == (16, 512)
    assert not os.path.exists(out / "ncsn" / "collection.pkl")

    cfg, env = _train(tmp_path, "tr", TRANSFORMER_FLAGS)
    _sample(cfg, env, "--sample_size=8")
    gen = _load(tmp_path / "tr" / "samples", "generated.pkl")
    assert gen.shape == (8, 32, 42) and np.isfinite(gen).all()
    # infill with the annealed chain: the held latents end at samples + sigma_L z (no denoising step; sigma_L = 1e-3,
    # and real.pkl is in the de-normalised units of the data)
    _sample(cfg, env, "--sample_size=8", "--infill", "--sampling_dir=infill", "--nodenoise")
    out = tmp_path / "tr" / "infill"
    gen, real = _load(out, "generated.pkl"), _load(out, "real.pkl")
    assert gen.shape == (8, 32, 42) and np.isfinite(gen).all()
    np.testing.assert_allclose(gen[:, :8], real[:, :8], rtol=0, atol=0.03)
    np.testing.assert_allclose(gen[:, -8:], real[:, -8:], rtol=0, atol=0.03)
    assert np.abs(gen[:, 8:-8] - real[:, 8:-8]).mean() > 10 * np.abs(gen[:, :8] - real[:, :8]).mean()
    # consistent Langevin dynamics has no infilling (NotImplementedError upstream as well)
    r = subprocess.run([sys.executable, "-m", "smd_b200.sample_ncsn", f"--flagfile={cfg}", "--sample_size=8",
                        "--infill", "--sampling=cas", "--sampling_dir=cas_infill"], capture_output=True, text=True,
                       timeout=600, env=env, cwd=ROOT)
    assert r.returncode != 0 and "NotImplementedError" in r.stderr


def test_sample_ncsn_ald_under_torchrun_equals_one_rank(lib, tmp_path):
    if torch.cuda.device_count() < 2 or shutil.which("torchrun") is None:
        pytest.skip("the torchrun comparison needs 2 GPUs")
    cfg, env = _train(tmp_path, "tr", TRANSFORMER_FLAGS)
    _sample(cfg, env, "--sample_size=8")
    _sample(cfg, env, "--sample_size=8", "--sampling_dir=dp", launcher=("torchrun", "--nproc-per-node", "2"))
    one = _load(tmp_path / "tr" / "samples", "generated.pkl")
    two = _load(tmp_path / "tr" / "dp", "generated.pkl")
    assert two.shape == one.shape
    np.testing.assert_array_equal(two, one)
