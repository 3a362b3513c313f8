"""TransformerMDN autoregressive sampling (sample_mdn.py) through the C ABI: the plan-free mixture sampler against the
CPU oracle (tests/mdn_sample_reference.py), a known mixture end to end, a teacher-forced replay of the decoded chain
through the bf16-emulating oracle, the key/value cache, reproducibility and sharding, argument errors and the
command line.

Tolerances are about twice the errors measured on an H100 with bf16 tensor-core operands."""
import ctypes as C
import os
import pickle
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import threefry as TF
from smd_b200 import lib as L
from tests import mdn_reference as MR
from tests import mdn_sample_reference as R
from tests.util import params_torch, rel_l2

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KW = dict(num_layers=2, num_heads=8, num_mlp_layers=2, mlp_dims=2048, mdn_components=100)
CH = 42
S = 32
KEY = TF.split(TF.prng_key(1), 2)[0]    # rng after `rng, model_rng = split(PRNGKey(sample_seed))`


def _engine(n, training=False, **over):
    from smd_b200 import Engine, ModelConfig
    kw = dict(KW, **over)
    eng = Engine(ModelConfig(arch="TransformerMDN", channels=CH, **kw), max_batch=n, training=training, sampler_T=S)
    flat = eng.init_params(seed=5, perturb=0.02)
    eng.set_params(flat)
    return eng, flat


def _plan_free(pi, mu, ls, key, first_row=0, total_rows=0):
    rows, kc = pi.shape
    out = torch.empty((rows, mu.shape[1] // kc), dtype=torch.float32, device="cuda")
    comp = torch.empty((rows,), dtype=torch.int32, device="cuda")
    k = (C.c_uint32 * 2)(int(key[0]), int(key[1]))
    L.check(L.load_library().smd_mdn_mixture_sample(pi.data_ptr(), mu.data_ptr(), ls.data_ptr(), rows, out.shape[1], kc,
                                                    k, first_row, total_rows, out.data_ptr(), comp.data_ptr(),
                                                    torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return out.cpu().numpy(), comp.cpu().numpy()


def _gap(pi, key):
    """Top-two gap of pi + g per row, and the scale of pi + g (for the fp32-rounding band of a component tie)."""
    _, mix_key = R.mixture_sample_keys(key)
    n, kc = pi.shape
    u01 = R._u01(R.random_bits_at(mix_key, np.arange(n)[:, None] * kc + np.arange(kc), n * kc))
    tiny = np.float32(np.finfo(np.float32).tiny)
    g = -np.log(-np.log(np.maximum(tiny, u01 * (np.float32(1) - tiny) + tiny)))
    v = np.sort(pi.astype(np.float64) + g, axis=-1)
    return v[:, -1] - v[:, -2], np.abs(v).max(axis=-1)


def test_plan_free_sampler_matches_oracle(lib):
    rows, kc = 3000, 100
    rng = np.random.default_rng(0)
    pi = rng.normal(0, 3, (rows, kc)).astype(np.float32)
    mu = rng.normal(0, 1, (rows, kc * CH)).astype(np.float32)
    ls = rng.uniform(-3, 1.5, (rows, kc * CH)).astype(np.float32)
    d = [torch.from_numpy(a).cuda() for a in (pi, mu, ls)]
    key = TF.prng_key(7)
    x, k = _plan_free(*d, key)
    xr, kr = R.mixture_sample(pi, mu, ls, key)
    gap, scale = _gap(pi, key)
    flip = k != kr
    assert np.all(gap[flip] <= 4 * np.finfo(np.float32).eps * scale[flip]), np.nonzero(flip)
    err = np.abs(x[~flip] - xr[~flip]) / np.maximum(np.abs(xr[~flip]), 1.0)
    print(f"plan-free mixture sample: {int(flip.sum())} component flips in {rows} rows, max rel err {err.max():.3e}")
    assert err.max() <= 2e-6
    xs, ks = _plan_free(*(t[1000:1500].contiguous() for t in d), key, first_row=1000, total_rows=rows)
    assert np.array_equal(xs, x[1000:1500]) and np.array_equal(ks, k[1000:1500])


def _set(eng, flat, name, value):
    off, shape = next((o, s) for nm, o, s in eng.layout if nm == name)
    flat[off:off + int(np.prod(shape))] = np.asarray(value, np.float32).reshape(-1)


def test_known_mixture_end_to_end(lib):
    """Zero head kernels: every position's mixture is the head biases, so the decoded chain and the last step's draws
    must both follow it.  Component means 10 k apart identify a chain token's component."""
    n, kc = 2048, 100
    eng, flat = _engine(n, mlp_dims=256)
    pi_b = np.random.default_rng(3).normal(0, 1, kc).astype(np.float32)
    mu_b = (10.0 * np.arange(kc)[:, None] + np.linspace(-1, 1, CH)[None]).astype(np.float32)
    ls_b = (np.linspace(-1.5, 0.0, CH)[None] + 0.005 * np.arange(kc)[:, None]).astype(np.float32)
    for part, bias in (("pi", pi_b), ("mu", mu_b), ("log_sigma", ls_b)):
        _set(eng, flat, f"mdn.{part}.kernel", 0.0)
        _set(eng, flat, f"mdn.{part}.bias", bias)
    eng.set_params(flat)
    out, chain, comp = eng.mdn_sample(KEY, n, chain=True, components=True)
    out, chain, comp = out.cpu().numpy(), chain.cpu().numpy(), comp.cpu().numpy()
    assert np.all(chain[:, 0] == 0)
    p = np.exp(pi_b.astype(np.float64) - pi_b.max())
    p /= p.sum()
    sig = np.exp(ls_b.astype(np.float64))
    toks = chain[:, 1:].reshape(-1, CH)
    k_chain = np.clip(np.rint(toks.mean(-1) / 10.0).astype(int), 0, kc - 1)
    for name, x, k in (("final", out.reshape(-1, CH), comp.reshape(-1)), ("chain", toks, k_chain)):
        counts = np.bincount(k, minlength=kc)
        pv = stats.chisquare(counts, p * counts.sum()).pvalue
        print(f"known mixture ({name}): chi-square p = {pv:.3f} over {counts.sum()} draws")
        assert pv > 1e-4, (name, counts)
        for j in np.nonzero(counts >= 2)[0]:
            xj = (x[k == j] - mu_b[j]) / sig[j]               # standardised: N(0, 1) per channel
            m = len(xj)
            assert np.all(np.abs(xj.mean(0)) < 6.0 / np.sqrt(m)), (name, j)
            if m >= 50:
                assert np.all(np.abs(xj.std(0) - 1.0) < 6.0 / np.sqrt(2 * m)), (name, j)


@pytest.mark.parametrize("heads", [8, 32])
def test_teacher_forced_replay_matches_oracle(lib, heads):
    n = 64
    eng, flat = _engine(n, num_heads=heads)
    out, chain, comp = eng.mdn_sample(KEY, n, chain=True, components=True)
    out, chain, comp = out.cpu().numpy(), chain.cpu().numpy(), comp.cpu().numpy()
    pe = params_torch(eng, flat, torch.float32)
    with torch.no_grad():
        pi, mu, ls = (a.numpy().reshape(n * S, -1) for a in
                      MR.transformer_mdn(pe, torch.from_numpy(chain), shift=False, emulate_bf16=True,
                                         **dict(KW, num_heads=heads)))
    keys = R.step_keys(KEY, S)
    rows = np.arange(n) * S
    got, want = [], []
    for i in range(S - 1):       # chain position i + 1 is row b * S + i of step i's draw
        xr, _ = R.mixture_sample(pi[rows + i], mu[rows + i], ls[rows + i], keys[i], total_rows=n * S, row_index=rows + i)
        got.append(chain[:, i + 1]); want.append(xr)
    xr, kr = R.mixture_sample(pi, mu, ls, keys[-1])
    final_flip = comp.reshape(-1) != kr
    got, want = np.concatenate(got + [out.reshape(-1, CH)]), np.concatenate(want + [xr])
    # a component flip moves the token by O(1); bf16 moves it by ~1e-2 of its size
    row_err = np.linalg.norm(got - want, axis=-1) / np.maximum(np.linalg.norm(want, axis=-1), 1e-6)
    flip = row_err > 0.2
    flip[-n * S:] |= final_flip
    frac = float(flip.mean())
    err = rel_l2(torch.from_numpy(got[~flip]), torch.from_numpy(want[~flip]))
    print(f"teacher-forced replay heads={heads}: component flips {frac:.4f} of {len(flip)} (row, step) pairs "
          f"(final step {float(final_flip.mean()):.4f}), rel-L2 of the rest {err:.3e}")
    assert frac <= 0.005 and err < 8e-3


def test_key_value_cache_matches_the_full_forward(lib):
    """A training plan keeps one qkv region per layer: after sampling, t.qkv{l} holds the last step's full forward over
    the chain, whose first S - 1 positions the decode steps cached in mdn.kv{l}."""
    n = 16
    eng, _ = _engine(n, training=True)
    eng.mdn_sample(KEY, n)
    torch.cuda.synchronize()
    for l in range(KW["num_layers"]):
        kv = _region(eng, f"mdn.kv{l}", (n, S, 384))[:, :S - 1]
        full = _region(eng, f"t.qkv{l}", (n, S, 384))[:, :S - 1]
        err = rel_l2(kv, full)
        print(f"mdn.kv{l} vs t.qkv{l}: rel-L2 {err:.3e}")
        assert err < 3e-3


class _DeviceBytes:
    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "strides": None,
                                         "version": 3}


def _region(eng, name, shape):
    ptr, nbytes = C.c_void_p(), C.c_size_t()
    L.check(eng.lib.smd_debug_buffer(eng._plan, name.encode(), C.byref(ptr), C.byref(nbytes)))
    need = int(np.prod(shape)) * 4
    assert need <= nbytes.value, (name, need, nbytes.value)
    raw = torch.as_tensor(_DeviceBytes(ptr.value, nbytes.value), device="cuda")
    return raw[:need].view(torch.float32).reshape(shape).cpu()


def test_reproducible_and_shards_equal_the_whole_batch(lib):
    n = 96                        # 96 and 48 samples: both below the fused-FFN threshold of the final forward
    eng, _ = _engine(n)
    a, ca = eng.mdn_sample(KEY, n, components=True)
    b, cb = eng.mdn_sample(KEY, n, components=True)
    c = eng.mdn_sample(TF.split(TF.prng_key(2), 2)[0], n)
    assert torch.equal(a, b) and torch.equal(ca, cb) and not torch.equal(a, c)
    half = n // 2
    parts = [eng.mdn_sample(KEY, half, first_row=r * half, total_rows=n, chain=True) for r in range(2)]
    whole, chain = eng.mdn_sample(KEY, n, chain=True)
    assert torch.equal(torch.cat([p[0] for p in parts]), whole)
    assert torch.equal(torch.cat([p[1] for p in parts]), chain)
    assert torch.isfinite(whole).all()


def test_argument_errors(lib):
    from smd_b200 import Engine, ModelConfig
    eng, _ = _engine(4)
    with pytest.raises(ValueError, match="max_batch|out of range"):
        eng.mdn_sample(KEY, 5)
    with pytest.raises(ValueError, match="total_rows"):
        eng.mdn_sample(KEY, 4, first_row=2, total_rows=5)
    with pytest.raises(ValueError, match="2\\^32"):
        eng.mdn_sample(KEY, 4, first_row=0, total_rows=40000)        # 40000 * 32 * 100 * 42 counters
    plain = Engine(ModelConfig(arch="TransformerMDN", channels=CH, **KW), max_batch=4)
    plain.set_params(plain.init_params(seed=0))
    with pytest.raises(L.SmdError, match="sampler_T"):
        plain.mdn_sample(KEY, 4)
    ddpm = Engine(ModelConfig(channels=CH), max_batch=4)
    ddpm.set_params(ddpm.init_params(seed=0))
    with pytest.raises(ValueError, match="TransformerMDN"):
        Engine.mdn_sample(ddpm, KEY, 4)
    pi = torch.zeros((10, KW["mdn_components"]), device="cuda")
    mu = torch.zeros((10, KW["mdn_components"] * CH), device="cuda")
    with pytest.raises(ValueError, match="2\\^32"):
        eng.mdn_mixture_sample(pi, mu, mu, KEY, total_rows=2_000_000)
    with pytest.raises(ValueError, match="total_rows"):
        eng.mdn_mixture_sample(pi, mu, mu, KEY, first_row=5, total_rows=12)
    with pytest.raises(ValueError):
        eng.mdn_mixture_sample(pi[:, :-1].contiguous(), mu, mu, KEY)


def test_sample_mdn_cli(tmp_path):
    cfg = tmp_path / "mdn.cfg"
    cfg.write_text(textwrap.dedent(f"""\
        --architecture=TransformerMDN
        --num_layers=2
        --num_heads=8
        --num_mlp_layers=2
        --mlp_dims=512
        --mdn_components=20
        --data_shape=32,42
        --batch_size=16
        --learning_rate=1e-3
        --logging_freq=5
        --snapshot_freq=10
        --nosnapshot_sampling
        --synthetic
        --synthetic_examples=640
        --model_dir={tmp_path / 'run'}
        """))
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "smd_b200.train_mdn", f"--flagfile={cfg}", "--max_steps=12"],
                       capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    outs = []
    for ranks in ((1, 2) if torch.cuda.device_count() >= 2 else (1,)):
        d = tmp_path / f"sample{ranks}"
        launch = [sys.executable] if ranks == 1 else [sys.executable, "-m", "torch.distributed.run", "--nnodes=1",
                                                     f"--nproc-per-node={ranks}", "--master-addr", "127.0.0.1",
                                                     "--master-port", "29547"]
        r = subprocess.run(launch + ["-m", "smd_b200.sample_mdn", f"--flagfile={cfg}", "--sample_size=64",
                                     f"--sampling_dir={d}"], capture_output=True, text=True, timeout=600, env=env,
                           cwd=ROOT)
        assert r.returncode == 0, r.stderr[-3000:]
        with open(d / "mdn" / "generated.pkl", "rb") as f:
            gen = np.asarray(pickle.load(f))
        with open(d / "mdn" / "real.pkl", "rb") as f:
            real = np.asarray(pickle.load(f))
        assert gen.shape == real.shape == (64, 32, 42) and np.isfinite(gen).all() and np.isfinite(real).all()
        outs.append(gen)
    if len(outs) == 2:
        np.testing.assert_array_equal(outs[0], outs[1])
