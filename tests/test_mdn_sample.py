"""TransformerMDN autoregressive sampling on the CPU: the random-number recipe of the sampling oracle
(tests/mdn_sample_reference.py), its mixture draws against the distribution they sample, the reference's last-step
resample, the decode-state workspace of sampler plans, spill-free SASS of the new kernels and the sample_mdn flags."""
import hashlib
import json
import math
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import threefry as TF
from tests import mdn_reference as MR
from tests import mdn_sample_reference as R
from tests.test_sass_evidence import _get, table  # noqa: F401  (module-scoped fixture: one cuobjdump pass)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_fold_in_and_salt_follow_their_definitions():
    assert R.MIXTURE_SALT == int(hashlib.sha512(b"MixtureSameFamily").hexdigest(), 16) & 0xFFFFFFFF
    for seed, data in ((0, 0), (1, R.MIXTURE_SALT), (12345, 7)):
        key = TF.prng_key(seed)
        # jax 0.2.8: fold_in(key, d) = threefry_2x32(key, threefry_seed(d)), threefry_seed(d) = [d >> 32, d & mask]
        np.testing.assert_array_equal(R.fold_in(key, data), TF.threefry_2x32(key, np.array([0, data], np.uint32)))
    comp, mix = R.mixture_sample_keys(TF.prng_key(4))
    np.testing.assert_array_equal(np.stack([comp, mix]), TF.split(R.fold_in(TF.prng_key(4), R.MIXTURE_SALT), 2))
    for n in (1, 8, 101):
        idx = np.arange(n)
        np.testing.assert_array_equal(R.random_bits_at(TF.prng_key(9), idx, n), TF.random_bits(TF.prng_key(9), (n,)))


def test_mixture_draw_is_the_jax_draw_at_the_chosen_component():
    rows, kc, C = 6, 4, 3
    rng = np.random.default_rng(0)
    pi = rng.normal(0, 1, (rows, kc)).astype(np.float32)
    mu = rng.normal(0, 1, (rows, kc * C)).astype(np.float32)
    ls = rng.uniform(-1, 0.5, (rows, kc * C)).astype(np.float32)
    key = TF.prng_key(11)
    x, k = R.mixture_sample(pi, mu, ls, key)
    comp_key, mix_key = R.mixture_sample_keys(key)
    g = -np.log(-np.log(TF.uniform(mix_key, (rows, kc), np.finfo(np.float32).tiny, 1.0)))
    np.testing.assert_array_equal(k, np.argmax(pi + g, axis=-1))
    z = TF.normal(comp_key, (rows, kc, C))
    sel = np.arange(rows)
    ref = mu.reshape(rows, kc, C)[sel, k] + np.exp(ls.reshape(rows, kc, C)[sel, k]) * z[sel, k]
    np.testing.assert_allclose(x, ref, rtol=1e-6, atol=1e-6)
    # a slice of a larger draw is the same rows of the whole draw
    xs, ks = R.mixture_sample(pi[2:5], mu[2:5], ls[2:5], key, first_row=2, total_rows=rows)
    np.testing.assert_array_equal(xs, x[2:5])
    np.testing.assert_array_equal(ks, k[2:5])


def test_mixture_draws_follow_the_mixture():
    rows, kc, C = 40000, 5, 3
    pi_row = np.array([0.5, -1.0, 1.2, 0.0, -0.3], np.float32)
    mu_row = np.arange(kc * C, dtype=np.float32) * 0.5 - 3.0
    ls_row = np.linspace(-1.5, 0.5, kc * C).astype(np.float32)
    x, k = R.mixture_sample(np.tile(pi_row, (rows, 1)), np.tile(mu_row, (rows, 1)), np.tile(ls_row, (rows, 1)),
                            TF.prng_key(21))
    p = np.exp(pi_row.astype(np.float64) - pi_row.max())
    p /= p.sum()
    counts = np.bincount(k, minlength=kc)
    assert stats.chisquare(counts, p * rows).pvalue > 1e-3
    for j in range(kc):
        xj = x[k == j]
        m, s = mu_row[j * C:(j + 1) * C], np.exp(ls_row[j * C:(j + 1) * C])
        for c in range(C):
            assert stats.kstest((xj[:, c] - m[c]) / s[c], "norm").pvalue > 1e-3, (j, c)


def _tiny_model(C=4, kc=3):
    kw = dict(num_layers=1, num_heads=8, num_mlp_layers=1, mlp_dims=64, mdn_components=kc)
    g = torch.Generator().manual_seed(0)
    p = {}
    for name, shape in MR.param_shapes(C, 1, 64, 1, kc).items():
        scale = 1.0 / math.sqrt(shape[0]) if name.endswith(".kernel") else 0.1
        p[name] = torch.randn(*shape, generator=g) * scale + (1.0 if name.endswith(".scale") else 0.0)

    def model(tokens):
        with torch.no_grad():
            return [a.numpy() for a in MR.transformer_mdn(p, torch.from_numpy(tokens), shift=False, **kw)]
    return model


def test_last_step_resamples_every_position():
    n, S, C = 3, 32, 4
    model = _tiny_model(C)
    key = TF.split(TF.prng_key(1), 2)[0]          # rng after `rng, model_rng = split(rng)`
    out, chain = R.sample_mdn(model, key, n, S, C)
    assert out.shape == chain.shape == (n, S, C) and np.isfinite(out).all()
    assert np.all(chain[:, 0] == 0) and np.all(chain[:, 1:] != 0)
    # the result is a fresh draw at every position of one pass over the chain, not the chain shifted by one
    assert not np.any(out[:, :-1] == chain[:, 1:])
    pi, mu, ls = (a.reshape(n * S, -1) for a in model(chain))
    last = R.step_keys(key, S)[-1]
    x, _ = R.mixture_sample(pi, mu, ls, last)
    np.testing.assert_array_equal(out, x.reshape(n, S, C))
    # sharded: samples [1, 3) of the 3-sample run
    out2, chain2 = R.sample_mdn(model, key, 2, S, C, first_row=1, total_rows=n)
    np.testing.assert_allclose(out2, out[1:], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(chain2, chain[1:], rtol=1e-5, atol=1e-5)


# smd_workspace_bytes of TransformerMDN plans without decode state, recorded at the commit before sampler plans existed
_WS_BEFORE = {("large", False, 128): 354553856, ("large", False, 1000): 2008482816,
              ("large", True, 128): 1138153472, ("large", True, 1000): 8130562048,
              ("small", False, 2): 3054592, ("small", False, 64): 14274560,
              ("small", True, 2): 8095744, ("small", True, 64): 65730560}
_CFGS = {"large": dict(num_layers=6, num_heads=8, num_mlp_layers=2, mlp_dims=2048, channels=42, mdn_components=100),
         "small": dict(num_layers=2, num_heads=32, num_mlp_layers=1, mlp_dims=256, channels=8, mdn_components=4)}


def test_plans_without_decode_state_keep_their_workspace(lib):
    from smd_b200 import Engine, ModelConfig
    for (name, training, mb), nbytes in _WS_BEFORE.items():
        eng = Engine(ModelConfig(arch="TransformerMDN", **_CFGS[name]), max_batch=mb, training=training)
        assert eng.workspace_bytes == nbytes, (name, training, mb)


def test_sampler_plan_reserves_the_decode_state(lib):
    from smd_b200 import Engine, ModelConfig
    kib = lambda b: (b + 1023) // 1024 * 1024  # noqa: E731  (regions are 1024-byte aligned)
    for name, mb in (("large", 1000), ("small", 64)):
        c = _CFGS[name]
        cfg = ModelConfig(arch="TransformerMDN", **c)
        base = Engine(cfg, max_batch=mb)
        for asked in (1, 32, 1000):   # any sampler_T > 0 asks for the decode state of seq_len steps
            eng = Engine(cfg, max_batch=mb, sampler_T=asked)
            kv = c["num_layers"] * kib(mb * 32 * 384 * 4)
            assert eng.workspace_bytes == base.workspace_bytes + kv + kib(mb * c["channels"] * 4)


def test_sampling_kernels_do_not_spill(table):  # noqa: F811
    rows = _get(table, "mdn_decode_attention_kernel<")
    assert len(rows) == 4                                   # head dims 4, 8, 16, 32
    for c in rows + _get(table, "mdn_mixture_sample_kernel"):
        assert c.get("STL", 0) == 0 and c.get("LDL", 0) == 0, c


_PARSE = """
import json, sys
from absl import flags
from smd_b200 import sample_mdn
FLAGS = flags.FLAGS
FLAGS(["sample_mdn"] + sys.argv[1:])
names = ["sample_seed", "sampling_dir", "sample_size", "flush", "architecture", "num_layers", "num_heads",
         "num_mlp_layers", "mlp_dims", "mdn_components", "data_shape", "model_dir", "slice_ckpt", "synthetic"]
print(json.dumps({n: getattr(FLAGS, n) for n in names}))
"""


def _parse(*argv):
    r = subprocess.run([sys.executable, "-c", _PARSE, *argv], capture_output=True, text=True, timeout=300, cwd=ROOT,
                       env=dict(os.environ, PYTHONPATH=ROOT))
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_sample_mdn_flags_follow_the_reference(tmp_path):
    d = _parse()
    assert d["sample_seed"] == 1 and d["sampling_dir"] == "sample" and d["sample_size"] == 1000 and d["flush"]
    assert d["architecture"] == "TransformerMDN" and d["mdn_components"] == 100 and not d["synthetic"]
    base = tmp_path / "mdn-base.cfg"
    base.write_text(textwrap.dedent("""\
        --epochs=1000
        --learning_rate=3e-4
        --batch_size=128
        --max_steps=250000
        --mdn_components=100
        --num_layers=4
        --num_heads=8
        --num_mlp_layers=2
        --mlp_dims=2048
        """))
    cfg = tmp_path / "mdn-mel-32seq-512.cfg"
    cfg.write_text(textwrap.dedent(f"""\
        --flagfile={base}
        --architecture=TransformerMDN
        --num_layers=6
        --num_heads=8
        --num_mlp_layers=2
        --mlp_dims=2048
        --data_shape=32,512
        --dataset=./output/mel-32step-512
        --slice_ckpt=./checkpoints/slice-mel-512.pkl
        --model_dir=save/mel512-mdn-32seq
        """))
    d = _parse(f"--flagfile={cfg}", "--sample_size=64")
    assert d["num_layers"] == 6 and d["data_shape"] == ["32", "512"] and d["model_dir"] == "save/mel512-mdn-32seq"
    assert d["slice_ckpt"] == "./checkpoints/slice-mel-512.pkl" and d["sample_size"] == 64 and d["sample_seed"] == 1
