"""train_mdn on the CPU: the flag surface parsed from a flagfile with the mdn-base / mdn-mel-32seq-512 values, the
stepped learning-rate schedule with and without warmup, the flax parameter-tree paths of TransformerMDN, and the
(optimizer, early_stop) state-dict layout."""
import json
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_PARSE = """
import json, sys
from absl import flags
from smd_b200 import train_mdn
FLAGS = flags.FLAGS
FLAGS(["train_mdn"] + sys.argv[1:])
names = ["architecture", "num_layers", "num_heads", "num_mlp_layers", "mlp_dims", "mdn_components", "data_shape",
         "batch_size", "learning_rate", "max_steps", "epochs", "lr_schedule_interval", "lr_gamma", "lr_warmup",
         "dataset", "slice_ckpt", "model_dir", "synthetic"]
out = {n: getattr(FLAGS, n) for n in names}
out["lr"] = [train_mdn.lr_at(s) for s in (0, 1, 4000, 4001, 8001, 20000)]
print(json.dumps(out))
"""


def _parse(*argv):
    r = subprocess.run([sys.executable, "-c", _PARSE, *argv], capture_output=True, text=True, timeout=300, cwd=ROOT,
                       env=dict(os.environ, PYTHONPATH=ROOT))
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_defaults_follow_the_reference():
    d = _parse()
    assert d["lr_schedule_interval"] == 4000 and d["max_steps"] == 100000 and d["architecture"] == "TransformerMDN"
    assert d["mdn_components"] == 100 and d["epochs"] == 1000 and d["lr_warmup"] == 0 and not d["synthetic"]


def test_flagfile_with_the_mdn_configs(tmp_path):
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
    d = _parse(f"--flagfile={cfg}")
    assert d["num_layers"] == 6 and d["max_steps"] == 250000 and d["batch_size"] == 128
    assert d["data_shape"] == ["32", "512"] and d["slice_ckpt"] == "./checkpoints/slice-mel-512.pkl"
    assert d["model_dir"] == "save/mel512-mdn-32seq" and d["mdn_components"] == 100


def test_stepped_lr_schedule_with_and_without_warmup():
    # flax create_stepped_learning_rate_schedule: boundaries i * interval, values lr * [1, gamma^0, gamma^1, ...]
    def flax_lr(step, lr=3e-4, interval=4000, gamma=0.98, warmup=0.0):
        boundaries = np.array([i * interval for i in range(1000)])
        values = np.array([1.0] + [gamma ** i for i in range(1000)]) * lr
        v = values[int(np.sum(boundaries < step))]
        if warmup > 0:
            v = v * min(1.0, step / float(warmup) / interval)
        return v
    steps = (0, 1, 4000, 4001, 8001, 20000)
    np.testing.assert_allclose(_parse()["lr"], [flax_lr(s) for s in steps], rtol=1e-12)
    np.testing.assert_allclose(_parse("--lr_warmup=2")["lr"], [flax_lr(s, warmup=2.0) for s in steps], rtol=1e-12)
    np.testing.assert_allclose(_parse("--lr_warmup=0.5", "--lr_schedule_interval=1000", "--lr_gamma=0.5")["lr"],
                               [flax_lr(s, interval=1000, gamma=0.5, warmup=0.5) for s in steps], rtol=1e-12)


def test_flax_path_map_of_transformer_mdn():
    from smd_b200 import flax_compat
    from smd_b200.engine import ModelConfig
    from tests import mdn_reference as R
    cfg = ModelConfig(arch="TransformerMDN", num_layers=2, num_heads=8, num_mlp_layers=2, mlp_dims=64, channels=4,
                      mdn_components=3)
    paths = flax_compat._tree_paths(cfg)
    L, K = 2, 2
    assert paths["in"] == (("Dense_1",), "dense")
    assert paths["l1.ln1"] == (("LayerNorm_7",), "ln")
    assert paths["post"] == ((f"Dense_{3 + 5 * L}",), "dense")
    assert paths["k0.res.a"] == (("DenseResBlock_14", "Dense_2"), "dense")          # DenseResBlock_{4 + 5L + k}
    assert paths["k1.res.ln_b"] == (("DenseResBlock_15", "LayerNorm_3"), "ln")
    assert paths["out_ln"] == ((f"LayerNorm_{4 + 5 * L + K}",), "ln")
    assert paths["mdn.mu"] == (("mdn", "Dense_0"), "dense") and paths["mdn.log_sigma"] == (("mdn", "Dense_1"), "dense")
    assert paths["mdn.pi"] == (("mdn", "Dense_2"), "dense")
    assert not any("film" in k for k in paths)
    shapes = R.param_shapes(4, L, 64, K, 3)
    rng = np.random.default_rng(0)
    named = {n: rng.standard_normal(s).astype(np.float32) for n, s in shapes.items()}
    back = flax_compat.params_from_flax(flax_compat.params_to_flax(named, cfg), cfg)
    assert sorted(back) == sorted(named)
    for n in named:
        np.testing.assert_array_equal(back[n], named[n])
