"""CPU tests of snapshot sampling in train_ncsn.train (train_ncsn.py:405-486 of the reference): the steps at which
the hook runs, the key it hands to sample(), and the files it writes.  The train step, the evaluation, the sampler
and the metric are stubs, so no device is needed; the GPU suite runs the real chain."""
import json
import os

import numpy as np
import torch
from absl import flags
from absl.testing import flagsaver

from oracle import threefry as tf

FLAGS = flags.FLAGS
SHAPE = (8,)
STUB_SCORES = {"frechet_distance": 1.5, "mmd_rbf": 0.25, "mmd_polynomial": 0.125}


def _flags(**kw):
    from smd_b200 import train_ncsn  # noqa: F401  (defines the flags)
    if not FLAGS.is_parsed():
        FLAGS.mark_as_parsed()
    base = dict(architecture="DenseNCSN", loss="dsm", num_layers=1, mlp_dims=256, data_shape=[str(SHAPE[0])],
                problem="vae", batch_size=4, epochs=2, snapshot_freq=2, eval_samples=4, num_sigmas=3, ld_steps=5,
                synthetic=True, synthetic_examples=24, logging_freq=1000, save_ckpt=False, verbose=False, seed=3)
    base.update(kw)
    return flagsaver.flagsaver(**base)


def _run(tmp_path, monkeypatch, **kw):
    """A stubbed train() over 2 epochs of 6 batches; returns the recorded train keys and sample() calls."""
    from smd_b200 import ebm_utils, input_pipeline, metrics, train_ncsn
    calls = {"train": [], "sample": [], "metrics": []}

    def train_step(objective, batch, optimizer, sigmas, rng, learning_rate, ema=None):
        calls["train"].append(np.asarray(rng).copy())
        return optimizer, {"loss": 0.0}

    def sample(scorenet, sigmas, rng, sample_shape, num_samples=2400, sampling="ald", epsilon=1e-3, steps=100,
               denoise=True, shard=None):
        calls["sample"].append(dict(rng=np.asarray(rng).copy(), n=num_samples, shard=shard, params=scorenet.arena))
        gen = torch.full((num_samples, *sample_shape), 0.5)
        coll = torch.zeros((102, num_samples, *sample_shape))
        coll[0] = -0.5
        return gen, coll, ebm_utils.collate_sampling_metrics(np.ones((4, len(sigmas), steps), np.float32))

    def latent_metrics(real, fake):
        calls["metrics"].append((np.asarray(real).shape, np.asarray(fake).shape))
        return dict(STUB_SCORES)

    monkeypatch.setattr(train_ncsn, "train_step", train_step)
    monkeypatch.setattr(train_ncsn, "evaluate", lambda *a: {"loss": 1.0})
    monkeypatch.setattr(train_ncsn, "sample", sample)
    monkeypatch.setattr(metrics, "latent_metrics", latent_metrics)
    with _flags(**kw):
        train_ds, eval_ds = input_pipeline.get_dataset(data_shape=SHAPE, problem="vae", batch_size=4, synthetic=True,
                                                       synthetic_examples=24, seed=3)
        sigmas = ebm_utils.create_noise_schedule(1.0, 0.01, 3, "geometric")
        opt = train_ncsn.train(train_ds, eval_ds, sigmas, str(tmp_path), verbose=False)
    return calls, opt


def reference_keys(seed, examples, epochs, snapshot_freq):
    """The key schedule of the reference's train() on jax 0.2.8 threefry: per step `rng, train_rng = split(rng)`, and
    at a snapshot `rng, eval_rng = split(rng)`, then `rng, sample_rng = split(rng)` with `rng` passed to sample().
    Returns (train keys, [(global_step, sample key, unused sample_rng)])."""
    rng = tf.prng_key(seed)
    rng = tf.split(rng, 3)[0]
    train_keys, snaps = [], []
    for epoch in range(epochs):
        for step in range(examples):
            rng, train_rng = tf.split(rng)
            train_keys.append(train_rng)
            if (step % snapshot_freq == 0 and step > 0) or step == examples - 1:
                rng = tf.split(rng)[0]
                rng, sample_rng = tf.split(rng)
                snaps.append((step + epoch * examples, rng, sample_rng))
    return train_keys, snaps


def test_hook_runs_at_the_reference_steps_with_the_reference_key(lib, tmp_path, monkeypatch):
    calls, opt = _run(tmp_path, monkeypatch)
    train_keys, snaps = reference_keys(3, 6, 2, 2)
    assert [s[0] for s in snaps] == [2, 4, 5, 8, 10, 11]
    np.testing.assert_array_equal(np.stack(calls["train"]), np.stack(train_keys))
    assert len(calls["sample"]) == len(snaps)
    for call, (_, key, unused) in zip(calls["sample"], snaps):
        np.testing.assert_array_equal(call["rng"], key)
        assert not np.array_equal(call["rng"], unused)
        assert call["n"] == 4 and call["shard"] == (0, 1)


def test_hook_samples_from_the_ema_arena(lib, tmp_path, monkeypatch):
    calls, opt = _run(tmp_path, monkeypatch, epochs=1)
    assert all(c["params"] is not opt.target.arena for c in calls["sample"])
    calls, opt = _run(tmp_path / "noema", monkeypatch, epochs=1, ema=False)
    assert all(c["params"] is opt.target.arena for c in calls["sample"])


def test_hook_writes_the_reference_file_tree(lib, tmp_path, monkeypatch):
    from smd_b200 import input_pipeline
    calls, _ = _run(tmp_path, monkeypatch)
    steps = [2, 4, 5, 8, 10, 11]
    for cat in ("init", "real", "fake"):
        assert sorted(os.listdir(tmp_path / "samples" / cat)) == sorted(f"{s}.pkl" for s in steps)
    assert sorted(d for d in os.listdir(tmp_path) if d.startswith("sampling_epoch")) == \
        [f"sampling_epoch{k}" for k in range(6)]
    ld = np.load(tmp_path / "sampling_epoch3" / "ld_metrics.npz")
    assert sorted(ld.files) == ["alpha", "noise", "slope", "step"] and ld["slope"].shape == (3, 5)
    lines = [json.loads(x) for x in open(tmp_path / "samples" / "metrics.jsonl")]
    assert [x["global_step"] for x in lines] == steps
    assert all({k: x[k] for k in STUB_SCORES} == STUB_SCORES for x in lines)
    assert calls["metrics"] == [((4,) + SHAPE, (4,) + SHAPE)] * 6
    # init is collection[0] and fake the final samples, both mapped back with the train split's min / max
    train_ds, eval_ds = input_pipeline.get_dataset(data_shape=SHAPE, problem="vae", batch_size=4, synthetic=True,
                                                   synthetic_examples=24, seed=3)
    inv = lambda v, ds: (v + 1.0) / 2.0 * (ds.max - ds.min) + ds.min  # noqa: E731
    init, fake = input_pipeline.load(tmp_path / "samples/init/5.pkl"), input_pipeline.load(tmp_path / "samples/fake/5.pkl")
    np.testing.assert_allclose(init, np.full((4,) + SHAPE, inv(-0.5, train_ds)), rtol=1e-6)
    np.testing.assert_allclose(fake, np.full((4,) + SHAPE, inv(0.5, train_ds)), rtol=1e-6)
    real = input_pipeline.load(tmp_path / "samples/real/5.pkl")
    assert real.shape == (4,) + SHAPE
    lo, hi = float(eval_ds.min), float(eval_ds.max)
    assert real.min() >= lo - 1e-5 and real.max() <= hi + 1e-5


def test_nosnapshot_sampling_writes_nothing(lib, tmp_path, monkeypatch):
    calls, _ = _run(tmp_path, monkeypatch, snapshot_sampling=False)
    assert calls["sample"] == [] and calls["metrics"] == []
    assert not os.path.exists(tmp_path / "samples")
    assert not [d for d in os.listdir(tmp_path) if d.startswith("sampling_epoch")]


def test_metrics_skipped_above_the_latent_stats_cap(lib, tmp_path, monkeypatch):
    calls, _ = _run(tmp_path, monkeypatch, epochs=1, eval_samples=8193)
    assert calls["sample"] and calls["metrics"] == []
    assert not os.path.exists(tmp_path / "samples" / "metrics.jsonl")
    assert os.path.exists(tmp_path / "samples" / "fake" / "5.pkl")


def test_dataset_take_leaves_the_next_pass_unchanged():
    from smd_b200 import input_pipeline
    a, _ = input_pipeline.get_dataset(data_shape=SHAPE, problem="vae", batch_size=4, synthetic=True,
                                      synthetic_examples=24, seed=1)
    b, _ = input_pipeline.get_dataset(data_shape=SHAPE, problem="vae", batch_size=4, synthetic=True,
                                      synthetic_examples=24, seed=1)
    first = a.take(6)
    assert first.shape == (6,) + SHAPE
    pass_a, pass_b = np.concatenate(list(a)), np.concatenate(list(b))
    np.testing.assert_array_equal(pass_a, pass_b)
    np.testing.assert_array_equal(first, pass_a[:6])
    assert a.take(1000).shape == (24,) + SHAPE
