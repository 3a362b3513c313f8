"""Snapshot sampling in train_ncsn.train on the GPU: the samples a snapshot writes equal a standalone chain on the
saved EMA arena with the key the hook derives (DenseNCSN with ALD / CAS, TransformerDDPM 32x42 with ALD / DDPM),
sampling leaves training alone, memory does not grow from one snapshot to the next, the logged metrics match the
pickles, the command line writes the reference's file tree, and a DDPM chain shorter than the 40 collection points
writes no row past the collection."""
import json
import os
import shutil
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch
from absl import flags
from absl.testing import flagsaver

from oracle import threefry as tf

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLAGS = flags.FLAGS

DENSE = dict(architecture="DenseNCSN", loss="dsm", num_layers=2, mlp_dims=256, data_shape=["64"], num_sigmas=3,
             sigma_begin=15.0, ld_steps=5, ld_epsilon=9.64e-7)
TRANSFORMER = dict(architecture="TransformerDDPM", loss="ddpm", num_layers=1, num_heads=8, num_mlp_layers=1,
                   mlp_dims=2048, data_shape=["32", "42"], num_sigmas=8, sigma_begin=1e-4, sigma_end=0.02,
                   schedule_type="linear", ld_steps=5)
CASES = {"dense-ald": dict(DENSE, sampling="ald"), "dense-cas": dict(DENSE, sampling="cas"),
         "transformer-ald": dict(TRANSFORMER, sampling="ald"), "transformer-ddpm": dict(TRANSFORMER, sampling="ddpm")}
# two snapshots (global steps 2 and 4) of a 16-row batch, 64 samples each
RUN = dict(problem="vae", batch_size=16, epochs=1, max_steps=4, snapshot_freq=2, eval_samples=64, synthetic=True,
           synthetic_examples=512, logging_freq=1000, verbose=False, seed=5, mu=0.9, learning_rate=1e-3)


def _flags(**kw):
    from smd_b200 import train_ncsn  # noqa: F401  (defines the flags)
    if not FLAGS.is_parsed():
        FLAGS.mark_as_parsed()
    return flagsaver.flagsaver(**dict(RUN, **kw))


def _data():
    from smd_b200 import ebm_utils, input_pipeline
    train_ds, eval_ds = input_pipeline.get_dataset(data_shape=FLAGS.data_shape, problem="vae",
                                                   batch_size=FLAGS.batch_size, synthetic=True,
                                                   synthetic_examples=FLAGS.synthetic_examples, seed=FLAGS.seed)
    sigmas = ebm_utils.create_noise_schedule(FLAGS.sigma_begin, FLAGS.sigma_end, FLAGS.num_sigmas, FLAGS.schedule_type)
    return train_ds, eval_ds, sigmas


def _train(out, **kw):
    """train() in this process; returns (optimizer, train_ds, eval_ds, sigmas) with the flags still applied."""
    from smd_b200 import train_ncsn
    train_ds, eval_ds, sigmas = _data()
    opt = train_ncsn.train(train_ds, eval_ds, sigmas, str(out), verbose=False)
    torch.cuda.synchronize()
    return opt, train_ds, eval_ds, sigmas


def snapshot_keys(seed, examples, snapshot_freq, max_steps):
    """{global step: key sample() receives}: train_ncsn.py's schedule on the jax 0.2.8 threefry restatement, `rng`
    after `rng, sample_rng = split(rng)`."""
    rng = tf.split(tf.prng_key(seed), 3)[0]
    keys = {}
    for step in range(examples):
        rng = tf.split(rng)[0]
        if (step % snapshot_freq == 0 and step > 0) or step == examples - 1:
            rng = tf.split(rng)[0]
            rng = tf.split(rng)[0]
            keys[step] = rng
        if step >= max_steps:
            break
    return keys


def _load(path):
    from smd_b200 import input_pipeline
    return input_pipeline.load(path)


def _standalone(out, k, key, shape, sigmas, train_ds, use_ema=True):
    """train_ncsn.sample on a freshly created inference model holding checkpoint k's EMA (or trained) arena, mapped
    back like the fake pickle."""
    from smd_b200 import checkpoints, input_pipeline, jrandom as random, train_ncsn, train_utils
    model = train_ncsn.create_model(random.PRNGKey(99), shape, train_ncsn.model_kwargs(), batch_size=1)
    opt = train_ncsn.create_optimizer(model, FLAGS.learning_rate)
    ema = train_utils.EMAHelper(mu=0, params=model.arena.clone())
    opt, ema, _ = checkpoints.restore_checkpoint(str(out), (opt, ema, train_utils.EarlyStopping()), step=k)
    net = model.replace(params=ema.params if use_ema else opt.target.arena)
    gen, _, _ = train_ncsn.sample(net, sigmas, key, shape, num_samples=FLAGS.eval_samples, sampling=FLAGS.sampling,
                                  epsilon=FLAGS.ld_epsilon, steps=FLAGS.ld_steps, denoise=FLAGS.denoise)
    return input_pipeline.inverse_data_transform(gen.cpu().numpy(), FLAGS.normalize, None, train_ds.min, train_ds.max,
                                                 out_channels=int(FLAGS.data_shape[-1]))


@pytest.mark.parametrize("case", sorted(CASES))
def test_fake_pickle_equals_a_standalone_chain_on_the_saved_ema(lib, tmp_path, case):
    with _flags(**CASES[case]):
        opt, train_ds, eval_ds, sigmas = _train(tmp_path)
        shape = tuple(int(s) for s in FLAGS.data_shape)
        keys = snapshot_keys(FLAGS.seed, train_ds.examples, FLAGS.snapshot_freq, FLAGS.max_steps)
        assert sorted(keys) == [2, 4]
        for k, step in enumerate(sorted(keys)):
            fake = _load(tmp_path / "samples" / "fake" / f"{step}.pkl")
            assert fake.shape == (FLAGS.eval_samples,) + shape and np.isfinite(fake).all()
            np.testing.assert_array_equal(fake, _standalone(tmp_path, k, keys[step], shape, sigmas, train_ds))
        # the EMA (mu = 0.9) has not caught up with the trained parameters: their samples differ
        raw = _standalone(tmp_path, 1, keys[4], shape, sigmas, train_ds, use_ema=False)
        assert not np.array_equal(fake, raw)


def test_noema_samples_the_trained_parameters(lib, tmp_path):
    with _flags(**CASES["dense-ald"], ema=False):
        opt, train_ds, _, sigmas = _train(tmp_path)
        shape = (64,)
        keys = snapshot_keys(FLAGS.seed, train_ds.examples, FLAGS.snapshot_freq, FLAGS.max_steps)
        fake = _load(tmp_path / "samples" / "fake" / "4.pkl")
        np.testing.assert_array_equal(fake, _standalone(tmp_path, 1, keys[4], shape, sigmas, train_ds, use_ema=False))


def test_snapshot_leaves_training_alone(lib, tmp_path, monkeypatch):
    from smd_b200 import jrandom as random, nn, train_ncsn
    run = {}
    hook = train_ncsn.snapshot_sampling

    def spy(optimizer, ema, *a, **kw):        # keeps the run's own EMA helper, the arena clip + Adam updates
        run["ema"] = ema
        return hook(optimizer, ema, *a, **kw)
    monkeypatch.setattr(train_ncsn, "snapshot_sampling", spy)
    with _flags(**CASES["dense-ald"]):
        opt, train_ds, eval_ds, sigmas = _train(tmp_path / "with")
    with _flags(**CASES["dense-ald"], snapshot_sampling=False):
        _train(tmp_path / "without")
        assert not os.path.exists(tmp_path / "without" / "samples")
    # checkpoint 0 is written before the first snapshot samples
    a = open(tmp_path / "with" / "checkpoint_0", "rb").read()
    b = open(tmp_path / "without" / "checkpoint_0", "rb").read()
    assert a == b

    with _flags(**CASES["dense-ald"]):
        eng = [e for e in opt.target.module._engines if e.training]
        assert len(eng) == 1
        eng = eng[0]
        batch = nn._as_device_f32(next(iter(train_ds)))
        key = random.PRNGKey(123)

        def grads():
            used, eps = eng.dsm_draws((int(key[0]), int(key[1])), batch.shape[0], global_batch=batch.shape[0])
            eng.compute_dsm_grads(batch, used, eps, global_batch=batch.shape[0])
            torch.cuda.synchronize()
            return eng.grads.clone(), eng.loss_sum.clone()

        ema = run["ema"]
        g0, l0 = grads()
        state0 = [t.clone() for t in (eng._ws, eng.params, ema.params.flat, opt.grad_ema, opt.grad_sq_ema)]
        rng = hook(opt, ema, sigmas, random.PRNGKey(7), (64,), train_ds, eval_ds, 100, 9,
                                           str(tmp_path / "with"))
        torch.cuda.synchronize()
        state1 = [t.clone() for t in (eng._ws, eng.params, ema.params.flat, opt.grad_ema, opt.grad_sq_ema)]
        for x, y in zip(state0, state1):
            assert torch.equal(x, y)
        g1, l1 = grads()
        assert torch.equal(g0, g1) and torch.equal(l0, l1)
        mem1 = torch.cuda.memory_allocated()
        # a second snapshot allocates nothing that outlives it
        hook(opt, ema, sigmas, rng, (64,), train_ds, eval_ds, 101, 10, str(tmp_path / "with"))
        torch.cuda.synchronize()
        assert torch.cuda.memory_allocated() == mem1
        # the sampler ran on one inference engine whose max_batch holds the snapshot's samples
        samplers = [e for e in opt.target.module._engines if not e.training and e.max_batch >= FLAGS.eval_samples]
        assert len(samplers) == 1


@pytest.mark.parametrize("case", ["dense-ald", "transformer-ddpm"])
def test_metrics_jsonl_matches_the_pickles(lib, tmp_path, case):
    from smd_b200 import input_pipeline, metrics
    with _flags(**CASES[case]):
        _, train_ds, eval_ds, _ = _train(tmp_path)
        lines = [json.loads(x) for x in open(tmp_path / "samples" / "metrics.jsonl")]
        assert [x["global_step"] for x in lines] == [2, 4]
        for line in lines:
            step = line["global_step"]
            real = input_pipeline.normalize_dataset(_load(tmp_path / f"samples/real/{step}.pkl"), eval_ds.min,
                                                    eval_ds.max).astype(np.float32)
            fake = input_pipeline.normalize_dataset(_load(tmp_path / f"samples/fake/{step}.pkl"), train_ds.min,
                                                    train_ds.max).astype(np.float32)
            want = metrics.latent_metrics(real, fake)
            for k, v in want.items():
                assert line[k] == pytest.approx(v, rel=1e-3, abs=1e-5), k


def test_rejected_chain_raises_at_the_first_snapshot(lib, tmp_path):
    from smd_b200 import jrandom as random, train_ncsn
    with _flags(**dict(CASES["dense-ald"], ld_steps=0)):
        with pytest.raises(ValueError, match="steps_per_level out of range"):
            _train(tmp_path)
        assert os.path.exists(tmp_path / "checkpoint_0") and not os.path.exists(tmp_path / "checkpoint_1")
        # the same message as a standalone sample() (what sample_ncsn runs)
        model = train_ncsn.create_model(random.PRNGKey(1), (64,), train_ncsn.model_kwargs(), batch_size=1)
        with pytest.raises(ValueError, match="steps_per_level out of range"):
            train_ncsn.sample(model, [15.0, 1.0, 0.01], random.PRNGKey(2), (64,), num_samples=8, steps=0)


def test_short_ddpm_chain_writes_only_collection_rows(lib):
    """Below T = 40, linspace(1, T, 40) repeats indices and the reference's summed slot passes the 41 collection rows
    (up to 184 at T = 8); XLA's scatter drops those updates.  The chain must write rows 1..40 at the slots the rule
    leaves in range and nothing behind them."""
    from smd_b200 import Engine, ModelConfig, ebm_utils
    eng = Engine(ModelConfig(arch="TransformerDDPM", num_layers=1, num_mlp_layers=1, seq_len=32, channels=42),
                 max_batch=4)
    eng.set_params(eng.init_params(seed=2, perturb=0.02))
    T = 8
    eng.sampler_setup(ebm_utils.create_noise_schedule(1e-4, 0.02, T, "linear"), key=(0, 3))
    idx = np.linspace(1, T, 40).astype(np.int32)
    slots = [int(np.sum(np.arange(40) * (idx == T - t + 1))) + 1 for t in range(T) if (idx == T - t + 1).any()]
    assert max(slots) == 184
    want = sorted(s for s in slots if s < 41)
    x = torch.from_numpy(np.random.default_rng(0).uniform(-1, 1, (4, 32, 42)).astype(np.float32)).cuda()
    guarded = torch.full((200, 4, 32, 42), -7.0, device="cuda")          # 41 rows, then 159 guard rows
    eng.sample(x, steps=T, collection=guarded, metrics=torch.zeros((4, T), device="cuda"))
    torch.cuda.synchronize()
    written = [r for r in range(200) if not bool((guarded[r] == -7.0).all())]
    assert written == want == [40]
    assert torch.isfinite(guarded[40]).all() and torch.isfinite(x).all()


# ------------------------------------------------------------------------------------------------- command lines
MEL_FLAGS = """\
    --architecture=DenseNCSN
    --epochs=1
    --sigma_begin=15
    --num_sigmas=3
    --ld_epsilon=9.64e-7
    --ld_steps=5
    --problem=vae
    --ema
    --normalize
    --data_shape=64
    --model_dir={run}
    --num_layers=2
    --mlp_dims=256
    --batch_size=16
    --max_steps=4
    --snapshot_freq=2
    --eval_samples=64
    --synthetic
    --synthetic_examples=512
    """


def _cli(tmp_path, name, launcher=()):
    cfg = tmp_path / f"{name}.cfg"
    cfg.write_text(textwrap.dedent(MEL_FLAGS).format(run=tmp_path / name))
    env = dict(os.environ, PYTHONPATH=ROOT)
    cmd = list(launcher) + ([sys.executable, "-m"] if not launcher else ["-m"]) + ["smd_b200.train_ncsn",
                                                                                f"--flagfile={cfg}"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    return tmp_path / name


def test_train_ncsn_command_line_writes_the_snapshot_tree(lib, tmp_path):
    run = _cli(tmp_path, "mel")
    for step in (2, 4):
        for cat in ("init", "real", "fake"):
            a = _load(run / "samples" / cat / f"{step}.pkl")
            assert a.shape == (64, 64) and np.isfinite(a).all()
    for k in (0, 1):
        ld = np.load(run / f"sampling_epoch{k}" / "ld_metrics.npz")
        assert ld["slope"].shape == (3, 5) and np.isfinite(ld["slope"]).all()
    lines = [json.loads(x) for x in open(run / "samples" / "metrics.jsonl")]
    assert [x["global_step"] for x in lines] == [2, 4]
    assert all(np.isfinite(x["frechet_distance"]) for x in lines)


def test_two_ranks_gather_the_single_rank_samples(lib, tmp_path):
    if torch.cuda.device_count() < 2 or shutil.which("torchrun") is None:
        pytest.skip("the torchrun comparison needs 2 GPUs")
    two = _cli(tmp_path, "two", launcher=("torchrun", "--nproc-per-node", "2"))
    # the gathered rows equal one process's chain on the same checkpoint (the data-parallel gradient sum need not
    # round like the single-rank one, so the comparison is on the two-rank run's own EMA arena)
    with _flags(**CASES["dense-ald"], seed=0, mu=0.999, learning_rate=3e-4):
        train_ds, _, sigmas = _data()
        keys = snapshot_keys(0, train_ds.examples, 2, 4)
        for k, step in enumerate((2, 4)):
            np.testing.assert_array_equal(_load(two / "samples/fake" / f"{step}.pkl"),
                                          _standalone(two, k, keys[step], (64,), sigmas, train_ds))
