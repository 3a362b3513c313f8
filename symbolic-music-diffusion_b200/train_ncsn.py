"""Training entry point with the reference's flag surface (train_ncsn.py:48-128), so configs/ddpm-*.cfg run
unchanged:  python -m smd_b200.train_ncsn --flagfile=configs/ddpm-mel-32seq-512.cfg [--synthetic]

Objectives: --loss=ddpm (TransformerDDPM, TransformerDDPM4, DenseDDPM), --loss=dsm and --loss=ssm (DenseNCSN; ssm
with any other architecture raises ValueError).  Other values raise ValueError exactly where the reference would
dispatch on them.  Data-parallel: launch with torchrun (one process per GPU); the batch is sharded across ranks
and gradients are summed with one NCCL all-reduce over the flat arena (SURVEY section 8(e)).
--snapshot_sampling (the default, as in the reference) draws --eval_samples samples from the EMA parameters at every
snapshot and writes them under --model_dir (snapshot_sampling).
"""
from __future__ import annotations

import functools
import json
import os
import time

import numpy as np
import torch
from absl import app, flags, logging

from smd_b200 import (checkpoints, ebm_utils, input_pipeline, jrandom as random, metrics, ncsn, nn, optim, parallel,
                      train_utils)
from smd_b200.losses import denoising_score_matching_loss, diffusion_loss, sliced_score_matching_loss

FLAGS = flags.FLAGS
_D = flags.DEFINE_integer, flags.DEFINE_float, flags.DEFINE_bool, flags.DEFINE_string, flags.DEFINE_enum

# --- optimisation ------------------------------------------------------------------------------------------
flags.DEFINE_integer("seed", 0, "PRNG seed (jax.random.PRNGKey).")
flags.DEFINE_enum("loss", "dsm", ["dsm", "ssm", "ddpm"], "Training objective.")
flags.DEFINE_bool("continuous_noise", True, "Condition on the continuous noise level sqrt(alpha_bar).")
flags.DEFINE_float("learning_rate", 3e-4, "Base learning rate.")
flags.DEFINE_integer("batch_size", 128, "GLOBAL batch size (sharded over ranks when launched with torchrun).")
flags.DEFINE_integer("epochs", 10, "Number of epochs.")
flags.DEFINE_integer("max_steps", None, "Stop after this many optimizer steps.")
flags.DEFINE_bool("early_stopping", False, "Stop on a non-improving evaluation loss.")
flags.DEFINE_float("grad_clip", 1.0, "Global-norm gradient clipping threshold.")
flags.DEFINE_float("lr_gamma", 0.98, "Multiplicative LR decay per interval.")
flags.DEFINE_integer("lr_schedule_interval", 10000, "Steps per LR decay interval.")
# --- model -------------------------------------------------------------------------------------------------
flags.DEFINE_string("architecture", "TransformerDDPM", "Score-network class name in models/ncsn.py.")
flags.DEFINE_integer("num_layers", 6, "Transformer layers (or DenseDDPM res-blocks).")
flags.DEFINE_integer("num_heads", 8, "Attention heads.")
flags.DEFINE_integer("num_mlp_layers", 2, "FiLM residual MLP blocks after the trunk.")
flags.DEFINE_integer("mlp_dims", 2048, "Width of the residual MLP blocks.")
# --- noise schedule / sampling -----------------------------------------------------------------------------
flags.DEFINE_float("sigma_begin", 1.0, "First value of the noise schedule.")
flags.DEFINE_float("sigma_end", 1e-2, "Last value of the noise schedule.")
flags.DEFINE_enum("schedule_type", "geometric", ["geometric", "linear", "fibonacci"], "Noise schedule.")
flags.DEFINE_integer("num_sigmas", 15, "Length of the noise schedule.")
flags.DEFINE_integer("ld_steps", 100, "Langevin steps per noise level (null for ddpm).")
flags.DEFINE_float("ld_epsilon", 2e-6, "Langevin step size (null for ddpm).")
flags.DEFINE_enum("sampling", "ald", ["ald", "cas", "ddpm", "ddim", "dpm"],
                  "Sampling algorithm (ddim and dpm are additions of this implementation, see --ddim_steps and "
                  "--dpm_steps).")
flags.DEFINE_bool("ema", True, "Track an exponential moving average of the parameters.")
flags.DEFINE_float("mu", 0.999, "EMA momentum.")
flags.DEFINE_bool("denoise", True, "Expected-denoised-sample step (null for ddpm).")
# --- data --------------------------------------------------------------------------------------------------
flags.DEFINE_list("data_shape", [2], "Shape of one example, e.g. 32,512.")
flags.DEFINE_enum("problem", "toy", ["toy", "mnist", "vae"], "Problem family.")
flags.DEFINE_string("dataset", "./output/mix2d", "Dataset directory ({train,eval}-*.tfrecord).")
flags.DEFINE_string("pca_ckpt", "", "PCA transform pickle.")
flags.DEFINE_string("slice_ckpt", "", "Pickle of latent dimensions to keep.")
flags.DEFINE_string("dim_weights_ckpt", "", "Pickle of per-dimension weights.")
flags.DEFINE_bool("normalize", True, "Min/max normalise to [-1, 1].")
# --- logging / checkpoints ---------------------------------------------------------------------------------
flags.DEFINE_integer("logging_freq", 100, "Steps between log lines.")
flags.DEFINE_integer("snapshot_freq", 5000, "Steps between evaluation + checkpoint.")
flags.DEFINE_bool("snapshot_sampling", True, "Sample at every snapshot.")
flags.DEFINE_integer("eval_samples", 3000, "Samples drawn at a snapshot.")
flags.DEFINE_integer("checkpoints_to_keep", 50, "Checkpoints retained.")
flags.DEFINE_bool("save_ckpt", True, "Write checkpoints.")
flags.DEFINE_string("model_dir", "./save/ncsn", "Output directory.")
flags.DEFINE_bool("verbose", True, "Verbose logging.")
# --- additions of this implementation (not in the reference) ------------------------------------------------
flags.DEFINE_bool("synthetic", False, "Use synthetic N(0,1) latents of --data_shape instead of reading --dataset.")
flags.DEFINE_integer("synthetic_examples", 4096, "Examples per split with --synthetic.")
flags.DEFINE_integer("ddim_steps", 50, "--sampling=ddim: noise levels of the DDPM schedule the chain visits.")
flags.DEFINE_float("ddim_eta", 0.0, "--sampling=ddim: noise scale (0: deterministic; 1 with all levels: ddpm).")
flags.DEFINE_enum("ddim_schedule", "uniform", ["uniform", "quadratic"], "--sampling=ddim: spacing of the levels.")
flags.DEFINE_integer("dpm_steps", 20, "--sampling=dpm: noise levels of the DDPM schedule the DPM-Solver++ chain "
                     "visits.")
flags.DEFINE_integer("dpm_order", 2, "--sampling=dpm: solver order (1: the DDIM eta = 0 step).", lower_bound=1,
                     upper_bound=3)
flags.DEFINE_enum("dpm_schedule", "uniform", ["uniform", "quadratic"], "--sampling=dpm: spacing of the levels.")


def model_kwargs():
    return dict(num_layers=FLAGS.num_layers, num_heads=FLAGS.num_heads, num_mlp_layers=FLAGS.num_mlp_layers,
                mlp_dims=FLAGS.mlp_dims)


def create_optimizer(model, learning_rate):
    """train_ncsn.py:187-190."""
    return optim.Adam(learning_rate=learning_rate).create(model)


def create_model(rng, input_shape, model_kwargs, batch_size=32, verbose=False):
    """train_ncsn.py:193-203: getattr(ncsn, FLAGS.architecture).partial(**kw).init_by_shape(...) -> nn.Model."""
    clazz = getattr(ncsn, FLAGS.architecture, None)
    if clazz is None:
        raise ValueError(f"Unknown architecture {FLAGS.architecture!r} (models/ncsn.py has no such class)")
    module = clazz.partial(**model_kwargs)
    _, params = module.init_by_shape(rng, [((batch_size, *input_shape), np.float32),
                                           ((batch_size, *([1] * len(input_shape))), np.float32)])
    model = nn.Model(module, params)
    if verbose:
        train_utils.report_model(model)
    return model


def _objective():
    if FLAGS.loss == "ddpm":
        return diffusion_loss
    if FLAGS.loss == "dsm":
        return denoising_score_matching_loss
    if FLAGS.loss == "ssm":
        # sliced score matching (utils/losses.py:182-247): its Jacobian-vector product and second-order backward are
        # written for the dense score network only
        if FLAGS.architecture != "DenseNCSN":
            raise ValueError(f"--loss=ssm needs --architecture=DenseNCSN (got {FLAGS.architecture})")
        return sliced_score_matching_loss
    raise ValueError(f"Unsupported objective {FLAGS.loss}")


def eval_step(objective, batch, model, sigmas, rng):
    """train_ncsn.py:206-221: summed loss of one batch."""
    return objective(batch, model, sigmas, rng, FLAGS.continuous_noise, "sum")


def evaluate(dataset, model, sigmas, rng):
    """train_ncsn.py:224-257."""
    objective = _objective()
    count, total = 0, 0.0
    for inputs in dataset:
        count += inputs.shape[0]
        rng, eval_rng = random.split(rng)
        total += float(eval_step(objective, inputs, model, sigmas, eval_rng))
    return {"loss": total / max(count, 1)}


def lr_at(step: int) -> float:
    """flax create_stepped_learning_rate_schedule as called at train_ncsn.py:340-342, evaluated at the 0-based
    global step like lr_scheduler(global_step) at train_ncsn.py:362: lr0 * gamma^max(0, ceil(step/interval) - 1)."""
    n = 0 if step <= 0 else (step - 1) // FLAGS.lr_schedule_interval
    return FLAGS.learning_rate * (FLAGS.lr_gamma ** n)


def train_step(objective, batch, optimizer, sigmas, rng, learning_rate, ema=None):
    """train_ncsn.py:260-288 on this rank's shard: grads -> all-reduce -> clip -> Adam (one fused pass)."""
    if objective not in (diffusion_loss, denoising_score_matching_loss, sliced_score_matching_loss):
        raise ValueError("only the ddpm, dsm and ssm objectives have a hand-written backward")
    ssm = objective is sliced_score_matching_loss
    dsm = objective is denoising_score_matching_loss
    model = optimizer.target
    world, rank = parallel.world_size(), parallel.rank()
    x0 = nn._as_device_f32(batch)
    local = x0.shape[0]
    eng = model.engine(local, training=True)
    betas = np.asarray(sigmas, np.float32)
    if dsm or ssm:
        if getattr(eng, "_dsm_sigmas", None) is None or not np.array_equal(eng._dsm_sigmas, betas):
            eng.dsm_setup(betas)
            eng._dsm_sigmas = betas.copy()
    elif getattr(eng, "_obj_betas", None) is None or not np.array_equal(eng._obj_betas, betas):
        eng.objective_setup(betas)
        eng._obj_betas = betas.copy()
    if not hasattr(eng, "grads"):
        eng.init_train_state(ema=False)
    # every rank holds the SAME key and consumes rows [rank*local, (rank+1)*local) of the global batch's threefry
    # streams (labels, alpha-bar, eps): an N-GPU run with seed s sees exactly the noise of the 1-GPU run with seed s
    if ssm:
        used, eps, v = eng.ssm_draws((int(rng[0]), int(rng[1])), local, global_batch=local * world,
                                     first_row=rank * local, continuous_noise=FLAGS.continuous_noise)
        eng.compute_ssm_grads(x0, used, eps, v, global_batch=local * world)
    elif dsm:
        used, eps = eng.dsm_draws((int(rng[0]), int(rng[1])), local, global_batch=local * world, first_row=rank * local,
                                  continuous_noise=FLAGS.continuous_noise)
        eng.compute_dsm_grads(x0, used, eps, global_batch=local * world)
    else:
        used, eps = eng.draws((int(rng[0]), int(rng[1])), local, global_batch=local * world, first_row=rank * local,
                              continuous_noise=FLAGS.continuous_noise)
        eng.compute_grads(x0, used, eps, global_batch=local * world)
    eng.reduce_grads(world)     # tail gradients are reduced underneath the trunk backward
    optimizer.apply_gradient(eng.grads, learning_rate=learning_rate, max_norm=FLAGS.grad_clip, ema=ema, mu=FLAGS.mu,
                             engine=eng)
    metrics = {"loss": eng.loss_mean, "grad": optimizer.grad_norm, "lr": learning_rate}
    return optimizer, metrics


def _summary_writer(path):
    """A tensorboard SummaryWriter logging to `path`, or None when tensorboard cannot be imported (it is optional)."""
    try:
        from torch.utils.tensorboard import SummaryWriter
        return SummaryWriter(path)
    except Exception:
        return None


LD_METRICS = ("slope", "step", "alpha", "noise")


def log_langevin_dynamics(ld_metrics, step, output_dir):
    """train_ncsn.py:166-184: the per-step statistics of one sampling run, `ld_metrics` as collate_sampling_metrics
    returns them (num_sigmas lists of T dicts).  Logged to a SummaryWriter under output_dir/sampling_epoch{step} when
    tensorboard is available, and always written there as ld_metrics.npz: one (num_sigmas, T) float32 array per
    statistic (slope, step, alpha, noise)."""
    out = os.path.join(output_dir, f"sampling_epoch{step}")
    os.makedirs(out, exist_ok=True)
    arrays = {k: np.asarray([[m[k] for m in level] for level in ld_metrics], np.float32) for k in LD_METRICS}
    np.savez(os.path.join(out, "ld_metrics.npz"), **arrays)
    writer = _summary_writer(out)
    if writer is not None:
        for i, sigma_metrics in enumerate(ld_metrics):
            for j, metric in enumerate(sigma_metrics):
                train_utils.log_metrics(metric, j, len(sigma_metrics), epoch=i, summary_writer=writer, verbose=False)
        writer.close()
    return out


def log_samples(step, init, real, fake, output_dir, flush=True):
    """train_ncsn.py:137-163 without the image tiles and scatter plots (out of scope): with `flush`, each set is
    pickled to output_dir/samples/{init,real,fake}/{step}.pkl."""
    if flush:
        for category, samples in (("init", init), ("real", real), ("fake", fake)):
            input_pipeline.save(samples, os.path.join(output_dir, f"samples/{category}/{step}.pkl"))


LATENT_STATS_MAX_ROWS = 16384      # n + m cap of smd_latent_stats (include/smd.h)


def snapshot_sampling(optimizer, ema, sigmas, rng, input_shape, train_batches, valid_batches, global_step,
                      sampling_step, output_dir, writer=None):
    """train_ncsn.py:405-486: draws --eval_samples samples from the EMA parameters (the trained ones with --noema),
    logs the Langevin statistics, and writes the initial, real and generated sets.  Returns the advanced `rng`.

    The samples come from the spec's inference engine, which packs its bf16 operands from the EMA arena on the device
    whenever the arena's version has moved; the training engine is not used.  Every rank draws its rows of the
    sample (shard=(rank, world), like sample_ncsn.generate_samples), the rows are gathered, and rank 0 alone does the
    host work.  Deviations from the reference:
      - `real` is the first --eval_samples examples of the next pass over `valid_batches`.  Upstream takes them after
        a tf.data shuffle(8 * batch_size) of the unbatched split, which cannot be restated.  A smaller split gives
        fewer real rows than init and fake (logged as a warning); upstream's log_samples asserts equal shapes.
      - The pickles are written for every problem (upstream: vae only); the image tiles, scatter plots and score
        fields are not drawn.
      - The final samples are scored against `real` on the normalised data with metrics.latent_metrics, logged and
        appended with global_step to output_dir/samples/metrics.jsonl.  Scoring is skipped with a warning when
        2 * --eval_samples exceeds the 16384 rows smd_latent_stats takes."""
    scorenet = optimizer.target.replace(params=ema.params if FLAGS.ema else optimizer.target.arena)
    # upstream splits off sample_rng but hands `rng` itself to sample() (train_ncsn.py:407-411); reproduced here, so
    # the sampling key is the training key's next state
    rng, sample_rng = random.split(rng)
    del sample_rng
    world, rank = parallel.world_size(), parallel.rank()
    generated, collection, ld_metrics = sample(scorenet, sigmas, rng, input_shape, num_samples=FLAGS.eval_samples,
                                               sampling=FLAGS.sampling, epsilon=FLAGS.ld_epsilon, steps=FLAGS.ld_steps,
                                               denoise=FLAGS.denoise, shard=(rank, world))
    generated = parallel.gather_rows(generated)
    init = None if collection is None else parallel.gather_rows(collection[0].contiguous())
    if rank != 0:
        return rng
    if init is None:
        # consistent Langevin dynamics keeps no collection: regenerate the initial draw from sample()'s init_rng
        init = initial_draw(random.split(rng)[0], (FLAGS.eval_samples, *input_shape), FLAGS.sampling)
    generated, init = generated.cpu().numpy(), init.cpu().numpy()
    real = valid_batches.take(FLAGS.eval_samples)
    if len(real) < FLAGS.eval_samples:
        logging.warning("the validation split holds %d examples: the real set is smaller than --eval_samples=%d",
                        len(real), FLAGS.eval_samples)
    if output_dir:
        log_langevin_dynamics(ld_metrics, sampling_step, output_dir)
        load = lambda p: input_pipeline.load(os.path.expanduser(p)) if p else None  # noqa: E731
        pca, slice_idx, dim_w = load(FLAGS.pca_ckpt), load(FLAGS.slice_ckpt), load(FLAGS.dim_weights_ckpt)

        def inv(a, ds):
            return input_pipeline.inverse_data_transform(a, FLAGS.normalize, pca, ds.min, ds.max, slice_idx, dim_w,
                                                         out_channels=int(FLAGS.data_shape[-1]))
        log_samples(global_step, inv(init, train_batches), inv(real, valid_batches), inv(generated, train_batches),
                    output_dir, flush=True)
    if 2 * FLAGS.eval_samples > LATENT_STATS_MAX_ROWS:
        logging.warning("snapshot metrics skipped: 2 * --eval_samples=%d exceeds the %d rows the GPU metrics take",
                        FLAGS.eval_samples, LATENT_STATS_MAX_ROWS)
        return rng
    scores = metrics.latent_metrics(real, generated)
    train_utils.log_metrics(scores, global_step, train_batches.examples * FLAGS.epochs, summary_writer=writer)
    if output_dir:
        with open(os.path.join(output_dir, "samples", "metrics.jsonl"), "a") as f:
            f.write(json.dumps({"global_step": int(global_step), **scores}) + "\n")
    return rng


def train(train_batches, valid_batches, sigmas, output_dir=None, verbose=True):
    """train_ncsn.py:291-496 (the MNIST / toy plotting branches are out of scope)."""
    objective = _objective()
    if torch.cuda.is_available() and torch.cuda.current_stream().cuda_stream == 0:
        # the legacy default stream cannot be captured: a private stream lets libsmd replay the step from a CUDA graph
        torch.cuda.set_stream(torch.cuda.Stream())
    first = next(iter(valid_batches))
    input_shape = tuple(first.shape[1:])
    rng = random.PRNGKey(FLAGS.seed)
    rng, model_rng, _ = random.split(rng, 3)
    local_bs = parallel.shard_size(FLAGS.batch_size)
    model = create_model(model_rng, input_shape, model_kwargs(), batch_size=local_bs, verbose=verbose)
    optimizer = create_optimizer(model, FLAGS.learning_rate)
    ema = train_utils.EMAHelper(FLAGS.mu, model.arena.clone()) if FLAGS.ema else None
    early_stop = train_utils.EarlyStopping(patience=1)
    writer = None
    if output_dir and parallel.rank() == 0:
        os.makedirs(output_dir, exist_ok=True)
        writer = _summary_writer(os.path.join(output_dir, "train"))
    examples = train_batches.examples            # batches per epoch (utils/data_utils.py:63-90)

    class _LocalRows:                            # rows [rank*B/W, (rank+1)*B/W) of every global batch
        def __iter__(self_inner):
            return (parallel.shard_rows(b) for b in train_batches)
    # input_pipeline.py:209-210 prefetch: pinned staging + host->device copy on a side stream, 2 batches ahead
    loader = input_pipeline.DevicePrefetcher(_LocalRows(), depth=2)
    sampling_step = -1
    for epoch in range(FLAGS.epochs):
        start_time = time.time()
        for step, batch in enumerate(loader):                           # this rank's rows, already on the device
            rng, train_rng = random.split(rng)
            global_step = step + epoch * examples                       # train_ncsn.py:359 (0-based)
            optimizer, metrics = train_step(objective, batch, optimizer, sigmas, train_rng,
                                            lr_at(global_step), ema)    # EMA (train_ncsn.py:364-365) is fused in
            if step % FLAGS.logging_freq == 0 and parallel.rank() == 0:
                elapsed = time.time() - start_time
                metrics.update({"batch/s": (step + 1) / elapsed, "ms/batch": elapsed * 1000 / (step + 1)})
                train_utils.log_metrics(metrics, step, examples, epoch=epoch, summary_writer=writer, verbose=verbose)
            if (step % FLAGS.snapshot_freq == 0 and step > 0) or step == examples - 1:     # train_ncsn.py:380-381
                sampling_step += 1
                rng, eval_rng = random.split(rng)
                ev = evaluate(valid_batches, optimizer.target, sigmas, eval_rng)
                improved, early_stop = early_stop.update(ev["loss"])
                if parallel.rank() == 0:
                    train_utils.log_metrics(ev, global_step, examples * FLAGS.epochs, summary_writer=None,
                                            verbose=verbose)
                    # train_ncsn.py:395-399: with --early_stopping only improved models are written
                    if FLAGS.save_ckpt and output_dir and (not FLAGS.early_stopping or improved):
                        checkpoints.save_checkpoint(output_dir, (optimizer, ema, early_stop), sampling_step,
                                                    keep=FLAGS.checkpoints_to_keep)
                if FLAGS.early_stopping and early_stop.should_stop:
                    logging.info("EARLY STOP: Ended training after %s epochs.", epoch + 1)
                    return optimizer
                if FLAGS.snapshot_sampling:                                 # train_ncsn.py:405-486
                    rng = snapshot_sampling(optimizer, ema, sigmas, rng, input_shape, train_batches, valid_batches,
                                            global_step, sampling_step, output_dir, writer)
            if FLAGS.max_steps is not None and global_step >= FLAGS.max_steps:             # train_ncsn.py:492-494
                if writer is not None:
                    writer.flush()
                return optimizer
    if writer is not None:
        writer.flush()
    return optimizer


def sample(scorenet, sigmas, rng, sample_shape, num_samples=2400, sampling="ald", epsilon=1e-3, steps=100,
           denoise=True, shard=None):
    """train_ncsn.py:499-551: initial noise from `rng`, dispatch on the sampler, collate metrics.

    shard=(rank, world) (not in the reference): this process generates rows [rank*n/world, (rank+1)*n/world) of the
    num_samples-sample run -- its slice of the initial draw and of every step's noise stream."""
    if sampling == "ddpm":
        algorithm = ebm_utils.diffusion_dynamics
    elif sampling == "ddim":
        algorithm = ddim_algorithm()
    elif sampling == "dpm":
        algorithm = dpm_algorithm()
    elif sampling == "ald":
        algorithm = ebm_utils.annealed_langevin_dynamics
    elif sampling == "cas":
        algorithm = ebm_utils.consistent_langevin_dynamics
    else:
        raise ValueError(f"Unknown sampling algorithm: {sampling}")
    init_rng, ld_rng = random.split(rng)
    rows, kw = None, {}
    if shard is not None and shard[1] > 1:
        local = parallel.shard_size(num_samples)
        rows, kw = (shard[0] * local, local), dict(shard=(shard[0] * local, num_samples))
    init = initial_draw(init_rng, (num_samples, *sample_shape), sampling, rows=rows)
    generated, collection, ld_metrics = algorithm(ld_rng, scorenet, sigmas, init, epsilon, steps, denoise, False, **kw)
    return generated, collection, ebm_utils.collate_sampling_metrics(ld_metrics)


def ddim_algorithm():
    """ebm_utils.ddim_dynamics with --ddim_steps, --ddim_eta and --ddim_schedule bound: the signature of the other
    samplers."""
    return functools.partial(ebm_utils.ddim_dynamics, steps=FLAGS.ddim_steps, eta=FLAGS.ddim_eta,
                             schedule=FLAGS.ddim_schedule)


def dpm_algorithm():
    """ebm_utils.dpm_solver_dynamics with --dpm_steps, --dpm_order and --dpm_schedule bound: the signature of the other
    samplers."""
    return functools.partial(ebm_utils.dpm_solver_dynamics, steps=FLAGS.dpm_steps, order=FLAGS.dpm_order,
                             schedule=FLAGS.dpm_schedule)


def initial_draw(init_rng, shape, sampling, rows=None):
    """The start of sample()'s chain (train_ncsn.py:541-549): N(0, 1) for ddpm, ddim and dpm, otherwise uniform with
    zero mean and unit variance.  rows=(first, count): only those rows of the draw."""
    if sampling not in ("ddpm", "ddim", "dpm"):
        rho = float(np.sqrt(np.float32(12)) / 2)
        return random.uniform(init_rng, shape, -rho, rho, rows=rows)
    return random.normal(init_rng, shape, rows=rows)


def main(argv):
    del argv
    parallel.init_from_env()
    logging.info("platform: cuda (%s), ranks: %d", torch.cuda.get_device_name() if torch.cuda.is_available() else "none",
                 parallel.world_size())
    train_ds, eval_ds = input_pipeline.get_dataset(
        dataset=FLAGS.dataset, data_shape=FLAGS.data_shape, problem=FLAGS.problem, batch_size=FLAGS.batch_size,
        normalize=FLAGS.normalize, pca_ckpt=FLAGS.pca_ckpt, slice_ckpt=FLAGS.slice_ckpt,
        dim_weights_ckpt=FLAGS.dim_weights_ckpt, synthetic=FLAGS.synthetic,
        synthetic_examples=FLAGS.synthetic_examples, seed=FLAGS.seed)
    sigmas = ebm_utils.create_noise_schedule(FLAGS.sigma_begin, FLAGS.sigma_end, FLAGS.num_sigmas, FLAGS.schedule_type)
    train(train_ds, eval_ds, sigmas, FLAGS.model_dir, FLAGS.verbose)
    parallel.shutdown()


if __name__ == "__main__":
    app.run(main)
