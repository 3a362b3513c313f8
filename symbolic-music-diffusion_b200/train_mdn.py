"""Training entry point of the autoregressive baseline with the reference's flag surface (train_mdn.py:49-97), so
configs/mdn-*.cfg run unchanged:  python -m smd_b200.train_mdn --flagfile=configs/mdn-mel-32seq-512.cfg [--synthetic]

TransformerMDN only, sequences of 32 latents, bf16 tensor-core operands.  Data-parallel: launch with torchrun (one
process per GPU); the batch is sharded across ranks and gradients are summed with one NCCL all-reduce over the flat
arena, as in train_ncsn.  This module does not import train_ncsn: both define the same absl flag names.
"""
from __future__ import annotations

import os
import time

import numpy as np
import torch
from absl import app, flags, logging

from smd_b200 import autoregressive as ar
from smd_b200 import checkpoints, input_pipeline, jrandom as random, lib as _lib, nn, optim, parallel, train_utils
from smd_b200.losses import reduce_fn

FLAGS = flags.FLAGS

flags.DEFINE_integer("seed", 0, "Random seed for network initialization.")
# --- training ----------------------------------------------------------------------------------------------
flags.DEFINE_float("learning_rate", 3e-4, "Learning rate for optimizer.")
flags.DEFINE_integer("batch_size", 128, "GLOBAL batch size (sharded over ranks when launched with torchrun).")
flags.DEFINE_integer("epochs", 1000, "Number of training epochs.")
flags.DEFINE_integer("max_steps", 100000, "Maximum number of training steps.")
# --- training stability ------------------------------------------------------------------------------------
flags.DEFINE_boolean("early_stopping", False, "Use early stopping to prevent overfitting.")
flags.DEFINE_float("grad_clip", 1.0, "Max gradient norm for training.")
flags.DEFINE_float("lr_gamma", 0.98, "Gamma for learning rate scheduler.")
flags.DEFINE_integer("lr_schedule_interval", 4000, "Number of steps between LR changes.")
flags.DEFINE_float("lr_warmup", 0, "Learning rate warmup (in units of lr_schedule_interval, flax's 'epochs').")
# --- model -------------------------------------------------------------------------------------------------
flags.DEFINE_string("architecture", "TransformerMDN", "Class name of model architecture.")
flags.DEFINE_integer("mdn_components", 100, "Number of mixtures.")
flags.DEFINE_integer("num_heads", 8, "Number of attention heads.")
flags.DEFINE_integer("num_layers", 6, "Number of encoder layers.")
flags.DEFINE_integer("num_mlp_layers", 2, "Number of output MLP layers.")
flags.DEFINE_integer("mlp_dims", 2048, "Number of channels per MLP layer.")
# --- data --------------------------------------------------------------------------------------------------
flags.DEFINE_list("data_shape", [32, 512], "Shape of data.")
flags.DEFINE_string("dataset", "./output/mel-32step-512", "Directory with train/eval tfrecord files.")
flags.DEFINE_string("pca_ckpt", "", "PCA transform.")
flags.DEFINE_string("slice_ckpt", "", "Slice transform.")
flags.DEFINE_string("dim_weights_ckpt", "", "Dimension scale transform.")
flags.DEFINE_boolean("normalize", True, "Normalize dataset to [-1, 1].")
# --- logging, checkpointing, evaluation --------------------------------------------------------------------
flags.DEFINE_integer("logging_freq", 100, "Logging frequency.")
flags.DEFINE_integer("snapshot_freq", 5000, "Evaluation and checkpoint frequency.")
flags.DEFINE_boolean("snapshot_sampling", True, "Sample during evaluation (as in the reference, train_mdn never samples; sample_mdn does).")
flags.DEFINE_integer("eval_samples", 3000, "Number of samples to generate.")
flags.DEFINE_integer("checkpoints_to_keep", 50, "Number of checkpoints to keep.")
flags.DEFINE_boolean("save_ckpt", True, "Save model checkpoints at each evaluation step.")
flags.DEFINE_string("model_dir", "./save/mdn", "Directory to store model data.")
flags.DEFINE_boolean("verbose", True, "Toggle logging to stdout.")
# --- additions of this implementation (not in the reference) ------------------------------------------------
flags.DEFINE_bool("synthetic", False, "Use synthetic N(0,1) latents of --data_shape instead of reading --dataset.")
flags.DEFINE_integer("synthetic_examples", 4096, "Examples per split with --synthetic.")


def mdn_loss(pi, mu, log_sigma, x, reduction="mean"):
    """train_mdn.py:100-133: negative log-likelihood of x under the mixture, one value per row of x.reshape(-1, C)
    (smd_mdn_nll), then reduced."""
    x = nn._as_device_f32(x)
    channels = x.shape[-1]
    pi, mu, log_sigma = (nn._as_device_f32(a) for a in (pi, mu, log_sigma))
    kc = pi.shape[-1]
    rows = x.numel() // channels
    if pi.numel() != rows * kc or mu.numel() != rows * kc * channels or log_sigma.numel() != mu.numel():
        raise ValueError("pi / mu / log_sigma do not match x's rows and channels")
    loss = torch.empty((rows,), dtype=torch.float32, device=x.device)
    lib = _lib.load_library()
    _lib.check(lib.smd_mdn_nll(pi.data_ptr(), mu.data_ptr(), log_sigma.data_ptr(), x.data_ptr(), rows, channels, kc,
                               loss.data_ptr(), torch.cuda.current_stream().cuda_stream))
    return reduce_fn(loss, reduction)


def create_optimizer(model, learning_rate):
    return optim.Adam(learning_rate=learning_rate).create(model)


def create_model(rng, input_shape, model_kwargs, batch_size=32, verbose=False):
    """train_mdn.py:143-152."""
    clazz = getattr(ar, FLAGS.architecture, None)
    if clazz is None:
        raise ValueError(f"Unknown architecture {FLAGS.architecture!r} (models/autoregressive.py has no such class)")
    module = clazz.partial(**model_kwargs)
    _, params = module.init_by_shape(rng, [((batch_size, *input_shape), np.float32)])
    model = nn.Model(module, params)
    if verbose:
        train_utils.report_model(model)
    return model


def eval_step(batch, model):
    """train_mdn.py:155-168: (summed token loss, number of tokens) of one batch; model(batch) + mdn_loss as one
    device call (smd_mdn_loss)."""
    x = nn._as_device_f32(batch)
    loss = model.engine(x.shape[0]).mdn_loss(x)
    return loss.sum(), loss.shape[0]


def evaluate(dataset, model):
    """train_mdn.py:171-195."""
    count, total = 0, 0.0
    for inputs in dataset:
        loss, examples = eval_step(inputs, model)
        count += examples
        total += float(loss)
    return {"loss": total / max(count, 1)}


def lr_at(step: int) -> float:
    """flax create_stepped_learning_rate_schedule(lr, lr_schedule_interval, [(i, gamma^i)], warmup_length=lr_warmup)
    at the 0-based global step (train_mdn.py:240-245): lr gamma^max(0, ceil(step / interval) - 1), times
    min(1, step / warmup / interval) while warming up."""
    interval = FLAGS.lr_schedule_interval
    n = 0 if step <= 0 else (step - 1) // interval
    lr = FLAGS.learning_rate * (FLAGS.lr_gamma ** n)
    if FLAGS.lr_warmup > 0:
        lr *= min(1.0, step / float(FLAGS.lr_warmup) / interval)
    return lr


def train_step(batch, optimizer, learning_rate):
    """train_mdn.py:198-224 on this rank's shard: grads -> all-reduce -> clip -> Adam."""
    model = optimizer.target
    world = parallel.world_size()
    x = nn._as_device_f32(batch)
    local = x.shape[0]
    eng = model.engine(local, training=True)
    if not hasattr(eng, "grads"):
        eng.init_train_state(ema=False)
    eng.compute_mdn_grads(x, global_batch=local * world)
    eng.reduce_grads(world)
    optimizer.apply_gradient(eng.grads, learning_rate=learning_rate, max_norm=FLAGS.grad_clip, engine=eng)
    return optimizer, {"loss": eng.loss_mean, "grad": optimizer.grad_norm, "lr": learning_rate}


def train(train_batches, valid_batches, output_dir=None, verbose=True):
    """train_mdn.py:227-312."""
    if torch.cuda.is_available() and torch.cuda.current_stream().cuda_stream == 0:
        # the legacy default stream cannot be captured: a private stream lets libsmd replay the step from a CUDA graph
        torch.cuda.set_stream(torch.cuda.Stream())
    first = next(iter(valid_batches))
    input_shape = tuple(first.shape[1:])
    rng = random.PRNGKey(FLAGS.seed)
    rng, model_rng = random.split(rng)
    lm_kwargs = dict(num_layers=FLAGS.num_layers, num_heads=FLAGS.num_heads, mdn_mixtures=FLAGS.mdn_components,
                     num_mlp_layers=FLAGS.num_mlp_layers, mlp_dims=FLAGS.mlp_dims)
    local_bs = parallel.shard_size(FLAGS.batch_size)
    model = create_model(model_rng, input_shape, lm_kwargs, local_bs, verbose=verbose)
    optimizer = create_optimizer(model, FLAGS.learning_rate)
    early_stop = train_utils.EarlyStopping(patience=1)
    writer = None
    if output_dir and parallel.rank() == 0:
        os.makedirs(output_dir, exist_ok=True)
        try:
            from torch.utils.tensorboard import SummaryWriter
            writer = SummaryWriter(os.path.join(output_dir, "train"))
        except Exception:  # tensorboard is optional
            writer = None
    if FLAGS.snapshot_sampling:
        logging.warning("--snapshot_sampling: train_mdn does not sample during evaluation (use sample_mdn); ignored")
    examples = train_batches.examples

    class _LocalRows:                            # rows [rank*B/W, (rank+1)*B/W) of every global batch
        def __iter__(self_inner):
            return (parallel.shard_rows(b) for b in train_batches)
    loader = input_pipeline.DevicePrefetcher(_LocalRows(), depth=2)
    sampling_step = -1
    for epoch in range(FLAGS.epochs):
        start_time = time.time()
        batches = iter(loader)
        try:
            done = _train_epoch(batches, epoch, optimizer, early_stop, sampling_step, writer, output_dir, verbose,
                                valid_batches, examples, start_time)
        finally:
            batches.close()          # stops the prefetch thread now, not at interpreter exit
        optimizer, early_stop, sampling_step, stop = done
        if stop:
            break
    if writer is not None:
        writer.flush()
    return optimizer


def _train_epoch(batches, epoch, optimizer, early_stop, sampling_step, writer, output_dir, verbose, valid_batches,
                 examples, start_time):
    """One pass of train_mdn.py:256-310; returns (optimizer, early_stop, sampling_step, stop training)."""
    for step, batch in enumerate(batches):
        global_step = step + epoch * examples
        optimizer, metrics = train_step(batch, optimizer, lr_at(global_step))
        if step % FLAGS.logging_freq == 0 and parallel.rank() == 0:
            elapsed = time.time() - start_time
            metrics.update({"batch/s": (step + 1) / elapsed, "ms/batch": elapsed * 1000 / (step + 1)})
            train_utils.log_metrics(metrics, step, examples, epoch=epoch, summary_writer=writer, verbose=verbose)
        if (step % FLAGS.snapshot_freq == 0 and step > 0) or step == examples - 1:
            sampling_step += 1
            ev = evaluate(valid_batches, optimizer.target)
            improved, early_stop = early_stop.update(ev["loss"])
            if parallel.rank() == 0:
                train_utils.log_metrics(ev, global_step, examples * FLAGS.epochs, summary_writer=None,
                                        verbose=verbose)
                if FLAGS.save_ckpt and output_dir and (not FLAGS.early_stopping or improved):
                    checkpoints.save_checkpoint(output_dir, (optimizer, early_stop), sampling_step,
                                                keep=FLAGS.checkpoints_to_keep)
            if FLAGS.early_stopping and early_stop.should_stop:
                logging.info("EARLY STOP: Ended training after %s epochs.", epoch + 1)
                return optimizer, early_stop, sampling_step, True
        if FLAGS.max_steps is not None and global_step >= FLAGS.max_steps:
            return optimizer, early_stop, sampling_step, True
    return optimizer, early_stop, sampling_step, False


def main(argv):
    del argv
    parallel.init_from_env()
    logging.info("platform: cuda (%s), ranks: %d", torch.cuda.get_device_name() if torch.cuda.is_available() else "none",
                 parallel.world_size())
    train_ds, eval_ds = input_pipeline.get_dataset(
        dataset=FLAGS.dataset, data_shape=FLAGS.data_shape, problem="vae", batch_size=FLAGS.batch_size,
        normalize=FLAGS.normalize, pca_ckpt=FLAGS.pca_ckpt, slice_ckpt=FLAGS.slice_ckpt,
        dim_weights_ckpt=FLAGS.dim_weights_ckpt, synthetic=FLAGS.synthetic,
        synthetic_examples=FLAGS.synthetic_examples, seed=FLAGS.seed)
    train(train_ds, eval_ds, FLAGS.model_dir, FLAGS.verbose)
    parallel.shutdown()


if __name__ == "__main__":
    app.run(main)
