"""Sampling entry point of the autoregressive baseline with the reference's flag surface (sample_mdn.py:47-51 on top of
train_mdn.py's flags), so configs/mdn-*.cfg run unchanged:

  python -m smd_b200.sample_mdn --flagfile=configs/mdn-mel-32seq-512.cfg --sample_size=1000 [--synthetic]

Restores the newest (optimizer, early_stop) checkpoint of --model_dir into a freshly created model, decodes
--sample_size sequences on the GPU (smd_mdn_sample: each step runs the network at one position per sample and reads
the keys and values of earlier positions from a cache) and writes mdn/real.pkl and mdn/generated.pkl under
--sampling_dir (sample_mdn.py:122-176).  With torchrun the samples are sharded across ranks (replicated parameters, no
per-step exchange) and gathered on rank 0.  Every rank draws its rows of the one global draw, so the result does not
depend on the number of ranks.
"""
from __future__ import annotations

import os
import time

import numpy as np
import torch
from absl import app, flags, logging

from smd_b200 import checkpoints, input_pipeline, jrandom as random, parallel, train_utils
from smd_b200 import train_mdn  # (defines the shared training flags)
from smd_b200.engine import Engine

FLAGS = flags.FLAGS
flags.DEFINE_integer("sample_seed", 1, "Random number generator seed for sampling.")
flags.DEFINE_string("sampling_dir", "sample", "Sampling directory.")
flags.DEFINE_integer("sample_size", 1000, "Number of samples.")
flags.DEFINE_boolean("flush", True, "Flush generated samples to disk.")


def sample(num_samples=2400, steps=32, embedding_dims=42, rng_seed=1, real=None):
    """sample_mdn.py:54-119: autoregressive decoding of (num_samples, steps, embedding_dims) from the checkpoint in
    --model_dir.  Under torchrun each rank decodes its shard of the num_samples rows; every rank returns the gathered
    (num_samples, steps, embedding_dims) tensor."""
    del real
    rng = random.PRNGKey(rng_seed)
    rng, model_rng = random.split(rng)
    lm_kwargs = dict(num_layers=FLAGS.num_layers, num_heads=FLAGS.num_heads, mdn_mixtures=FLAGS.mdn_components,
                     num_mlp_layers=FLAGS.num_mlp_layers, mlp_dims=FLAGS.mlp_dims)
    model = train_mdn.create_model(model_rng, (steps, embedding_dims), lm_kwargs, batch_size=1, verbose=True)
    optimizer = train_mdn.create_optimizer(model, 0)
    early_stop = train_utils.EarlyStopping()
    optimizer, early_stop = checkpoints.restore_checkpoint(FLAGS.model_dir, (optimizer, early_stop))
    arena = optimizer.target.arena
    local = parallel.shard_size(num_samples)
    first = parallel.rank() * local
    eng = Engine(arena.spec.model_config(arena.input_shape), max_batch=local, sampler_T=steps)
    eng.set_params(arena.flat)
    t0 = time.time()
    generated = eng.mdn_sample(rng, local, first_row=first, total_rows=num_samples)
    torch.cuda.synchronize()
    logging.info("Generated samples in %f seconds", time.time() - t0)
    return parallel.gather_rows(generated)


def main(argv):
    del argv
    parallel.init_from_env()
    logging.info(FLAGS.flags_into_string())
    train_ds, eval_ds = input_pipeline.get_dataset(
        dataset=FLAGS.dataset, data_shape=FLAGS.data_shape, problem="vae", batch_size=FLAGS.batch_size,
        normalize=FLAGS.normalize, pca_ckpt=FLAGS.pca_ckpt, slice_ckpt=FLAGS.slice_ckpt,
        dim_weights_ckpt=FLAGS.dim_weights_ckpt, include_cardinality=False, synthetic=FLAGS.synthetic,
        synthetic_examples=max(FLAGS.synthetic_examples, FLAGS.sample_size), seed=FLAGS.seed)
    real = []
    for batch in eval_ds:                                  # eval_ds.unbatch().take(sample_size)
        real.append(np.asarray(batch))
        if sum(len(b) for b in real) >= FLAGS.sample_size:
            break
    real = np.concatenate(real)[:FLAGS.sample_size]
    shape = real[0].shape
    generated = sample(FLAGS.sample_size, shape[-2], shape[-1], FLAGS.sample_seed, real)
    generated = generated.cpu().numpy()
    if FLAGS.flush and parallel.rank() == 0:
        pca = input_pipeline.load(os.path.expanduser(FLAGS.pca_ckpt)) if FLAGS.pca_ckpt else None
        slice_idx = input_pipeline.load(os.path.expanduser(FLAGS.slice_ckpt)) if FLAGS.slice_ckpt else None
        dim_w = input_pipeline.load(os.path.expanduser(FLAGS.dim_weights_ckpt)) if FLAGS.dim_weights_ckpt else None
        inv = lambda a, lo, hi: input_pipeline.inverse_data_transform(  # noqa: E731
            a, normalize=FLAGS.normalize, pca=pca, data_min=lo, data_max=hi, slice_idx=slice_idx, dim_weights=dim_w,
            out_channels=int(FLAGS.data_shape[-1]))
        # generated samples are scaled back with the training set's range, the real ones with the eval set's
        input_pipeline.save(inv(real, eval_ds.min, eval_ds.max), os.path.join(FLAGS.sampling_dir, "mdn/real.pkl"))
        input_pipeline.save(inv(generated, train_ds.min, train_ds.max),
                            os.path.join(FLAGS.sampling_dir, "mdn/generated.pkl"))
    parallel.shutdown()


if __name__ == "__main__":
    app.run(main)
