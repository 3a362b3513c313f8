"""Sampling entry point with the reference's flag surface (sample_ncsn.py:51-66 on top of train_ncsn.py:48-128):

  python -m smd_b200.sample_ncsn --flagfile=configs/ddpm-mel-32seq-512.cfg --sample_size=1000 [--synthetic]

Restores the newest checkpoint of --model_dir into a freshly created model (sample_ncsn.py:331-342; like upstream
it samples from optimizer.target, never from the EMA parameters), runs the full reverse chain on the GPU and
writes ncsn/{real,generated,collection}.pkl under --sampling_dir (sample_ncsn.py:453-471).  --interpolate with
--interpolate_encoder=ddim encodes with the deterministic DDIM encoder instead and also writes
ncsn/reconstruction.json.  With torchrun the sample_size is sharded across ranks (replicated parameters, no per-step
exchange) and gathered at the end.
--compute_metrics then scores the samples against the real examples on the GPU (ncsn/metrics.json); with
--full_metrics also by the coverage metrics (PRD, improved precision / recall, realism, NDB).
"""
from __future__ import annotations

import json
import os
import pickle
import time
import warnings

import numpy as np
import torch
from absl import app, flags, logging

from smd_b200 import checkpoints, ebm_utils, input_pipeline, jrandom as random, metrics, parallel, train_utils
from smd_b200 import train_ncsn  # noqa: F401  (defines the shared training flags)

FLAGS = flags.FLAGS
flags.DEFINE_integer("sample_seed", 1, "PRNG seed of the sampler.")
flags.DEFINE_string("sampling_dir", "samples", "Output directory (relative to --model_dir).")
flags.DEFINE_integer("sample_size", 1000, "Number of samples to draw.")
flags.DEFINE_bool("compute_metrics", False, "Frechet distance and RBF / polynomial MMD against the real examples of 20 "
                  "points of the sampling collection and of a random and a real baseline, written to "
                  "ncsn/metrics.json.")
flags.DEFINE_bool("compute_final_only", False, "Metrics on the final samples only.")
flags.DEFINE_bool("full_metrics", False, "With --compute_metrics, also PRD precision / recall / F1, improved precision / "
                  "recall / F1, realism and NDB (sample_ncsn.py:132-159 of the reference, which never defines them; "
                  "see metrics.py), k-means seeded from --sample_seed.  Not a reference flag.")
flags.DEFINE_bool("flush", True, "Write pickles.")
flags.DEFINE_bool("animate", False, "Write sampling animations (not supported: raises ValueError).")
flags.DEFINE_bool("infill", False, "Infill the middle 16 latents of real examples (sample_ncsn.py:408-427).")
flags.DEFINE_bool("interpolate", False, "Interpolate between real examples in the diffusion latent space.")
flags.DEFINE_enum("interpolate_encoder", "stochastic", ["stochastic", "ddim"],
                  "--interpolate: stochastic is the reference's q(x_T | x_0) encoder with linear interpolation and the "
                  "ddpm decoder; ddim (needs --sampling=ddim and --ddim_eta=0) encodes with the deterministic DDIM "
                  "encoder over --ddim_steps / --ddim_schedule, interpolates spherically and decodes with the eta = 0 "
                  "DDIM chain, and writes ncsn/reconstruction.json.  ddim is not a reference option.")


def _restore(model_dir, shape, batch_size=1):
    """sample_ncsn.py:331-342: dummy-initialised (optimizer, ema, early_stop) filled from the newest checkpoint."""
    rng = random.PRNGKey(FLAGS.sample_seed)
    rng, model_rng = random.split(rng)
    model = train_ncsn.create_model(model_rng, shape, train_ncsn.model_kwargs(), batch_size=batch_size)
    optimizer = train_ncsn.create_optimizer(model, FLAGS.learning_rate)
    ema = train_utils.EMAHelper(mu=0, params=model.arena.clone())
    early_stop = train_utils.EarlyStopping()
    optimizer, ema, early_stop = checkpoints.restore_checkpoint(model_dir, (optimizer, ema, early_stop))
    return rng, optimizer


def generate_samples(sample_shape, num_samples, rng_seed=1):
    """sample_ncsn.py:313-365."""
    del rng_seed
    rng, optimizer = _restore(FLAGS.model_dir, sample_shape)
    sigmas = ebm_utils.create_noise_schedule(FLAGS.sigma_begin, FLAGS.sigma_end, FLAGS.num_sigmas, FLAGS.schedule_type)
    world, rank = parallel.world_size(), parallel.rank()
    rng, sample_rng = random.split(rng)          # sample_ncsn.py:350
    t0 = time.time()
    # every rank holds the same key; rank r generates rows [r*N/W, (r+1)*N/W) of the N-sample run (its slice of the
    # initial draw and of each step's noise), so the gathered result is the single-process result
    generated, collection, ld_metrics = train_ncsn.sample(optimizer.target, sigmas, sample_rng, sample_shape,
                                                          num_samples=num_samples, sampling=FLAGS.sampling,
                                                          epsilon=FLAGS.ld_epsilon, steps=FLAGS.ld_steps,
                                                          denoise=FLAGS.denoise, shard=(rank, world))
    torch.cuda.synchronize()
    logging.info("Generated samples in %f seconds", time.time() - t0)
    generated = parallel.gather_rows(generated)
    if collection is not None:      # consistent Langevin dynamics keeps no collection
        collection = parallel.gather_rows(collection.transpose(0, 1).contiguous()).transpose(0, 1).cpu().numpy()
    return generated.cpu().numpy(), collection, ld_metrics


def infill_samples(samples, masks, rng_seed=1):
    """sample_ncsn.py:189-242: keep the masked (=1) entries of `samples`, regenerate the rest with the --sampling
    chain (ald, ddpm, ddim or dpm; cas has no infilling, as upstream)."""
    del rng_seed
    if FLAGS.sampling == "ald":
        algorithm = ebm_utils.annealed_langevin_dynamics
    elif FLAGS.sampling == "cas":
        algorithm = ebm_utils.consistent_langevin_dynamics
    elif FLAGS.sampling == "ddpm":
        algorithm = ebm_utils.diffusion_dynamics
    elif FLAGS.sampling == "ddim":
        algorithm = train_ncsn.ddim_algorithm()
    elif FLAGS.sampling == "dpm":
        algorithm = train_ncsn.dpm_algorithm()
    else:
        raise ValueError(f"Unknown sampling algorithm: {FLAGS.sampling}")
    rng, optimizer = _restore(FLAGS.model_dir, samples.shape[1:])
    sigmas = ebm_utils.create_noise_schedule(FLAGS.sigma_begin, FLAGS.sigma_end, FLAGS.num_sigmas, FLAGS.schedule_type)
    init_rng, ld_rng = random.split(rng)
    init = random.uniform(init_rng, samples.shape)      # upstream initialises the infill chain with uniform noise
    generated, collection, ld_metrics = algorithm(ld_rng, optimizer.target, sigmas, init, FLAGS.ld_epsilon,
                                                  FLAGS.ld_steps, FLAGS.denoise, True, samples, masks)
    return generated.cpu().numpy(), collection.cpu().numpy(), ebm_utils.collate_sampling_metrics(ld_metrics)


def diffusion_stochastic_encoder(samples, rng_seed=1):
    """sample_ncsn.py:245-265: z ~ q(x_T | x_0).  Upstream indexes ``alphas_prod[T]`` (one past the end), which jax
    clamps to the last element; the first output of ``split(rng)`` is the noise key."""
    assert FLAGS.sampling == "ddpm"
    rng = random.PRNGKey(rng_seed)
    betas = ebm_utils.create_noise_schedule(FLAGS.sigma_begin, FLAGS.sigma_end, FLAGS.num_sigmas, FLAGS.schedule_type)
    alphas_prod = np.cumprod((np.float32(1.0) - betas).astype(np.float32), dtype=np.float32)
    rng, _ = random.split(rng)
    x = torch.as_tensor(np.ascontiguousarray(samples, np.float32), device="cuda")
    noise = random.normal(rng, x.shape)
    last = alphas_prod[-1]                        # alphas_prod[T] clamped
    return float(np.sqrt(last)) * x + float(np.sqrt(np.float32(1.0) - last)) * noise


def diffusion_decoder(z_list, rng_seed=1):
    """sample_ncsn.py:268-310: one reverse chain per latent, all with the same sampling key."""
    assert FLAGS.sampling == "ddpm"
    rng = random.PRNGKey(rng_seed)
    rng, ld_rng, model_rng = random.split(rng, 3)
    del model_rng
    betas = ebm_utils.create_noise_schedule(FLAGS.sigma_begin, FLAGS.sigma_end, FLAGS.num_sigmas, FLAGS.schedule_type)
    _, optimizer = _restore(FLAGS.model_dir, tuple(z_list[0].shape[1:]))
    gen, collects, metrics = [], [], []
    for i, z in enumerate(z_list):
        generated, collection, ld_metrics = ebm_utils.diffusion_dynamics(ld_rng, optimizer.target, betas, z,
                                                                         FLAGS.ld_epsilon, FLAGS.ld_steps, FLAGS.denoise,
                                                                         False)
        gen.append(generated.cpu().numpy())
        collects.append(collection.cpu().numpy())
        metrics.append(ebm_utils.collate_sampling_metrics(ld_metrics))
        logging.info("Generated samples %i out of %i", i, len(z_list))
    return gen, collects, metrics


def ddim_interpolate(starts, rng_seed=1):
    """--interpolate_encoder=ddim (not in the reference): the deterministic DDIM encoder (Song et al. 2021, sections 4.3
    and 5.4) maps each start to its code; the goals' codes are the starts' codes rolled by one row, as the goals are
    the rolled starts and the encoder is deterministic.  Each of the 9 spherical interpolants (ebm_utils.slerp) is
    decoded by the eta = 0 DDIM chain over the same levels.  Under torchrun every rank encodes and decodes its own
    rows; the rows are gathered.  Returns generated (9, N, ...) and collection (9, 41, N, ...), normalised."""
    rng = random.PRNGKey(rng_seed)        # the decoder draws nothing at eta = 0: the key only fills the key table
    betas = ebm_utils.create_noise_schedule(FLAGS.sigma_begin, FLAGS.sigma_end, FLAGS.num_sigmas, FLAGS.schedule_type)
    _, optimizer = _restore(FLAGS.model_dir, starts.shape[1:])
    world, rank = parallel.world_size(), parallel.rank()
    local = parallel.shard_size(len(starts))
    rows = slice(rank * local, (rank + 1) * local)
    t0 = time.time()
    codes = ebm_utils.ddim_encode(optimizer.target, betas, starts[rows], steps=FLAGS.ddim_steps,
                                  schedule=FLAGS.ddim_schedule)
    codes = parallel.gather_rows(codes)
    goal_codes = torch.roll(codes, shifts=1, dims=0)
    kw = dict(shard=(rank * local, len(starts))) if world > 1 else {}
    gen, colls = [], []
    for i, alpha in enumerate(np.linspace(0.0, 1.0, 9)):
        z = ebm_utils.slerp(codes, goal_codes, float(alpha)).to(torch.float32)[rows].contiguous()
        x, collection, _ = ebm_utils.ddim_dynamics(rng, optimizer.target, betas, z, None, None, None, False,
                                                   steps=FLAGS.ddim_steps, eta=0.0, schedule=FLAGS.ddim_schedule, **kw)
        gen.append(parallel.gather_rows(x).cpu().numpy())
        colls.append(parallel.gather_rows(collection.transpose(0, 1).contiguous()).transpose(0, 1).cpu().numpy())
        logging.info("Generated samples %i out of %i", i, 9)
    torch.cuda.synchronize()
    logging.info("Encoded and decoded the interpolants in %f seconds", time.time() - t0)
    return np.stack(gen), np.stack(colls)


def reconstruction_errors(generated, starts, goals):
    """How far the alpha = 0 and alpha = 1 interpolants lie from the examples they encode, in normalised units: the mean
    squared and the largest absolute error of decode(encode(x)) against x."""
    out = {}
    for name, got, want in (("start", generated[0], starts), ("goal", generated[-1], goals)):
        d = np.asarray(got, np.float64) - np.asarray(want, np.float64)
        out[f"{name}_mse"] = float(np.mean(d * d))
        out[f"{name}_max_abs"] = float(np.max(np.abs(d)))
    return out


def _save(obj, path):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "wb") as f:
        pickle.dump(obj, f, protocol=4)
    logging.info("Saved to %s", path)


def evaluation_points(collection, final_only=False):
    """sample_ncsn.py:96-101: 20 points spread over the sampling collection, or its last point only."""
    points = collection[np.linspace(0, len(collection) - 1, 20).astype(np.uint32)]
    return [points[-1]] if final_only else list(points)


def evaluate(real, collection, seed, final_only=False, metric_fn=metrics.latent_metrics):
    """sample_ncsn.py:69-186 with the metrics utils/metrics.py defines (Frechet distance, RBF and polynomial MMD;
    upstream's precision/recall, realism and NDB calls name functions it never defines; metric_fn=full_metrics adds
    the published metrics of those names).  real (N, ...) and
    collection (steps, N, ...) are the normalised data.  Returns {model: {evaluation index: {metric: value}}} for
    model "ncsn" (the collection points), "random" (standard normals shaped like one point; seeded here, unseeded
    upstream) and "real" (real against itself)."""
    if collection.shape[1:] != real.shape:
        raise ValueError(f"collection points {collection.shape[1:]} do not match the real examples {real.shape}")
    logging.info("Generated sample range: [%f, %f]", collection[-1].min(), collection[-1].max())
    logging.info("Test sample range: [%f, %f]", real.min(), real.max())
    if collection[-1].min() < -1 or collection[-1].max() > 1 or real.min() < -1 or real.max() > 1:
        warnings.warn("Normalize test samples and generated samples to [-1, 1] range.")
    random_points = [np.random.default_rng(seed).standard_normal(collection[0].shape).astype(np.float32)]
    results = {}
    for model, points in [("ncsn", evaluation_points(collection, final_only)), ("random", random_points),
                          ("real", [real])]:
        results[model] = {str(i): metric_fn(real, p) for i, p in enumerate(points)}
    return results


def save_metrics(results, out_dir):
    path = os.path.join(out_dir, "metrics.json")
    os.makedirs(out_dir, exist_ok=True)
    with open(path, "w") as f:
        json.dump(results, f, indent=1, sort_keys=True)
    logging.info("Saved to %s", path)
    return path


def check_flags():
    if FLAGS.animate:
        raise ValueError("--animate writes matplotlib animations, which are out of scope")
    if FLAGS.compute_metrics and FLAGS.interpolate:
        # upstream's evaluate asserts collection.shape[1:] == real.shape, which the (9, steps, N, ...) collection of
        # the interpolation never meets
        raise ValueError("--compute_metrics does not apply to --interpolate")
    if FLAGS.full_metrics and not FLAGS.compute_metrics:
        raise ValueError("--full_metrics needs --compute_metrics")
    if FLAGS.interpolate and FLAGS.sampling == "dpm":
        raise ValueError("--interpolate does not take --sampling=dpm: its encoders and decoders are the ddpm and ddim "
                         "chains")
    if FLAGS.interpolate_encoder == "ddim":
        if not FLAGS.interpolate:
            raise ValueError("--interpolate_encoder=ddim needs --interpolate")
        if FLAGS.sampling != "ddim":
            raise ValueError("--interpolate_encoder=ddim needs --sampling=ddim")
        if FLAGS.ddim_eta != 0.0:
            raise ValueError("--interpolate_encoder=ddim needs --ddim_eta=0: the encoder inverts the deterministic "
                             "chain only")


def full_metrics(real, fake):
    """The eleven values sample_ncsn.py:132-170 logs: the three distance metrics and the eight coverage metrics."""
    return {**metrics.latent_metrics(real, fake), **metrics.coverage_metrics(real, fake, seed=FLAGS.sample_seed)}


def main(argv):
    del argv
    check_flags()
    parallel.init_from_env()
    _, eval_ds = input_pipeline.get_dataset(
        dataset=FLAGS.dataset, data_shape=FLAGS.data_shape, problem=FLAGS.problem, batch_size=FLAGS.batch_size,
        normalize=FLAGS.normalize, pca_ckpt=FLAGS.pca_ckpt, slice_ckpt=FLAGS.slice_ckpt,
        dim_weights_ckpt=FLAGS.dim_weights_ckpt, include_cardinality=False, synthetic=FLAGS.synthetic,
        synthetic_examples=max(FLAGS.synthetic_examples, 8 * FLAGS.sample_size), seed=FLAGS.seed)
    real = []
    for batch in eval_ds:                                  # sample_ncsn.py:397-402
        real.append(batch)
        if sum(len(b) for b in real) >= FLAGS.sample_size:
            break
    real = np.concatenate(real)[:FLAGS.sample_size]
    shape = real.shape[1:]
    if FLAGS.infill:                                       # sample_ncsn.py:408-427 (sequence branch)
        if real.ndim != 3 or real.shape[1] != 32:
            raise ValueError("--infill needs (N, 32, C) latent sequences")
        samples = np.copy(real)
        samples[:, 8:-8, :] = 0                            # the middle 16 latents are regenerated
        masks = np.zeros(samples.shape, np.float32)
        masks[:, :8, :] = 1
        masks[:, -8:, :] = 1                               # first and last 8 are held fixed
        generated, collection, _ = infill_samples(samples, masks, FLAGS.sample_seed)
    elif FLAGS.interpolate and FLAGS.interpolate_encoder == "ddim":
        starts = real
        goals = np.roll(starts, shift=1, axis=0)
        generated, collection = ddim_interpolate(starts, FLAGS.sample_seed)
        recon = reconstruction_errors(generated, starts, goals)
        logging.info("Reconstruction (normalised units): %s", json.dumps(recon, sort_keys=True))
        if parallel.rank() == 0:
            out = os.path.join(FLAGS.model_dir, FLAGS.sampling_dir, "ncsn")
            os.makedirs(out, exist_ok=True)
            with open(os.path.join(out, "reconstruction.json"), "w") as f:
                json.dump(dict(recon, ddim_steps=FLAGS.ddim_steps, ddim_schedule=FLAGS.ddim_schedule), f, indent=1,
                          sort_keys=True)
    elif FLAGS.interpolate:                                # sample_ncsn.py:429-438
        starts = real
        goals = np.roll(starts, shift=1, axis=0)
        starts_z = diffusion_stochastic_encoder(starts, FLAGS.sample_seed)
        goals_z = diffusion_stochastic_encoder(goals, FLAGS.sample_seed)
        interp_zs = [float(1 - alpha) * starts_z + float(alpha) * goals_z for alpha in np.linspace(0.0, 1.0, 9)]
        gen, coll, _ = diffusion_decoder(interp_zs, FLAGS.sample_seed)
        generated, collection = np.stack(gen), np.stack(coll)
    else:
        generated, collection, _ = generate_samples(shape, len(real), FLAGS.sample_seed)
    if FLAGS.flush and parallel.rank() == 0:
        slice_idx = input_pipeline.load(os.path.expanduser(FLAGS.slice_ckpt)) if FLAGS.slice_ckpt else None
        dim_w = input_pipeline.load(os.path.expanduser(FLAGS.dim_weights_ckpt)) if FLAGS.dim_weights_ckpt else None
        inv = lambda a: input_pipeline.inverse_data_transform(  # noqa: E731
            a, normalize=FLAGS.normalize, data_min=eval_ds.min, data_max=eval_ds.max, slice_idx=slice_idx,
            dim_weights=dim_w, out_channels=int(FLAGS.data_shape[-1]))
        out = os.path.join(FLAGS.model_dir, FLAGS.sampling_dir, "ncsn")
        if collection is not None:
            _save(inv(collection), os.path.join(out, "collection.pkl"))
        _save(inv(real), os.path.join(out, "real.pkl"))
        _save(inv(generated), os.path.join(out, "generated.pkl"))
    if FLAGS.compute_metrics and parallel.rank() == 0:     # sample_ncsn.py:474-477, on the normalised data
        metric_fn = full_metrics if FLAGS.full_metrics else metrics.latent_metrics
        if collection is None:                             # consistent Langevin dynamics: the final samples only
            results = evaluate(real, generated[None], FLAGS.sample_seed, True, metric_fn)
        else:
            results = evaluate(real, collection, FLAGS.sample_seed, FLAGS.compute_final_only, metric_fn)
        ncsn = results["ncsn"]
        train_utils.log_metrics(ncsn[str(len(ncsn) - 1)], 1, 1)
        save_metrics(results, os.path.join(FLAGS.model_dir, FLAGS.sampling_dir, "ncsn"))
    parallel.shutdown()


if __name__ == "__main__":
    app.run(main)
