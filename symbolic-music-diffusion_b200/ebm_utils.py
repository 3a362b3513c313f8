"""Noise schedule and the DDPM reverse sampler with the reference signatures (utils/ebm_utils.py)."""
from __future__ import annotations

import numpy as np
import torch


def _linspace_f32(start, stop, num):
    f32 = np.float32
    start, stop = f32(start), f32(stop)
    if num == 1:
        return np.asarray([start], f32)
    delta = f32(stop - start) / f32(num - 1)
    return (start + np.arange(num, dtype=f32) * delta).astype(f32)


def create_noise_schedule(sigma_begin=1, sigma_end=1e-2, L=10, schedule="geometric"):
    """utils/ebm_utils.py:62-86 (float32, like jnp)."""
    if schedule == "geometric":
        return np.exp(_linspace_f32(np.log(np.float32(sigma_begin)), np.log(np.float32(sigma_end)), L)).astype(np.float32)
    if schedule == "linear":
        return _linspace_f32(sigma_begin, sigma_end, L)
    if schedule == "fibonacci":
        s = [1e-6, 2e-6]
        for _ in range(L - 2):
            s.append(s[-1] + s[-2])
        return np.asarray(s, np.float32)
    raise ValueError(f"Unsupported schedule: {schedule}")


def diffusion_dynamics(rng, model, betas, init, epsilon, T, denoise, infill=False, infill_samples=None,
                       infill_masks=None, shard=None):
    """utils/ebm_utils.py:274-405.  Returns (state, collection (41, N, *shape), ld_metrics (4, len(betas), 1)).

    epsilon / T / denoise are null parameters upstream too.  The whole chain runs on the GPU (CUDA-graph replay of
    one reverse step); the noise of every step comes from `rng` with the reference's three splits per step."""
    del epsilon, T, denoise
    betas = np.asarray(betas, np.float32)

    def run(eng, x, ix, im, collection, metrics):
        eng.sampler_setup(betas, key=(int(rng[0]), int(rng[1])))
        eng.sample(x, steps=len(betas), infill_x=ix, infill_mask=im, collection=collection, metrics=metrics,
                   use_graph=True)
    x, collection, metrics = _device_chain(model, init, shard, (4, len(betas)), 41, infill, infill_samples,
                                           infill_masks, run)
    return x, collection, metrics.unsqueeze(2)


def _device_chain(model, init, shard, metrics_shape, collection_rows, infill, infill_samples, infill_masks, run):
    """What the sampler chains on the GPU share: x = a device copy of `init`, the engine for its batch with the shard
    (first_row, total_rows) set (`init` holds this rank's rows of a global batch; the per-step noise is the same slice
    of the global threefry stream), a collection of `collection_rows` rows (0: none) whose row 0 is the start, zeroed
    metrics; run(eng, x, infill_x, infill_mask, collection, metrics) sets up and runs the chain, then the batch-mean
    metrics are reduced over ranks.  Returns (x, collection, metrics)."""
    from .nn import _as_device_f32
    x = _as_device_f32(init).clone()
    n = x.shape[0]
    eng = model.engine(n)
    eng.set_sampler_shard(*(shard if shard is not None else (0, 0)))
    ix = _as_device_f32(infill_samples) if infill else None
    im = _as_device_f32(infill_masks) if infill else None
    collection = None
    if collection_rows:
        collection = torch.zeros((collection_rows,) + tuple(x.shape), dtype=torch.float32, device=x.device)
        # utils/ebm_utils.py:321-323,398: the merged start only goes to collection[0]; the scan itself starts from the
        # raw `init` (the first step's blend overwrites the masked entries anyway)
        collection[0] = x * (1 - im) + ix * im if infill else x
    metrics = torch.zeros(metrics_shape, dtype=torch.float32, device=x.device)
    run(eng, x, ix, im, collection, metrics)
    _reduce_sharded_metrics(metrics, n, shard)
    return x, collection, metrics


DDIM_SCHEDULES = ("uniform", "quadratic")


def ddim_schedule(T, K, schedule="uniform"):
    """The K indices tau_0 < ... < tau_{K-1} of a T-step schedule that the DDIM chain visits (int32):
    uniform tau_i = round(i (T-1) / (K-1)), quadratic tau_i = round((T-1) (i / (K-1))^2), both [T-1] for K = 1 (round
    half to even, in float64).  ValueError for K outside [1, T], an unknown schedule, or quadratic indices that are not
    strictly increasing (too many steps for T)."""
    T, K = int(T), int(K)
    if schedule not in DDIM_SCHEDULES:
        raise ValueError(f"unknown DDIM schedule {schedule!r} (expected one of {list(DDIM_SCHEDULES)})")
    if K < 1 or K > T:
        raise ValueError(f"the number of DDIM steps must be in [1, T = {T}], got {K}")
    if K == 1:
        return np.asarray([T - 1], np.int32)
    i = np.arange(K, dtype=np.float64)
    if schedule == "uniform":
        tau = np.rint(i * (T - 1) / (K - 1))
    else:
        tau = np.rint((T - 1) * (i / (K - 1)) ** 2)
    tau = tau.astype(np.int32)
    if np.any(np.diff(tau) <= 0):
        raise ValueError(f"the {schedule} schedule of {K} steps over T = {T} repeats indices")
    return tau


def ddim_dynamics(rng, model, betas, init, epsilon, T, denoise, infill=False, infill_samples=None, infill_masks=None,
                  shard=None, steps=50, eta=0.0, schedule="uniform"):
    """DDIM (Song et al. 2021) over `steps` levels of the DDPM schedule `betas` picked by `schedule` (ddim_schedule),
    with the clipped x0 estimate of diffusion_dynamics and noise scale eta (0: deterministic given `init`, 1 with all
    T levels: diffusion_dynamics itself).  Not in the reference.  Returns (state, collection (41, N, *shape),
    ld_metrics (4, steps, 1)); keys, collection rows, infill and shard as diffusion_dynamics with T replaced by the
    number of steps.  epsilon / T / denoise are null, as there."""
    del epsilon, T, denoise
    betas = np.asarray(betas, np.float32)
    tau = ddim_schedule(len(betas), steps, schedule)

    def run(eng, x, ix, im, collection, metrics):
        eng.ddim_setup(betas, tau, eta, key=(int(rng[0]), int(rng[1])))
        eng.ddim_sample(x, infill_x=ix, infill_mask=im, collection=collection, metrics=metrics, use_graph=True)
    x, collection, metrics = _device_chain(model, init, shard, (4, len(tau)), 41, infill, infill_samples,
                                           infill_masks, run)
    return x, collection, metrics.unsqueeze(2)


def ddim_encode(model, betas, x0, steps=50, schedule="uniform"):
    """The deterministic DDIM encoder (Song et al. 2021, sections 4.3 and 5.4): the eta = 0 DDIM chain run from the
    data x0 towards noise over the `steps` levels of `betas` that `schedule` picks (ddim_schedule), with the x0
    estimate unclipped.  Returns the codes x_T (float32, on the device); ddim_dynamics at eta = 0 over the same levels
    decodes them back to x0 up to discretisation error.  Not in the reference."""
    from .nn import _as_device_f32
    x = _as_device_f32(x0).clone()
    eng = model.engine(x.shape[0])
    betas = np.asarray(betas, np.float32)
    eng.ddim_encode_setup(betas, ddim_schedule(len(betas), steps, schedule))
    eng.ddim_encode(x, use_graph=True)
    return x


def slerp(z0, z1, alpha):
    """Spherical interpolation between the rows of z0 and z1 (each example flattened), in float64: sin((1-alpha)
    theta) / sin(theta) z0 + sin(alpha theta) / sin(theta) z1 with theta the angle between the two rows.  Exactly z0
    at alpha = 0 and z1 at alpha = 1; linear interpolation for rows whose angle is below 1e-6.  A linear mix of two
    near-Gaussian codes shrinks towards the origin (to about 0.7 of their norm at the midpoint), off the shell the
    decoder expects (Song et al. 2021, appendix D.5).  Returns a float64 tensor shaped like z0, on z0's device."""
    a = torch.as_tensor(z0).to(torch.float64)
    b = torch.as_tensor(z1).to(device=a.device, dtype=torch.float64)
    if a.shape != b.shape:
        raise ValueError(f"slerp needs equally shaped endpoints, got {tuple(a.shape)} and {tuple(b.shape)}")
    alpha = float(alpha)
    if alpha == 0.0:
        return a.clone()
    if alpha == 1.0:
        return b.clone()
    fa, fb = a.reshape(a.shape[0], -1), b.reshape(b.shape[0], -1)
    norms = fa.norm(dim=1) * fb.norm(dim=1)
    cos = torch.where(norms > 0, (fa * fb).sum(dim=1) / torch.where(norms > 0, norms, 1.0), 1.0)
    theta = torch.arccos(cos.clamp(-1.0, 1.0))
    linear = theta < 1e-6
    sin = torch.where(linear, 1.0, torch.sin(theta))
    w0 = torch.where(linear, 1.0 - alpha, torch.sin((1.0 - alpha) * theta) / sin)
    w1 = torch.where(linear, alpha, torch.sin(alpha * theta) / sin)
    return (w0[:, None] * fa + w1[:, None] * fb).reshape(a.shape)


def _reduce_sharded_metrics(metrics, n, shard):
    """The sampler metrics are means over the batch (utils/ebm_utils.py:166-170, 380-384): with shard = (first_row,
    total_rows) over several ranks, one weighted all-reduce at the end; row 2 (alpha / alpha_prod) is no batch mean."""
    if shard is None:
        return
    from . import parallel
    if parallel.world_size() > 1:
        w = float(n) / float(shard[1])
        alpha_row = metrics[2].clone()
        metrics.mul_(w)
        parallel.all_reduce_sum_(metrics)
        metrics[2] = alpha_row


def collate_sampling_metrics(ld_metrics):
    """utils/ebm_utils.py:408-428."""
    ld = ld_metrics.detach().cpu().numpy() if isinstance(ld_metrics, torch.Tensor) else np.asarray(ld_metrics)
    _, num_sigmas, num_steps = ld.shape
    out = [[] for _ in range(num_sigmas)]
    for i in range(num_sigmas):
        grad_norm, step_norm, alpha, noise_norm = ld[:, i, :]
        for j in range(num_steps):
            out[i].append({"slope": grad_norm[j], "step": step_norm[j], "alpha": alpha[j], "noise": noise_norm[j]})
    return out


def _collection_slot_fn(total_steps, collection_steps):
    idx = np.linspace(1, total_steps, collection_steps).astype(np.int32)      # utils/ebm_utils.py:127-129

    def slot(image_idx):
        mask = idx == image_idx
        return int(np.sum(np.arange(len(idx)) * mask) + 1) if mask.any() else -1
    return slot


def annealed_langevin_dynamics(rng, model, sigmas, init, epsilon, T, denoise, infill=False, infill_samples=None,
                               infill_masks=None, shard=None):
    """utils/ebm_utils.py:89-198 (Song & Ermon): for every noise level T steps x += alpha * score + sqrt(2 alpha) z with
    alpha = epsilon (sigma / sigma_L)^2.  Returns (state, collection (101 + denoise, N, ...), metrics (4, L, T)).

    The whole chain runs on the GPU (smd_langevin_sample: CUDA-graph replay of one step, keys from the scan carry
    `rng, step_rng, infill_rng = split(rng, 3)` derived on the device).  shard = (first_row, total_rows) as in
    diffusion_dynamics: `init` holds this rank's rows of a global batch."""
    sig = np.asarray(sigmas, np.float32)
    assert len(sig) >= 2

    def run(eng, x, ix, im, collection, metrics):
        eng.langevin_setup(sig, int(T), epsilon, "ald", key=(int(rng[0]), int(rng[1])))
        eng.langevin_sample(x, denoise=bool(denoise), infill_x=ix, infill_mask=im, collection=collection,
                            metrics=metrics)
    return _device_chain(model, init, shard, (4, len(sig), int(T)), 101 + int(bool(denoise)), infill, infill_samples,
                         infill_masks, run)


def consistent_langevin_dynamics(rng, model, sigmas, init, epsilon, T, denoise=True, infill=False, infill_samples=None,
                                 infill_masks=None, shard=None):
    """utils/ebm_utils.py:201-271 (Jolicoeur-Martineau et al.): one step per noise level,
    x += alpha * score + beta * sigma_{i+1} * z.  Returns (state, None, metrics (4, L, 1)) -- upstream returns two values
    although its caller unpacks three (SURVEY section 0); the missing collection is returned as None.  Runs on the GPU
    like annealed_langevin_dynamics (keys `rng, step_rng = split(rng)`); shard as there."""
    del T
    if infill:
        raise NotImplementedError
    sig = np.asarray(sigmas, np.float32)
    assert len(sig) >= 2

    def run(eng, x, ix, im, collection, metrics):
        eng.langevin_setup(sig, 1, epsilon, "cas", key=(int(rng[0]), int(rng[1])))
        eng.langevin_sample(x, denoise=bool(denoise), metrics=metrics)
    return _device_chain(model, init, shard, (4, len(sig), 1), 0, False, None, None, run)
