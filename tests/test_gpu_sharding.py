"""Data-parallel RNG slicing (SURVEY 8(e)): a rank consumes rows [r*B/W, (r+1)*B/W) of the single-process threefry
streams, so DP(seed) == single-GPU(seed) for the training draws, the sampler's initial state and every reverse step.
The ranks are simulated one after the other on one GPU (the slices are a property of the kernels, not of NCCL)."""
import numpy as np
import pytest
import torch

from oracle import ddpm_oracle as O
from oracle import threefry as tf

pytestmark = pytest.mark.gpu

TINY = dict(num_layers=1, num_heads=8, num_mlp_layers=1, channels=42)


def _engine(batch, training=False):
    from smd_b200 import Engine, ModelConfig
    eng = Engine(ModelConfig(**TINY), max_batch=batch, cta_group=2, training=training)
    eng.set_params(eng.init_params(seed=1, perturb=0.02))
    return eng


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_training_draws_are_slices_of_the_global_stream(lib, world):
    G = 8 * world
    eng = _engine(G)
    betas = O.create_noise_schedule(1e-6, 0.01, 1000, "linear")
    eng.objective_setup(betas)
    key = tf.prng_key(5)
    k = (int(key[0]), int(key[1]))
    used_g, eps_g, lab_g = eng.draws(k, G, want_labels=True)
    rl, ru, _ = O.diffusion_loss_draws(key, (G, 32, 42), betas, continuous_noise=True)
    np.testing.assert_array_equal(lab_g.cpu().numpy(), rl)
    np.testing.assert_array_equal(used_g.cpu().numpy(), ru)
    for r in range(world):
        used, eps, lab = eng.draws(k, 8, want_labels=True, global_batch=G, first_row=8 * r)
        sl = slice(8 * r, 8 * r + 8)
        assert torch.equal(used, used_g[sl]) and torch.equal(eps, eps_g[sl]) and torch.equal(lab, lab_g[sl])


def test_discrete_noise_label_range_matches_the_reference_branch(lib):
    """--continuous_noise=False (utils/losses.py:272-275): labels in [0, T); label 0 reads alphas_prod[-1]."""
    eng = _engine(256)
    betas = O.create_noise_schedule(1e-6, 0.01, 50, "linear")     # short schedule: label 0 shows up in 256 draws
    eng.objective_setup(betas)
    key = tf.prng_key(9)
    used, eps, lab = eng.draws((int(key[0]), int(key[1])), 256, want_labels=True, continuous_noise=False)
    rl, ru, re = O.diffusion_loss_draws(key, (256, 32, 42), betas, continuous_noise=False)
    assert rl.min() == 0 and rl.max() <= 49
    np.testing.assert_array_equal(lab.cpu().numpy(), rl)
    np.testing.assert_array_equal(used.cpu().numpy(), ru)
    np.testing.assert_allclose(eps.cpu().numpy(), re, rtol=2e-5, atol=2e-6)


def test_sharded_sampling_equals_the_single_process_chain(lib):
    """4 + 4 samples on two simulated ranks == 8 samples on one: same initial slice, same per-step noise slices;
    the weighted mean of the per-rank metrics is the single-process metric (utils/ebm_utils.py:380-384)."""
    from smd_b200 import jrandom
    betas = O.create_noise_schedule(1e-6, 0.01, 1000, "linear")
    key = (0, 21)
    steps = 5
    one = _engine(8)
    one.sampler_setup(betas, key=key)
    init_key = jrandom.PRNGKey(3)
    x_all = jrandom.normal(init_key, (8, 32, 42))
    m_all = torch.zeros((4, 1000), device="cuda")
    ref = x_all.clone()
    one.sample(ref, steps=steps, metrics=m_all, use_graph=True)
    m_sum = torch.zeros((4, 1000), device="cuda")
    for r in range(2):
        eng = _engine(4)
        eng.sampler_setup(betas, key=key)
        eng.set_sampler_shard(4 * r, 8)
        x = jrandom.normal(init_key, (8, 32, 42), rows=(4 * r, 4))
        assert torch.equal(x, x_all[4 * r:4 * r + 4])
        m = torch.zeros((4, 1000), device="cuda")
        eng.sample(x, steps=steps, metrics=m, use_graph=(r == 0))      # graph replay and plain launches alike
        # identical inputs and noise: the LayerNorm statistics partials (stats_part slots) are added in a fixed order, so
        # the forward pass is bit-reproducible and independent of where a row sits in the batch: the shards match exactly
        assert torch.equal(x, ref[4 * r:4 * r + 4]), float((x - ref[4 * r:4 * r + 4]).abs().max())
        m_sum += m * 0.5
    torch.testing.assert_close(m_sum[[0, 1, 3], :steps], m_all[[0, 1, 3], :steps], rtol=1e-5, atol=1e-7)


def test_device_prefetcher_yields_every_batch_in_order(lib):
    from smd_b200 import input_pipeline as ip
    batches = [np.full((4, 32, 42), i, np.float32) for i in range(7)]

    class DS:
        examples = 7

        def __iter__(self):
            return iter(batches)

    pf = ip.DevicePrefetcher(DS(), depth=2)
    assert pf.examples == 7
    for epoch in range(2):
        got = list(pf)
        assert len(got) == 7 and all(g.is_cuda for g in got)
        for i, g in enumerate(got):
            assert float(g.min()) == i == float(g.max())
