"""Rebinding a plan's workspace (smd_bind_workspace) forgets every setup that described the old workspace's contents:
the objective and DSM schedules and the sampler chain with its replay graph have to be set up again, after which they
compute what a freshly created engine computes."""
import numpy as np
import pytest
import torch

from oracle import ddpm_oracle as O
from oracle import threefry as tf

pytestmark = pytest.mark.gpu

CFG = dict(arch="DenseNCSN", channels=512, num_layers=2, mlp_dims=2048)
BETAS = O.create_noise_schedule(1e-4, 0.02, 10, "linear")
SIGMAS = O.create_noise_schedule(1.0, 0.05, 4, "geometric")
KEY = tf.prng_key(7)


def _engine(flat=None):
    from smd_b200 import Engine, ModelConfig
    eng = Engine(ModelConfig(**CFG), max_batch=8, sampler_T=16)
    flat = eng.init_params(seed=4, perturb=0.02) if flat is None else flat
    eng.set_params(flat)
    return eng, flat


def _setups(eng):
    eng.objective_setup(BETAS)
    eng.dsm_setup(SIGMAS)
    eng.langevin_setup(SIGMAS, 3, 2e-5, "ald", key=(int(KEY[0]), int(KEY[1])))


def test_rebind_forgets_every_setup(lib):
    from smd_b200 import lib as L
    init = torch.from_numpy(np.random.default_rng(0).uniform(-1, 1, (8, 512)).astype(np.float32)).cuda()
    eng, flat = _engine()
    _setups(eng)
    x = init.clone()
    coll = torch.zeros((102, 8, 512), device="cuda")
    mets = torch.zeros((4, 4, 3), device="cuda")
    eng.langevin_sample(x, collection=coll, metrics=mets)   # captures the chain's graph
    torch.cuda.synchronize()

    # a second workspace; the first one stays allocated, so a replay of the old graph would read live memory
    first_ws = eng._ws
    eng._ws = torch.empty_like(first_ws)
    aligned = (eng._ws.data_ptr() + 1023) // 1024 * 1024
    L.check(eng.lib.smd_bind_workspace(eng._plan, aligned, eng.workspace_bytes))
    eng.repack()   # same parameter tensor: the chain's arguments (params, x, collection, metrics) are unchanged
    with pytest.raises(L.SmdError, match="smd_objective_setup has not been called"):
        eng.draws(KEY, 8)
    with pytest.raises(L.SmdError, match="smd_dsm_setup has not been called"):
        eng.dsm_draws(KEY, 8)
    with pytest.raises(L.SmdError, match="smd_langevin_setup has not been called"):
        eng.langevin_sample(x.copy_(init), collection=coll.zero_(), metrics=mets.zero_())
    with pytest.raises(L.SmdError, match="smd_sampler_setup has not been called"):
        eng.sample(x)

    # set up again: the same results as an engine that never saw the first workspace
    _setups(eng)
    eng.langevin_sample(x.copy_(init), collection=coll.zero_(), metrics=mets.zero_())
    fresh, _ = _engine(flat)
    _setups(fresh)
    ref_x, ref_c, ref_m = init.clone(), torch.zeros_like(coll), torch.zeros_like(mets)
    fresh.langevin_sample(ref_x, collection=ref_c, metrics=ref_m)
    torch.cuda.synchronize()
    assert torch.equal(x, ref_x) and torch.equal(coll, ref_c)
    torch.testing.assert_close(mets, ref_m, rtol=1e-6, atol=0)
    for a, b in zip(eng.draws(KEY, 8) + eng.dsm_draws(KEY, 8), fresh.draws(KEY, 8) + fresh.dsm_draws(KEY, 8)):
        assert torch.equal(a, b)
