"""Score-network parity: CUDA path (through the C ABI) vs the CPU oracle on the same seeded inputs.

Tolerances (stated): vs the bf16-operand-emulating oracle rel-L2 <= 1e-2 (kernel logic; only accumulation order,
fast-exp and flipped bf16 roundings differ -- measured 2e-3 at 2 layers, 4e-3 at 6); vs the true fp32/fp64 oracle rel-L2
<= 1.2e-2 and max-abs <= 6e-2 on eps_hat, |d loss| <= 5e-3 loss per example (bf16 tensor-core operands, fp32 accumulate --
about 2x the errors tests/test_gpu_bench_shapes.py records at the benchmarked sizes; SURVEY section 7)."""
import os

import numpy as np
import pytest
import torch

from oracle import ddpm_oracle as O
from tests.util import TRANSFORMER_CASES, make_inputs, oracle_kwargs, params_torch, rel_l2

pytestmark = pytest.mark.gpu


def _engine(kw, batch, cg, arch="TransformerDDPM"):
    from smd_b200 import Engine, ModelConfig
    cfg = ModelConfig(arch=arch, **kw)
    eng = Engine(cfg, max_batch=batch, cta_group=cg)
    flat = eng.init_params(seed=1, perturb=0.02)
    eng.set_params(flat)
    return eng, flat


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("case", list(TRANSFORMER_CASES))
def test_transformer_forward_parity(lib, case, cg):
    kw, batch = TRANSFORMER_CASES[case]
    eng, flat = _engine(kw, batch, cg)
    x, t = make_inputs(7, batch, (32, kw["channels"]))
    y = eng.forward(torch.from_numpy(x).cuda(), torch.from_numpy(t).cuda())
    torch.cuda.synchronize()
    okw = oracle_kwargs(eng.cfg)
    p = params_torch(eng, flat)
    ref_bf = O.transformer_ddpm(p, torch.from_numpy(x), torch.from_numpy(t), emulate_bf16=True, **okw)
    ref32 = O.transformer_ddpm(p, torch.from_numpy(x), torch.from_numpy(t), **okw)
    assert rel_l2(y, ref_bf) < 1e-2
    assert rel_l2(y, ref32) < 1.2e-2
    assert float((y.cpu() - ref32).abs().max()) < 6e-2


def test_forward_batch_ragged_and_broadcast_t(lib):
    kw, _ = TRANSFORMER_CASES["tiny"]
    eng, flat = _engine(kw, 600, 2)
    p = params_torch(eng, flat)
    okw = oracle_kwargs(eng.cfg)
    # 32, 160, 416 token rows: partial 128/256-row tiles; 19200 rows: more tiles than SMs, several scheduling rounds
    for batch in (1, 5, 13, 600):
        x, _ = make_inputs(batch, batch, (32, 42))
        t = np.full((batch,), 0.37, np.float32)
        y = eng.forward(torch.from_numpy(x).cuda(), torch.tensor([0.37], device="cuda"))  # broadcast t
        ref = O.transformer_ddpm(p, torch.from_numpy(x), torch.from_numpy(t), emulate_bf16=True, **okw)
        assert rel_l2(y, ref) < 1e-2
    # the LayerNorm statistics are added in a fixed order: the same forward twice is bit-identical
    y2 = eng.forward(torch.from_numpy(x).cuda(), torch.tensor([0.37], device="cuda"))
    assert torch.equal(y, y2)


def test_dense_ddpm_forward_parity(lib):
    # configs/ddpm-mel-1seq-512.cfg: DenseDDPM, (B=8, 512) latents, num_layers = flag default 6
    eng, flat = _engine(dict(num_layers=6, channels=512), 8, 2, arch="DenseDDPM")
    x, t = make_inputs(3, 8, (512,))
    y = eng.forward(torch.from_numpy(x).cuda(), torch.from_numpy(t).cuda())
    p = params_torch(eng, flat)
    okw = oracle_kwargs(eng.cfg)
    ref_bf = O.dense_ddpm(p, torch.from_numpy(x), torch.from_numpy(t), emulate_bf16=True, **okw)
    ref32 = O.dense_ddpm(p, torch.from_numpy(x), torch.from_numpy(t), **okw)
    assert rel_l2(y, ref_bf) < 1e-2
    assert rel_l2(y, ref32) < 1.2e-2


def test_golden_fixture(lib):
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "transformer_tiny.npz"))
    kw = dict(num_layers=int(g["num_layers"]), num_heads=int(g["num_heads"]),
              num_mlp_layers=int(g["num_mlp_layers"]), channels=int(g["channels"]))
    from smd_b200 import Engine, ModelConfig
    eng = Engine(ModelConfig(**kw), max_batch=3, cta_group=2)
    eng.set_params(eng.init_params(int(g["param_seed"]), perturb=float(g["perturb"])))
    y = eng.forward(torch.from_numpy(g["x"]).cuda(), torch.from_numpy(g["t"]).cuda())
    assert rel_l2(y, torch.from_numpy(g["y64"])) < 1.2e-2
    loss = eng.ddpm_loss(torch.from_numpy(g["x"]).cuda(), torch.from_numpy(g["used_alpha"]).cuda(),
                         torch.from_numpy(g["eps"]).cuda())
    np.testing.assert_allclose(loss.cpu().numpy(), g["loss64"], rtol=5e-3)


def test_ddpm_loss_parity(lib):
    kw, batch = TRANSFORMER_CASES["base_c42"]
    eng, flat = _engine(kw, batch, 2)
    rng = np.random.default_rng(2)
    x0 = rng.uniform(-1, 1, (batch, 32, 42)).astype(np.float32)
    eps = rng.standard_normal((batch, 32, 42)).astype(np.float32)
    betas = O.create_noise_schedule(1e-6, 0.01, 1000, "linear")
    ap = O.alphas_prod_with_one(betas)
    used = ap[np.array([1, 250, 700, 1000]) - 1]
    loss, pred = eng.ddpm_loss(torch.from_numpy(x0).cuda(), torch.from_numpy(used).cuda(),
                               torch.from_numpy(eps).cuda(), want_pred=True)
    p = params_torch(eng, flat)
    okw = oracle_kwargs(eng.cfg)
    ref, ref_pred = O.diffusion_loss_tensors(lambda a, c: O.transformer_ddpm(p, a, c, **okw), torch.from_numpy(x0),
                                             torch.from_numpy(used), torch.from_numpy(eps), "none")
    assert rel_l2(pred, ref_pred) < 1.2e-2
    # |d loss| <= 5e-3 * loss per example (stated tolerance on ddpm_loss for bf16 operands; measured 2e-3 worst case)
    np.testing.assert_allclose(loss.cpu().numpy(), ref.numpy(), rtol=5e-3)


def test_fused_ffn_kernel(lib):
    """The fused FFN kernel (csrc/fused_wgmma.cuh) takes over each layer's two FFN GEMMs in inference from 8192 tokens
    on.  Parity with the oracle at exactly 8192 tokens, with a partial 128-row tile (259 samples) and with more tiles
    than SMs (600 samples: CTAs that run two tiles wrap every barrier phase); 255 samples still run the two GEMMs."""
    kw = dict(num_layers=2, num_heads=8, num_mlp_layers=1, channels=42)
    eng, flat = _engine(kw, 600, 2)
    p = params_torch(eng, flat)
    okw = oracle_kwargs(eng.cfg)
    launches = {}
    for batch in (255, 256, 259, 600):
        x, t = make_inputs(batch, batch, (32, 42))
        n0 = eng.launch_count()
        y = eng.forward(torch.from_numpy(x).cuda(), torch.from_numpy(t).cuda())
        torch.cuda.synchronize()
        launches[batch] = eng.launch_count() - n0
        ref = O.transformer_ddpm(p, torch.from_numpy(x), torch.from_numpy(t), emulate_bf16=True, **okw)
        assert rel_l2(y, ref) < 1e-2, batch
    assert launches[256] == launches[255] - kw["num_layers"], launches
