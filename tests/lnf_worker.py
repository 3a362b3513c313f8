"""Worker for tests/test_gpu_forward.py::test_ln_fused_epilogue.  Run with SMD_LNF=1 (and once more with
SMD_LNF_POST=1) so the res-block GEMMs finish the next LayerNorm -> FiLM -> swish in their epilogue (csrc/gemm_wgmma.cuh,
F_LNF).  Checks against the CPU oracle: forward at small / ragged / multi-round sizes (150 row blocks on at most 132 CTAs:
the inter-CTA statistics exchange crosses scheduling rounds), one reverse step through the graph + FiLM-table path,
gradient parity in training mode (the fused kernels also write the pre-LayerNorm copy and the statistics totals), and
that two runs are bit-identical."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ddpm_oracle as O  # noqa: E402
from tests.util import make_inputs, oracle_kwargs, params_torch, rel_l2  # noqa: E402


def main():
    assert os.environ.get("SMD_LNF") == "1"
    from smd_b200 import Engine, ModelConfig
    kw = dict(num_layers=1, num_heads=8, num_mlp_layers=2, channels=42)
    eng = Engine(ModelConfig(**kw), max_batch=600, cta_group=2)
    flat = eng.init_params(seed=1, perturb=0.02)
    eng.set_params(flat)
    p = params_torch(eng, flat)
    okw = oracle_kwargs(eng.cfg)
    for batch in (1, 5, 13, 600):
        x, t = make_inputs(batch, batch, (32, 42))
        n0 = eng.launch_count()
        y = eng.forward(torch.from_numpy(x).cuda(), torch.from_numpy(t).cuda())
        torch.cuda.synchronize()
        launches = eng.launch_count() - n0
        y2 = eng.forward(torch.from_numpy(x).cuda(), torch.from_numpy(t).cuda())
        ref = O.transformer_ddpm(p, torch.from_numpy(x), torch.from_numpy(t), emulate_bf16=True, **okw)
        ref32 = O.transformer_ddpm(p, torch.from_numpy(x), torch.from_numpy(t), **okw)
        e, e32 = rel_l2(y, ref), rel_l2(y, ref32)
        print(f"batch {batch}: rel-L2 vs bf16-emulating oracle {e:.3e}, vs fp32 {e32:.3e} ({launches} launches)", flush=True)
        assert e < 1e-2 and e32 < 1.2e-2, (e, e32)
        assert torch.equal(y, y2), "the fused forward pass must be bit-reproducible"
    # sampler: one reverse step with the FiLM table and the CUDA graph
    betas = O.create_noise_schedule(1e-6, 0.01, 1000, "linear")
    eng.sampler_setup(betas, key=(0, 3))
    rng = np.random.default_rng(0)
    x = torch.from_numpy(rng.standard_normal((600, 32, 42)).astype(np.float32))
    z = torch.from_numpy(rng.standard_normal((600, 32, 42)).astype(np.float32))
    nxt = eng.reverse_step(x.cuda(), 400, z=z.cuda())
    ref_next, _, _ = O.reverse_step(lambda a, c: O.transformer_ddpm(p, a, c, emulate_bf16=True, **okw), x, 400,
                                    O.reverse_coefficients(betas), z)
    e = rel_l2(nxt, ref_next)
    print(f"reverse step: rel-L2 {e:.3e}", flush=True)
    assert e < 1e-2
    del eng
    # training mode: gradients through the fused forward
    batch = 6
    eng = Engine(ModelConfig(**kw), max_batch=batch, cta_group=2, training=True)
    flat = eng.init_params(seed=2, perturb=0.05)
    eng.set_params(flat)
    eng.init_train_state()
    rng = np.random.default_rng(1)
    x0 = rng.uniform(-1, 1, (batch, 32, 42)).astype(np.float32)
    eps = rng.standard_normal((batch, 32, 42)).astype(np.float32)
    used = O.alphas_prod_with_one(betas)[rng.integers(1, 1001, batch) - 1].astype(np.float32)
    eng.compute_grads(torch.from_numpy(x0).cuda(), torch.from_numpy(used).cuda(), torch.from_numpy(eps).cuda())
    torch.cuda.synchronize()
    got = eng.flat_to_dict(eng.grads)
    pt = {k: v.clone().requires_grad_(True) for k, v in params_torch(eng, flat).items()}
    loss, _ = O.diffusion_loss_tensors(lambda a, c: O.transformer_ddpm(pt, a, c, **okw), torch.from_numpy(x0),
                                       torch.from_numpy(used), torch.from_numpy(eps), "mean")
    loss.backward()
    tot = sum(float((v.grad ** 2).sum()) for v in pt.values())
    dot = sum(float((torch.from_numpy(got[k]) * v.grad).sum()) for k, v in pt.items())
    nn_ = sum(float((torch.from_numpy(got[k]) ** 2).sum()) for k in pt)
    cos = dot / np.sqrt(nn_ * tot)
    print(f"training: loss {float(eng.loss_sum) / batch:.5f} vs {float(loss):.5f}, gradient cosine {cos:.6f}", flush=True)
    assert abs(float(eng.loss_sum) / batch - float(loss)) < 5e-3 * float(loss) and cos > 0.9995
    print("lnf-ok")


if __name__ == "__main__":
    main()
