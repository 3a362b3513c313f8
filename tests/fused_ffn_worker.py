"""Worker for tests/test_gpu_forward.py::test_fused_ffn_kernel.  Run with SMD_FFN_FUSED=2 so that the fused FFN kernel
(csrc/fused_wgmma.cuh) is used at every size and in training mode; checks it against the CPU oracle:
  * small and ragged batches (partial 128-token tiles), inference;
  * 600 samples = 150 tiles on at most 132 CTAs (CTAs that run two tiles exercise every barrier phase wrap);
  * training mode: saved hidden activations feed the backward pass -> gradient parity with torch autograd."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ddpm_oracle as O  # noqa: E402
from tests.util import make_inputs, oracle_kwargs, params_torch, rel_l2  # noqa: E402


def main():
    assert os.environ.get("SMD_FFN_FUSED") == "2"
    from smd_b200 import Engine, ModelConfig
    kw = dict(num_layers=2, num_heads=8, num_mlp_layers=1, channels=42)
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
        ref = O.transformer_ddpm(p, torch.from_numpy(x), torch.from_numpy(t), emulate_bf16=True, **okw)
        e = rel_l2(y, ref)
        print(f"batch {batch}: rel-L2 vs bf16-emulating oracle {e:.3e} ({launches} launches)", flush=True)
        assert e < 1e-2, e
    del eng
    # training mode
    batch = 6
    eng = Engine(ModelConfig(**kw), max_batch=batch, cta_group=2, training=True)
    flat = eng.init_params(seed=2, perturb=0.05)
    eng.set_params(flat)
    eng.init_train_state()
    rng = np.random.default_rng(5)
    x0 = rng.uniform(-1, 1, (batch, 32, 42)).astype(np.float32)
    used = rng.uniform(0.05, 0.99, (batch,)).astype(np.float32)
    eps = rng.standard_normal((batch, 32, 42)).astype(np.float32)
    eng.compute_grads(torch.from_numpy(x0).cuda(), torch.from_numpy(used).cuda(), torch.from_numpy(eps).cuda())
    torch.cuda.synchronize()
    got = eng.flat_to_dict(eng.grads)
    pr = {k: v.clone().requires_grad_(True) for k, v in params_torch(eng, flat).items()}
    loss, _ = O.diffusion_loss_tensors(lambda a, c: O.model_apply("TransformerDDPM", pr, a, c, emulate_bf16=False, **okw),
                                       torch.from_numpy(x0), torch.from_numpy(used), torch.from_numpy(eps), "mean")
    loss.backward()
    dot = n1 = n2 = 0.0
    for k, v in pr.items():
        g = v.grad if v.grad is not None else torch.zeros_like(v)
        gg = torch.from_numpy(got[k])
        dot += float((gg * g).sum()); n1 += float((gg ** 2).sum()); n2 += float((g ** 2).sum())
    cos = dot / np.sqrt(n1 * n2)
    print(f"training: gradient cosine {cos:.6f}, norm ratio {np.sqrt(n1 / n2):.4f}", flush=True)
    assert cos > 0.999 and abs(np.sqrt(n1 / n2) - 1) < 2e-2
    print("fused-ok", flush=True)


if __name__ == "__main__":
    main()
