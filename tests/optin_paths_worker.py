"""Worker for tests/test_gpu_train.py::test_opt_in_trunk_paths.  The switches are read once per process, so each variant
runs in its own process:
  SMD_ATTN_BLOCK_TRAIN=1  training forward through the attention block kernel (csrc/fused_wgmma.cuh: q | k | v,
                          probabilities and attention output written out for the backward pass);
  SMD_FFN_SPLITK=1        deterministic split-K (fp32 slabs) of the K = mlp_dims trunk GEMMs + ln128_reduce_fwd /
                          slab-summing ln128_bwd.
Checks: forward parity against the CPU oracle (inference engine), gradient parity with torch autograd on the oracle,
and bitwise repeatability of the gradients (both paths are atomics-free in the trunk forward)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ddpm_oracle as O  # noqa: E402
from tests.util import make_inputs, oracle_kwargs, params_torch, rel_l2  # noqa: E402


def main():
    assert os.environ.get("SMD_ATTN_BLOCK_TRAIN") == "1" or os.environ.get("SMD_FFN_SPLITK") == "1"
    from smd_b200 import Engine, ModelConfig
    for heads in (8, 16):
        kw = dict(num_layers=2, num_heads=heads, num_mlp_layers=1, channels=42)
        eng = Engine(ModelConfig(**kw), max_batch=40, cta_group=2)
        flat = eng.init_params(seed=1, perturb=0.02)
        eng.set_params(flat)
        p = params_torch(eng, flat)
        okw = oracle_kwargs(eng.cfg)
        for batch in (3, 40):       # 40 samples = 5 tiles of 256 tokens: several tiles, all splits
            x, t = make_inputs(batch, batch, (32, 42))
            y = eng.forward(torch.from_numpy(x).cuda(), torch.from_numpy(t).cuda())
            ref = O.transformer_ddpm(p, torch.from_numpy(x), torch.from_numpy(t), emulate_bf16=True, **okw)
            e = rel_l2(y, ref)
            print(f"heads {heads} batch {batch}: forward rel-L2 vs bf16-emulating oracle {e:.3e}", flush=True)
            assert e < 1e-2, e
        del eng
        batch = 9                    # 288 tokens: one full and one partial tile
        eng = Engine(ModelConfig(**kw), max_batch=batch, cta_group=2, training=True)
        flat = eng.init_params(seed=2, perturb=0.05)
        eng.set_params(flat)
        eng.init_train_state()
        rng = np.random.default_rng(5)
        x0 = rng.uniform(-1, 1, (batch, 32, 42)).astype(np.float32)
        used = rng.uniform(0.05, 0.99, (batch,)).astype(np.float32)
        eps = rng.standard_normal((batch, 32, 42)).astype(np.float32)
        args = (torch.from_numpy(x0).cuda(), torch.from_numpy(used).cuda(), torch.from_numpy(eps).cuda())
        eng.compute_grads(*args)
        torch.cuda.synchronize()
        loss1 = float(eng.loss_mean)
        got = eng.flat_to_dict(eng.grads)
        pr = {k: v.clone().requires_grad_(True) for k, v in params_torch(eng, flat).items()}
        loss, _ = O.diffusion_loss_tensors(lambda a, c: O.model_apply("TransformerDDPM", pr, a, c, emulate_bf16=False, **okw),
                                           torch.from_numpy(x0), torch.from_numpy(used), torch.from_numpy(eps), "mean")
        loss.backward()
        dot = n1 = n2 = 0.0
        worst = 0.0
        for k, v in pr.items():
            g = v.grad if v.grad is not None else torch.zeros_like(v)
            gg = torch.from_numpy(got[k])
            dot += float((gg * g).sum()); n1 += float((gg ** 2).sum()); n2 += float((g ** 2).sum())
            if float((g ** 2).sum()) > 0 and ("attn" in k or "ffn" in k or "ln" in k):
                worst = max(worst, rel_l2(gg, g))
        cos = dot / np.sqrt(n1 * n2)
        print(f"heads {heads}: loss {loss1:.6f} vs {float(loss):.6f}, gradient cosine {cos:.6f}, worst trunk tensor rel-L2 {worst:.3e}",
              flush=True)
        assert abs(loss1 - float(loss)) < 5e-3 * float(loss)
        assert cos > 0.9995, cos
        assert worst < 5e-2, worst
        # the loss (forward) is bit-reproducible on these paths
        eng.compute_grads(*args)
        torch.cuda.synchronize()
        assert float(eng.loss_mean) == loss1
        del eng
    print("optin-ok")


if __name__ == "__main__":
    main()
