"""Generates tests/golden/*.npz from the float64 oracle (the reference has no golden vectors and cannot be run:
JAX 0.2.8 / flax 0.3.0 are not installable here).  Re-run: python scripts/make_golden.py"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ddpm_oracle as O  # noqa: E402
from smd_b200 import Engine, ModelConfig  # noqa: E402
from tests.util import oracle_kwargs, params_torch  # noqa: E402


def main():
    out = os.path.join(ROOT, "tests", "golden")
    os.makedirs(out, exist_ok=True)
    cfg = dict(num_layers=2, num_heads=8, num_mlp_layers=1, channels=42)
    eng = Engine(ModelConfig(**cfg), 4)
    seed, perturb = 11, 0.02
    flat = eng.init_params(seed, perturb=perturb)
    rng = np.random.default_rng(5)
    x = rng.uniform(-1, 1, (3, 32, 42)).astype(np.float32)
    t = rng.uniform(0.05, 1.0, (3,)).astype(np.float32)
    p64 = params_torch(eng, flat, torch.float64)
    kw = oracle_kwargs(eng.cfg)
    y64 = O.transformer_ddpm(p64, torch.from_numpy(x).double(), torch.from_numpy(t).double(), **kw).numpy()
    # one reverse step at t=500 with supplied noise, and the loss on supplied draws
    betas = O.create_noise_schedule(1e-6, 0.01, 1000, "linear")
    coef = O.reverse_coefficients(betas)
    z = rng.standard_normal(x.shape).astype(np.float32)
    nxt, _, mets = O.reverse_step(lambda a, c: O.transformer_ddpm(p64, a, c, **kw), torch.from_numpy(x).double(), 500,
                                  coef, torch.from_numpy(z).double())
    ap = O.alphas_prod_with_one(betas)
    labels = np.array([1, 400, 1000])
    used = ap[labels - 1]
    eps = rng.standard_normal(x.shape).astype(np.float32)
    loss, _ = O.diffusion_loss_tensors(lambda a, c: O.transformer_ddpm(p64, a, c, **kw), torch.from_numpy(x).double(),
                                       torch.from_numpy(used).double(), torch.from_numpy(eps).double(), "none")
    np.savez_compressed(os.path.join(out, "transformer_tiny.npz"), x=x, t=t, y64=y64, z=z, next64=nxt.numpy(),
                        metrics64=np.array([float(m) for m in mets]), used_alpha=used, eps=eps, loss64=loss.numpy(),
                        param_seed=seed, perturb=perturb, **cfg)
    print("wrote", os.path.join(out, "transformer_tiny.npz"))


if __name__ == "__main__":
    main()
