"""torchrun worker: the data-parallel TransformerMDN gradient over W ranks (each rank its rows, scaled by the global
token count, SUM all-reduce) must equal the single-rank gradient of the whole batch up to summation order.  Launched by
tests/test_gpu_mdn.py; prints 'mdn-dp-ok' on rank 0."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from smd_b200 import Engine, ModelConfig, parallel  # noqa: E402


def main():
    parallel.init_from_env("nccl")
    w, r = parallel.world_size(), parallel.rank()
    cfg = ModelConfig(arch="TransformerMDN", num_layers=2, num_heads=8, num_mlp_layers=1, mlp_dims=512, channels=42,
                      mdn_components=16)
    B = 4 * w
    x = np.random.default_rng(0).uniform(-1, 1, (B, 32, 42)).astype(np.float32)
    dev = torch.device("cuda", torch.cuda.current_device())

    def make(max_batch):
        e = Engine(cfg, max_batch=max_batch, training=True)
        e.set_params(e.init_params(seed=7, perturb=0.02))
        e.init_train_state()
        return e

    e_dp = make(B // w)
    e_dp.compute_mdn_grads(torch.from_numpy(x[r * (B // w):(r + 1) * (B // w)]).to(dev), global_batch=B)
    e_dp.reduce_grads(w)
    e_1 = make(B)
    e_1.compute_mdn_grads(torch.from_numpy(x).to(dev))
    torch.cuda.synchronize()
    if r == 0:
        g_dp, g_1 = e_dp.grads.double(), e_1.grads.double()
        err = float((g_dp - g_1).norm() / g_1.norm())
        l_dp, l_1 = float(e_dp.loss_mean), float(e_1.loss_mean)
        print(f"mdn dp: grad rel-L2 {err:.3e}, mean loss {l_dp:.6f} vs {l_1:.6f}")
        assert err < 1e-2 and abs(l_dp - l_1) < 1e-5 * abs(l_1), (err, l_dp, l_1)
        print("mdn-dp-ok")
    parallel.shutdown()


if __name__ == "__main__":
    main()
