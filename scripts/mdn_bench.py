"""Times the TransformerMDN train step (grads -> clip -> Adam) and the eval loss at the mdn-mel-32seq-512 shape
(L6 H8 K2 M2048, C = 42 after --slice_ckpt, 100 mixture components, batch 128), plus the head GEMM on its own.
Prints one JSON line with the card's name and power limit read in the same run.

    python scripts/mdn_bench.py [--steps 50] [--batch 128]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _time(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=128)
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from smd_b200 import Engine, ModelConfig
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    cfg = ModelConfig(arch="TransformerMDN", num_layers=6, num_heads=8, num_mlp_layers=2, mlp_dims=2048, channels=42,
                      mdn_components=100)
    B = args.batch
    eng = Engine(cfg, max_batch=B, training=True)
    eng.set_params(eng.init_params(seed=0))
    eng.init_train_state()
    x = torch.from_numpy(np.random.default_rng(0).uniform(-1, 1, (B, 32, 42)).astype(np.float32)).cuda()
    stream = torch.cuda.Stream()
    out = {"card": card, "batch": B, "workspace_bytes": eng.workspace_bytes, "params": eng.num_params}
    with torch.cuda.stream(stream):
        def step():
            eng.compute_mdn_grads(x)
            eng.apply_grads(3e-4)
        out["train_step_ms"] = _time(step, args.steps, args.warmup)
        n0 = eng.launch_count()
        step()
        out["train_step_launches"] = eng.launch_count() - n0
        out["eval_loss_ms"] = _time(lambda: eng.mdn_loss(x), args.steps, args.warmup)
        n0 = eng.launch_count()
        eng.mdn_loss(x)
        out["eval_loss_launches"] = eng.launch_count() - n0
        # the head GEMM's shape alone: [B*S, Md] x [Md, Np] bf16 -> fp32 with bias, through the smd_gemm_bf16 hook
        M, K = B * 32, cfg.mlp_dims
        Np = 2 * ((100 * 42 + 63) // 64 * 64) + 128
        a16 = torch.randn(M, K, device="cuda").bfloat16()
        w16 = torch.randn(K, Np, device="cuda").bfloat16()
        bias = torch.zeros(Np, device="cuda")
        y = torch.empty(M, Np, device="cuda")
        lib = eng.lib
        st = stream.cuda_stream

        def head():
            rc = lib.smd_gemm_bf16(a16.data_ptr(), w16.data_ptr(), M, Np, K, 0, 1, 128, 1, bias.data_ptr(), None, 0,
                                   y.data_ptr(), None, None, None, None, st)
            assert rc == 0
        ms = _time(head, args.steps, args.warmup)
        out["head_gemm_ms"] = ms
        out["head_gemm_tflops"] = 2.0 * M * K * Np / (ms * 1e-3) / 1e12
    print(json.dumps(out))


if __name__ == "__main__":
    main()
