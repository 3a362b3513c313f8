"""Sliced vs denoising score matching on the ncsn-mel-1seq-512 shape (DenseNCSN, C = 512, 6 blocks, mlp 2048,
batch 128; single GPU, synthetic data, random-init weights): the DSM train step, the SSM train step (tangent pass +
second-order backward, CUDA-graph replay on a private stream) and the SSM eval loss.  Prints one JSON object: ms per
call, kernel launches per call, the SSM / DSM train-step ratio and the card's name and power limit read in the same
run.  Nothing about speed is asserted.
  python scripts/ssm_bench.py [--steps 50 --warmup 10]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from smd_b200 import Engine, ModelConfig  # noqa: E402

CFG = dict(arch="DenseNCSN", num_layers=6, mlp_dims=2048, channels=512)
BATCH = 128


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return r.stdout.strip()


def timed(eng, fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    l0 = eng.launch_count()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / steps, (eng.launch_count() - l0) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    torch.cuda.set_stream(torch.cuda.Stream())     # capturable: the train step replays from a CUDA graph
    sigmas = np.exp(np.linspace(np.log(1.0), np.log(0.01), 15)).astype(np.float32)
    eng = Engine(ModelConfig(**CFG), max_batch=BATCH, training=True)
    eng.set_params(eng.init_params(seed=1))
    eng.init_train_state()
    eng.dsm_setup(sigmas)
    x0 = torch.randn(BATCH, CFG["channels"], device="cuda")
    used, eps, v = eng.ssm_draws((0, 7), BATCH)

    def dsm_step():
        eng.compute_dsm_grads(x0, used, eps)
        eng.apply_grads(1e-4)

    def ssm_step():
        eng.compute_ssm_grads(x0, used, eps, v)
        eng.apply_grads(1e-4)

    inf = Engine(ModelConfig(**CFG), max_batch=BATCH)
    inf.set_params(eng.params.clone())
    out = {"config": dict(CFG, batch=BATCH), "card": card()}
    for name, e, fn in (("dsm_train_step", eng, dsm_step), ("ssm_train_step", eng, ssm_step),
                        ("ssm_eval_loss", inf, lambda: inf.ssm_loss(x0, used, eps, v))):
        ms, launches = timed(e, fn, args.steps, args.warmup)
        out[name] = {"ms": round(ms, 4), "launches": launches}
    out["ssm_over_dsm_train"] = round(out["ssm_train_step"]["ms"] / out["dsm_train_step"]["ms"], 3)
    out["workspace_mb"] = {"train": round(eng.workspace_bytes / 2 ** 20, 1), "inference": round(inf.workspace_bytes / 2 ** 20, 1)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
