"""TransformerDDPM at sequence lengths 32 / 64 / 128 with the token count per step held fixed (single GPU, synthetic
data, random-init weights):
  * train step, base config (ddpm-mel-32seq-512.cfg: L6 H8 K2 M2048, C = 42), 4096 tokens: batch 128 / 64 / 32;
  * one reverse-diffusion step (CUDA-graph replay), same model, 32 000 tokens: n = 1000 / 500 / 250.
Prints one JSON object: ms/step and tokens/s per length, the card's name and power limit read in the same run, and
smd_workspace_bytes of the training plans (base and large config) at 4096 tokens.  Nothing about speed is asserted.
  python scripts/seq_len_bench.py [--steps 30 --warmup 5]
  python scripts/seq_len_bench.py --profile      # torch.profiler run of its own: attention kernels' share of each step"""
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

BASE = dict(num_layers=6, num_heads=8, num_mlp_layers=2, mlp_dims=2048, channels=42)
LARGE = dict(num_layers=8, num_heads=16, num_mlp_layers=3, mlp_dims=2048, channels=42)
LENGTHS = (32, 64, 128)
TRAIN_TOKENS, SAMPLE_TOKENS = 4096, 32000
ATTENTION_KERNELS = ("attention_kernel", "attention_mma_kernel", "attention_bwd", "attn_block_kernel")


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return r.stdout.strip()


def train_job(S):
    B = TRAIN_TOKENS // S
    eng = Engine(ModelConfig(seq_len=S, **BASE), max_batch=B, cta_group=2, training=True)
    eng.set_params(eng.init_params(seed=1))
    eng.init_train_state(ema=False)
    eng.objective_setup(np.linspace(1e-6, 0.01, 1000, dtype=np.float32))
    x = torch.from_numpy(np.random.default_rng(0).uniform(-1, 1, (B, S, 42)).astype(np.float32)).cuda()

    def step(i):
        u, e = eng.draws((i, 17), B)
        eng.train_step(x, u, e, lr=1e-3)
    return step


def sample_job(S):
    n = SAMPLE_TOKENS // S
    eng = Engine(ModelConfig(seq_len=S, **BASE), max_batch=n, cta_group=2)
    eng.set_params(eng.init_params(seed=1))
    eng.sampler_setup(np.linspace(1e-6, 0.01, 1000, dtype=np.float32), key=(0, 5))
    x = torch.randn(n, S, 42, device="cuda")
    return lambda i: eng.sample(x, steps=1, use_graph=True)


def timed(step, steps, warmup):
    for i in range(warmup):
        step(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        step(warmup + i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def attention_share(step, warmup, steps):
    from torch.profiler import ProfilerActivity, profile
    for i in range(warmup):
        step(i)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(steps):
            step(warmup + i)
        torch.cuda.synchronize()
    total = attn = 0.0
    for ev in prof.key_averages():
        t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        total += t
        if any(k in ev.key for k in ATTENTION_KERNELS):
            attn += t
    return attn / total if total else float("nan")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "seq_len_bench.py needs a CUDA device"
    torch.cuda.set_stream(torch.cuda.Stream())
    out = {"card": card(), "train_tokens": TRAIN_TOKENS, "sample_tokens": SAMPLE_TOKENS}
    for S in LENGTHS:
        for name, make, tokens in (("train", train_job, TRAIN_TOKENS), ("sample", sample_job, SAMPLE_TOKENS)):
            step = make(S)
            if args.profile:
                out[f"{name}_S{S}_attention_share"] = round(attention_share(step, args.warmup, 10), 4)
            else:
                ms = timed(step, args.steps, args.warmup)
                out[f"{name}_S{S}_ms"] = round(ms, 4)
                out[f"{name}_S{S}_tokens_per_s"] = round(tokens / ms * 1e3, 1)
            del step
            torch.cuda.empty_cache()
    for cname, kw in (("base", BASE), ("large", LARGE)):
        for S in LENGTHS:
            eng = Engine(ModelConfig(seq_len=S, **kw), max_batch=TRAIN_TOKENS // S, training=True)
            out[f"train_workspace_MiB_{cname}_S{S}"] = round(eng.workspace_bytes / 2 ** 20, 1)
    # the bench.py batch (128 sequences) at S = 128: the [B][H][S][S] probabilities are 16x those at S = 32
    for S in (32, 128):
        eng = Engine(ModelConfig(seq_len=S, **LARGE), max_batch=128, training=True)
        out[f"train_workspace_MiB_large_S{S}_batch128"] = round(eng.workspace_bytes / 2 ** 20, 1)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
