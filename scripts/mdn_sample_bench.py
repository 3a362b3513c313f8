"""Times TransformerMDN autoregressive sampling (smd_mdn_sample) at the mdn-mel-32seq-512 shape (L6 H8 K2 M2048,
C = 42 after --slice_ckpt, 100 mixture components) for N = 1000 samples, against the recompute loop the forward ABI
alone allows: 32 x smd_mdn_forward(shift=0) over the whole (N, 32, C) batch, each followed by smd_mdn_mixture_sample
over all N * 32 rows.  The two alternate, so both see the same machine state.  One JSON line reports the whole-call
times (CUDA events), launches per call, workspace bytes, and the card's name and power limit read in the same run.

The split of one smd_mdn_sample call into its 31 decode steps and its final step comes from a separate profiled call
(torch.profiler kernel timeline): decode = first kernel start to the start of the last embedding kernel (the final
step's full forward begins there), final = from there to the end of the last kernel.

    python scripts/mdn_sample_bench.py [--n 1000] [--steps 3] [--warmup 1] [--reps 2]
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
    ap.add_argument("--n", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from smd_b200 import Engine, ModelConfig, jrandom as random
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    cfg = ModelConfig(arch="TransformerMDN", num_layers=6, num_heads=8, num_mlp_layers=2, mlp_dims=2048, channels=42,
                      mdn_components=100)
    n, S, C = args.n, 32, 42
    eng = Engine(cfg, max_batch=n, sampler_T=S)
    flat = eng.init_params(seed=0)
    eng.set_params(flat)
    plain = Engine(cfg, max_batch=n)          # the recompute baseline runs on a plan without decode state
    plain.set_params(flat)
    rng = random.split(random.PRNGKey(1))[0]  # rng after `rng, model_rng = split(rng)`
    keys, r = [], rng
    for _ in range(S):
        r, embed = random.split(r)
        keys.append(embed)

    def cached():
        return eng.mdn_sample(rng, n)

    def recompute():
        tokens = torch.zeros((n, S, C), dtype=torch.float32, device="cuda")
        for i in range(S):
            pi, mu, ls = plain.mdn_forward(tokens, shift=False)
            nxt = plain.mdn_mixture_sample(pi, mu, ls, keys[i])
            if i < S - 1:
                tokens[:, i + 1] = nxt[:, i]
            else:
                tokens = nxt
        return tokens

    out = {"card": card, "n": n, "config": "mdn-mel-32seq-512 (L6 H8 K2 M2048 C42 Kc100)",
           "workspace_bytes_sampler_plan": eng.workspace_bytes, "workspace_bytes_plain_plan": plain.workspace_bytes}
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        for name, fn in (("cached", cached), ("recompute", recompute)):
            n0 = eng.launch_count()
            fn()
            torch.cuda.synchronize()
            out[f"{name}_launches"] = eng.launch_count() - n0
        times = {"cached": [], "recompute": []}
        for _ in range(args.reps):
            for name, fn in (("cached", cached), ("recompute", recompute)):
                times[name].append(_time(fn, args.steps, args.warmup))
        for name, t in times.items():
            out[f"{name}_ms"] = t
        out["speedup_median"] = float(np.median(times["recompute"]) / np.median(times["cached"]))
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            cached()
            torch.cuda.synchronize()
    kern = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA),
                  key=lambda e: e.time_range.start)
    kern = [e for e in kern if "memcpy" not in e.name.lower() and "memset" not in e.name.lower()]
    last_embed = max(i for i, e in enumerate(kern) if "embed" in e.name)
    t0, tf, t1 = kern[0].time_range.start, kern[last_embed].time_range.start, max(e.time_range.end for e in kern)
    out["profiled_decode_steps_ms"] = (tf - t0) / 1e3
    out["profiled_final_step_ms"] = (t1 - tf) / 1e3
    out["profiled_kernels"] = len(kern)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
