"""Annealed Langevin dynamics: the former per-step Python loop (reproduced below) against the device chain
(smd_langevin_sample, CUDA-graph replay), alternated in one process on the same seeded inputs.

    python scripts/langevin_bench.py [--levels 20 --steps 100] [--repeats 3] [--out langevin_bench.json]

Workloads: DenseNCSN C = 512, 6 blocks, mlp 2048 (a slice of ncsn-mel-1seq-512) and TransformerDDPM 32x42 (the base
configuration), each at N = 1000 and at N = 125 (one rank's share of 8).  Prints one JSON line per workload with
ms per step, launches per step (smd_launch_count) and how far the two outputs are apart, plus the card's name and
power limit.  The per-step cost does not depend on the number of levels, so --levels / --steps may shorten a run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = {
    "dense512": (dict(arch="DenseNCSN", channels=512, num_layers=6, mlp_dims=2048), (512,), 20),
    "transformer32x42": (dict(arch="TransformerDDPM"), (32, 42), 15),
}


def python_loop(eng, sigmas, T, epsilon, key, x, infill=None):
    """The Python step loop annealed_langevin_dynamics ran before the device chain: a host split, Engine.forward and
    Engine.langevin_step per step (collection and metrics as there)."""
    from smd_b200 import ebm_utils, jrandom as random
    sig = np.asarray(sigmas, np.float32)
    L = len(sig)
    collection = torch.zeros((102,) + tuple(x.shape), device=x.device)
    collection[0] = x
    slot_of = ebm_utils._collection_slot_fn(L * T, 100)
    metrics = torch.zeros((L, T, 4), device=x.device)
    sigma_dev = torch.empty((1,), device=x.device)
    grad = torch.empty_like(x)
    k = np.asarray(key, np.uint32)
    for si in range(L):
        s = np.float32(sig[si])
        alpha = np.float32(epsilon) * (s / np.float32(sig[-1])) ** 2
        sigma_dev.copy_(torch.tensor([float(s)]))
        for i in range(T):
            k, step_key, infill_key = random.split(k, 3)
            eng.forward(x, sigma_dev, out=grad)
            slot = slot_of(si * T + i + 1)
            if slot >= collection.shape[0]:
                slot = -1
            eng.langevin_step(x, grad, float(alpha), float(np.sqrt(np.float32(2) * alpha)), step_key=step_key,
                              infill_sigma=float(s), infill_key=infill_key, x_next=x,
                              collection_slot=collection[slot] if slot >= 0 else None, metrics4=metrics[si, i])
    return x


def device_chain(eng, sigmas, T, epsilon, key, x):
    L = len(sigmas)
    collection = torch.zeros((102,) + tuple(x.shape), device=x.device)
    collection[0] = x
    metrics = torch.zeros((4, L, T), device=x.device)
    eng.langevin_setup(sigmas, T, epsilon, "ald", key=(int(key[0]), int(key[1])))
    eng.langevin_sample(x, denoise=False, collection=collection, metrics=metrics)
    return x


def timed(fn, eng):
    torch.cuda.synchronize()
    l0 = eng.launch_count()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0, eng.launch_count() - l0


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--levels", type=int, default=0, help="noise levels (0: the workload's 20 / 15)")
    ap.add_argument("--steps", type=int, default=100, help="steps per level")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--batches", default="1000,125")
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("langevin_bench needs a CUDA device")
    import __graft_entry__ as g
    g.build()
    from smd_b200 import Engine, ModelConfig, ebm_utils
    from smd_b200 import jrandom as random
    dev_card = card()
    lines = []
    for name in args.workloads.split(","):
        cfg, shape, levels = WORKLOADS[name]
        L = args.levels or levels
        sigmas = ebm_utils.create_noise_schedule(1.0, 0.01, L, "geometric")
        for n in (int(b) for b in args.batches.split(",")):
            eng = Engine(ModelConfig(**cfg), max_batch=n)
            eng.set_params(eng.init_params(seed=1, perturb=0.02))
            key = random.PRNGKey(7)
            rho = float(np.sqrt(np.float32(12)) / 2)
            init = random.uniform(random.PRNGKey(3), (n,) + shape, -rho, rho)
            steps = L * args.steps
            t_loop, t_chain, launches = [], [], {}
            # warm-up of both paths (module load, graph capture), then alternate
            python_loop(eng, sigmas[:2], 2, 2e-6, key, init.clone())
            device_chain(eng, sigmas[:2], 2, 2e-6, key, init.clone())
            for _ in range(args.repeats):
                a, dt, nl = timed(lambda: python_loop(eng, sigmas, args.steps, 2e-6, key, init.clone()), eng)
                t_loop.append(dt)
                launches["loop"] = nl / steps
                b, dt, nl = timed(lambda: device_chain(eng, sigmas, args.steps, 2e-6, key, init.clone()), eng)
                t_chain.append(dt)
                launches["chain"] = nl / steps
            diff = (a - b).abs()
            rec = dict(workload=name, n=n, levels=L, steps_per_level=args.steps, card=dev_card,
                       loop_ms_per_step=1e3 * min(t_loop) / steps, chain_ms_per_step=1e3 * min(t_chain) / steps,
                       loop_ms_spread=[1e3 * t / steps for t in t_loop],
                       chain_ms_spread=[1e3 * t / steps for t in t_chain],
                       loop_launches_per_step=launches["loop"], chain_launches_per_step=launches["chain"],
                       speedup=min(t_loop) / min(t_chain), bitwise_equal=bool(torch.equal(a, b)),
                       max_abs_diff=float(diff.max()),
                       rel_l2=float((a - b).norm() / b.norm()))
            print(json.dumps(rec), flush=True)
            lines.append(rec)
            del eng
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
