"""Cost of one training snapshot with --snapshot_sampling: the sampler chain train_ncsn.snapshot_sampling runs
(train_ncsn.sample on the inference engine bound to the EMA arena) and the GPU metrics it scores the samples with.

    python scripts/snapshot_bench.py [--schedules short,mel] [--eval_samples 3000] [--out snapshot_bench.json]

Workload: DenseNCSN C = 512, 6 blocks, mlp 2048 (ncsn-mel-1seq-512.cfg).  Schedules: "short" (10 levels x 10
steps) and "mel" (the config's 500 levels x 100 steps, sigma 15 -> 0.01, epsilon 9.64e-7), annealed Langevin
dynamics with the denoising step.  Prints one JSON line per schedule (seconds for the chain, launches, ms per step,
seconds for latent_metrics against 3000 real rows), one line with the workspace of the training plan (batch 128) and
of the inference plan the sampler adds, then a table.  The card's name and power limit are part of every line."""
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

SCHEDULES = {"short": (10, 10, 1.0, 2e-6), "mel": (500, 100, 15.0, 9.64e-7)}   # levels, steps, sigma_begin, epsilon


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--schedules", default="short,mel")
    ap.add_argument("--eval_samples", type=int, default=3000)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("snapshot_bench needs a CUDA device")
    import __graft_entry__ as g
    g.build()
    from smd_b200 import ebm_utils, jrandom as random, metrics, ncsn, nn, train_ncsn, train_utils
    torch.cuda.set_stream(torch.cuda.Stream())     # train() samples on a private (capturable) stream too
    dev_card = card()
    n, shape = args.eval_samples, (512,)
    module = ncsn.DenseNCSN.partial(num_layers=6, num_heads=8, num_mlp_layers=2, mlp_dims=2048)
    _, params = module.init_by_shape(random.PRNGKey(0), [((128, 512), np.float32), ((128, 1), np.float32)])
    model = nn.Model(module, params)
    train_eng = model.engine(128, training=True)
    train_eng.init_train_state()
    ema = train_utils.EMAHelper(0.999, model.arena.clone())
    scorenet = model.replace(params=ema.params)
    rng = np.random.default_rng(0)
    real = torch.from_numpy(rng.uniform(-1, 1, (n,) + shape).astype(np.float32)).cuda()
    lines = []
    for name in args.schedules.split(","):
        L, T, sigma_begin, eps = SCHEDULES[name]
        sigmas = ebm_utils.create_noise_schedule(sigma_begin, 0.01, L, "geometric")
        key = random.PRNGKey(11)
        # warm-up: engine creation, weight packing, graph capture of a two-level chain
        train_ncsn.sample(scorenet, sigmas[:2], key, shape, num_samples=n, epsilon=eps, steps=2)
        ema.params.bump()                      # the arena moved (as after a train step): the next call re-packs
        torch.cuda.synchronize()
        eng = scorenet.engine(n)
        l0 = eng.launch_count()
        t0 = time.perf_counter()
        gen, _, _ = train_ncsn.sample(scorenet, sigmas, key, shape, num_samples=n, epsilon=eps, steps=T)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        launches = eng.launch_count() - l0
        t1 = time.perf_counter()
        scores = metrics.latent_metrics(real, gen)
        torch.cuda.synchronize()
        dm = time.perf_counter() - t1
        rec = dict(schedule=name, levels=L, steps_per_level=T, eval_samples=n, card=dev_card, sample_s=dt,
                   ms_per_step=1e3 * dt / (L * T), launches=launches, launches_per_step=launches / (L * T),
                   metrics_s=dm, finite=bool(torch.isfinite(gen).all()), frechet_distance=scores["frechet_distance"])
        print(json.dumps(rec), flush=True)
        lines.append(rec)
    ws = dict(card=dev_card, training_plan_mib=train_eng.workspace_bytes / 2 ** 20,
              inference_plan_mib=scorenet.engine(n).workspace_bytes / 2 ** 20, inference_max_batch=n)
    print(json.dumps(ws), flush=True)
    print(f"\n{dev_card}: DenseNCSN C=512 L6 M2048, {n} samples")
    print("| schedule | steps | chain | ms / step | launches / step | latent_metrics |")
    print("|---|---|---|---|---|---|")
    for r in lines:
        print(f"| {r['schedule']} ({r['levels']} x {r['steps_per_level']}) | {r['levels'] * r['steps_per_level']} | "
              f"{r['sample_s']:.2f} s | {r['ms_per_step']:.3f} | {r['launches_per_step']:.2f} | {r['metrics_s']:.2f} s |")
    print(f"workspace: training plan (batch 128) {ws['training_plan_mib']:.1f} MiB, inference plan (max_batch {n}) "
          f"{ws['inference_plan_mib']:.1f} MiB")
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(lines + [ws], f, indent=1)


if __name__ == "__main__":
    main()
