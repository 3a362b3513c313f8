"""DPM-Solver++ (smd_dpm_sample) against DDIM at eta = 0 (smd_ddim_sample): per-step cost, and the ODE
discretisation error of each solver over the number of steps on a briefly trained model.

    python scripts/dpm_bench.py [--repeats 3] [--train_steps 400] [--out dpm_bench.json]

1. Per step: the DDIM chain and the order-2 and order-3 DPM-Solver++ chains on the same engine and init at N = 1000
   over a T = 1000 linear schedule (1e-4 .. 0.02), --chain_steps uniform levels each, alternated --repeats times (the
   fastest repeat is reported, with the spread).  Workloads: TransformerDDPM base (L6 H8, mlp 2048, C = 42) at S = 32
   and S = 128, and DenseDDPM C = 512 (3 blocks, mlp 2048).  Launches per step from smd_launch_count.
2. ODE error: train_ncsn trains a TransformerDDPM (L2, 32 x 42) on --synthetic latents for --train_steps steps.  From
   one x_T ~ N(0, 1) of 1000 samples, DDIM eta = 0, DPM order 2 and DPM order 3 run at K in {10, 20, 50, 100} uniform
   levels; each is compared with the same solver's K = 1000 solution, rel-L2 in normalised units.
Prints one JSON line per measurement, with the card's name and power limit; --out collects them."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import textwrap
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = {
    "transformer_s32_c42": (dict(arch="TransformerDDPM", seq_len=32), (32, 42)),
    "transformer_s128_c42": (dict(arch="TransformerDDPM", seq_len=128), (128, 42)),
    "dense_c512": (dict(arch="DenseDDPM", channels=512, num_layers=3), (512,)),
}
KS = (10, 20, 50, 100)
SOLVERS = ("ddim", "dpm2", "dpm3")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, eng):
    torch.cuda.synchronize()
    l0 = eng.launch_count()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, eng.launch_count() - l0


def per_step(args, betas, emit):
    from smd_b200 import Engine, ModelConfig
    from smd_b200 import jrandom as random
    n, k = 1000, args.chain_steps
    steps = np.linspace(0, 999, k).round().astype(np.int32)
    for name, (cfg, shape) in WORKLOADS.items():
        eng = Engine(ModelConfig(**cfg), max_batch=n)
        eng.set_params(eng.init_params(seed=1, perturb=0.02))
        init = random.normal(random.PRNGKey(3), (n,) + shape)
        coll = torch.zeros((41, n) + shape, device="cuda")
        mets = torch.zeros((4, k), device="cuda")

        def chain(solver):
            def run():
                if solver == "ddim":
                    eng.ddim_setup(betas, steps, 0.0, key=(0, 7))
                    eng.ddim_sample(init.clone(), collection=coll, metrics=mets)
                else:
                    eng.dpm_setup(betas, steps, int(solver[-1]), key=(0, 7))
                    eng.dpm_sample(init.clone(), collection=coll, metrics=mets)
            return run

        for s in SOLVERS:
            chain(s)()                                 # warm-up: module load, FiLM tables, graph capture, history
        t = {s: [] for s in SOLVERS}
        launches = {}
        for _ in range(args.repeats):
            for s in SOLVERS:
                dt, nl = timed(chain(s), eng)
                t[s].append(1e3 * dt / k)
                launches[s] = nl / k
        emit(dict(part="per_step", workload=name, n=n, steps=k,
                  **{f"{s}_ms_per_step": min(t[s]) for s in SOLVERS}, **{f"{s}_spread": t[s] for s in SOLVERS},
                  **{f"{s}_launches_per_step": launches[s] for s in SOLVERS}))
        del eng, coll, init
        torch.cuda.empty_cache()


TRAIN_FLAGS = """\
    --loss=ddpm
    --sampling=ddpm
    --schedule_type=linear
    --sigma_begin=1e-4
    --sigma_end=0.02
    --num_sigmas=1000
    --problem=vae
    --architecture=TransformerDDPM
    --num_layers=2
    --num_mlp_layers=2
    --data_shape=32,42
    --batch_size=64
    --learning_rate=1e-3
    --max_steps={steps}
    --snapshot_freq={steps}
    --nosnapshot_sampling
    --synthetic
    --synthetic_examples=8192
    --model_dir={run}
    """


def ode_error(args, emit):
    env = dict(os.environ, PYTHONPATH=ROOT)
    with tempfile.TemporaryDirectory() as tmp:
        cfg = os.path.join(tmp, "ddpm.cfg")
        run_dir = os.path.join(tmp, "run")
        with open(cfg, "w") as f:
            f.write(textwrap.dedent(TRAIN_FLAGS).format(steps=args.train_steps, run=run_dir))
        t0 = time.perf_counter()
        r = subprocess.run([sys.executable, "-m", "smd_b200.train_ncsn", f"--flagfile={cfg}"], capture_output=True,
                           text=True, env=env, cwd=ROOT)
        if r.returncode != 0:
            raise SystemExit(r.stderr[-3000:])
        emit(dict(part="train", steps=args.train_steps, seconds=time.perf_counter() - t0))

        from absl import flags
        from smd_b200 import ebm_utils, sample_ncsn
        from smd_b200 import jrandom as random
        flags.FLAGS([sys.argv[0], f"--flagfile={cfg}"])
        _, optimizer = sample_ncsn._restore(run_dir, (32, 42))
        model = optimizer.target
        betas = ebm_utils.create_noise_schedule(1e-4, 0.02, 1000, "linear")
        x_T = random.normal(random.PRNGKey(3), (1000, 32, 42))
        rng = random.PRNGKey(5)

        def solve(solver, k):
            if solver == "ddim":
                x, _, _ = ebm_utils.ddim_dynamics(rng, model, betas, x_T, None, None, None, steps=k, eta=0.0)
            else:
                x, _, _ = ebm_utils.dpm_solver_dynamics(rng, model, betas, x_T, None, None, None, steps=k,
                                                        order=int(solver[-1]))
            return x.double()

        for solver in SOLVERS:
            ref = solve(solver, 1000)
            for k in KS:
                x = solve(solver, k)
                emit(dict(part="ode_error", solver=solver, steps=k, reference_steps=1000,
                          rel_l2=float((x - ref).norm() / ref.norm())))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--chain_steps", type=int, default=100, help="steps timed per chain in the per-step part")
    ap.add_argument("--train_steps", type=int, default=400)
    ap.add_argument("--parts", default="per_step,ode_error")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dpm_bench needs a CUDA device")
    import __graft_entry__ as g
    g.build()
    from smd_b200 import ebm_utils
    betas = ebm_utils.create_noise_schedule(1e-4, 0.02, 1000, "linear")
    dev_card = card()
    lines = []

    def emit(rec):
        rec = dict(rec, card=dev_card)
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    parts = args.parts.split(",")
    if "per_step" in parts:
        per_step(args, betas, emit)
    if "ode_error" in parts:
        ode_error(args, emit)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
