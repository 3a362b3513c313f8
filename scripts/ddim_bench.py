"""DDIM (smd_ddim_sample) against the DDPM chain (smd_ddpm_sample): per-step cost, end-to-end time over the number of
steps, and how far K-step samples of a briefly trained model lie from its 1000-step DDPM samples.

    python scripts/ddim_bench.py [--repeats 3] [--train_steps 400] [--out ddim_bench.json]

1. Per step: both chains on the same engine and init at N = 1000 over a T = 1000 linear schedule (1e-4 .. 0.02),
   --chain_steps steps each, alternated --repeats times (the faster repeat is reported, with the spread).  Workloads:
   TransformerDDPM base (L6 H8, mlp 2048, C = 42) at S = 32 and S = 128, and DenseDDPM C = 512 (3 blocks, mlp 2048).
   Launches per step from smd_launch_count.
2. End to end: ebm_utils.ddim_dynamics at K in {10, 20, 50, 100, 1000} (uniform, eta = 0) and
   ebm_utils.diffusion_dynamics, TransformerDDPM base, S = 32, N = 1000 (table setup, chain, collection, metrics).
3. Sample quality: train_ncsn trains a TransformerDDPM (L2, 32 x 42) on --synthetic latents for --train_steps steps;
   sample_ncsn draws 1000 samples from it with --sampling=ddpm and with --sampling=ddim at each K (same seed, so the
   same initial draw).  metrics.latent_metrics scores every K-step set against the DDPM set and against the real set,
   in the de-normalised units sample_ncsn writes.
Prints one JSON line per measurement, with the card's name and power limit; --out collects them."""
from __future__ import annotations

import argparse
import json
import os
import pickle
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
KS = (10, 20, 50, 100, 1000)


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
    for name, (cfg, shape) in WORKLOADS.items():
        eng = Engine(ModelConfig(**cfg), max_batch=n)
        eng.set_params(eng.init_params(seed=1, perturb=0.02))
        init = random.normal(random.PRNGKey(3), (n,) + shape)
        coll = torch.zeros((41, n) + shape, device="cuda")
        mets = torch.zeros((4, 1000), device="cuda")
        steps = np.linspace(0, 999, k).round().astype(np.int32)

        def ddpm():
            eng.sampler_setup(betas, key=(0, 7))
            eng.sample(init.clone(), steps=k, collection=coll, metrics=mets)

        def ddim():
            eng.ddim_setup(betas, steps, 1.0, key=(0, 7))
            eng.ddim_sample(init.clone(), collection=coll, metrics=mets[:, :k].contiguous())

        ddpm()
        ddim()                                         # warm-up: module load, FiLM tables, graph capture
        t = {"ddpm": [], "ddim": []}
        launches = {}
        for _ in range(args.repeats):
            for key, fn in (("ddpm", ddpm), ("ddim", ddim)):
                dt, nl = timed(fn, eng)
                t[key].append(1e3 * dt / k)
                launches[key] = nl / k
        emit(dict(part="per_step", workload=name, n=n, steps=k, ddpm_ms_per_step=min(t["ddpm"]),
                  ddim_ms_per_step=min(t["ddim"]), ddpm_spread=t["ddpm"], ddim_spread=t["ddim"],
                  ddpm_launches_per_step=launches["ddpm"], ddim_launches_per_step=launches["ddim"]))
        del eng, coll, init
        torch.cuda.empty_cache()


def end_to_end(args, betas, emit):
    from smd_b200 import ebm_utils, nn
    from smd_b200 import jrandom as random
    n, shape = 1000, (32, 42)
    spec = nn.ModuleSpec("TransformerDDPM")
    _, arena = spec.init_by_shape(random.PRNGKey(1), [((n,) + shape, np.float32)])
    model = nn.Model(spec, arena)
    init = random.normal(random.PRNGKey(3), (n,) + shape)
    rng = random.PRNGKey(5)

    def run(k):
        if k is None:
            return lambda: ebm_utils.diffusion_dynamics(rng, model, betas, init, None, None, None)
        return lambda: ebm_utils.ddim_dynamics(rng, model, betas, init, None, None, None, steps=k)

    for k in (None,) + KS:
        run(k)()                                       # warm-up
    t = {k: [] for k in (None,) + KS}
    for _ in range(args.repeats):
        for k in (None,) + KS:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(k)()
            torch.cuda.synchronize()
            t[k].append(time.perf_counter() - t0)
    base = min(t[None])
    emit(dict(part="end_to_end", sampler="ddpm", steps=1000, n=n, seconds=base, spread=t[None]))
    for k in KS:
        emit(dict(part="end_to_end", sampler="ddim", steps=k, n=n, seconds=min(t[k]), spread=t[k],
                  speedup_vs_ddpm=base / min(t[k])))


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


def quality(args, emit):
    from smd_b200 import metrics
    env = dict(os.environ, PYTHONPATH=ROOT)
    with tempfile.TemporaryDirectory() as tmp:
        cfg = os.path.join(tmp, "ddpm.cfg")
        with open(cfg, "w") as f:
            f.write(textwrap.dedent(TRAIN_FLAGS).format(steps=args.train_steps, run=os.path.join(tmp, "run")))
        t0 = time.perf_counter()
        r = subprocess.run([sys.executable, "-m", "smd_b200.train_ncsn", f"--flagfile={cfg}"], capture_output=True,
                           text=True, env=env, cwd=ROOT)
        if r.returncode != 0:
            raise SystemExit(r.stderr[-3000:])
        emit(dict(part="train", steps=args.train_steps, seconds=time.perf_counter() - t0))
        sets = {}
        for k in (None,) + KS:
            name = "ddpm" if k is None else f"ddim{k}"
            extra = ["--sampling=ddpm"] if k is None else ["--sampling=ddim", f"--ddim_steps={k}"]
            r = subprocess.run([sys.executable, "-m", "smd_b200.sample_ncsn", f"--flagfile={cfg}", "--sample_size=1000",
                                f"--sampling_dir={name}", *extra], capture_output=True, text=True, env=env, cwd=ROOT)
            if r.returncode != 0:
                raise SystemExit(r.stderr[-3000:])
            out = os.path.join(tmp, "run", name, "ncsn")
            with open(os.path.join(out, "generated.pkl"), "rb") as f:
                sets[name] = np.asarray(pickle.load(f), np.float32)
            if k is None:
                with open(os.path.join(out, "real.pkl"), "rb") as f:
                    sets["real"] = np.asarray(pickle.load(f), np.float32)
        emit(dict(part="quality", samples="ddpm1000", vs_real=metrics.latent_metrics(sets["real"], sets["ddpm"])))
        for k in KS:
            s = sets[f"ddim{k}"]
            emit(dict(part="quality", samples=f"ddim{k}", eta=0.0, vs_ddpm1000=metrics.latent_metrics(sets["ddpm"], s),
                      vs_real=metrics.latent_metrics(sets["real"], s)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--chain_steps", type=int, default=100, help="steps timed per chain in the per-step part")
    ap.add_argument("--train_steps", type=int, default=400)
    ap.add_argument("--parts", default="per_step,end_to_end,quality")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ddim_bench needs a CUDA device")
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
    if "end_to_end" in parts:
        end_to_end(args, betas, emit)
    if "quality" in parts:
        quality(args, emit)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
