"""The DDIM encoder (smd_ddim_encode) against the DDIM chain (smd_ddim_sample): per-step cost, end-to-end
`sample_ncsn --interpolate` with the stochastic and the DDIM encoder, and the round-trip error decode(encode(x)).

    python scripts/ddim_encode_bench.py [--repeats 3] [--train_steps 400] [--out ddim_encode_bench.json]

1. Per step: both chains on the same engine and data at N = 1000 over a T = 1000 linear schedule (1e-4 .. 0.02),
   --chain_steps uniform levels each, after a warm-up call (FiLM table, graph capture), alternated --repeats times
   (the best repeat is reported, with the spread).  Workloads: TransformerDDPM base (L6 H8, mlp 2048, C = 42) at
   S = 32 and S = 128, and DenseDDPM C = 512 (3 blocks, mlp 2048).  Launches per step from smd_launch_count.
2. End to end: train_ncsn trains a TransformerDDPM (L2, 32 x 42) on --synthetic latents for --train_steps steps, as
   scripts/ddim_bench.py does.  On that checkpoint, `sample_ncsn --interpolate --sample_size=1000` runs with the
   stochastic encoder (--sampling=ddpm, 9 chains of 1000 steps) and with --interpolate_encoder=ddim at each K; the
   wall time of each process is reported.
3. Round trip: for each run of part 2, the error of the alpha = 0 interpolant against the starts and of the alpha = 1
   interpolant against the goals, from the written pickles (de-normalised units, the same for both encoders), and
   reconstruction.json (normalised units) for the DDIM runs.
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
    from smd_b200 import Engine, ModelConfig, ebm_utils
    n, k = 1000, args.chain_steps
    steps = ebm_utils.ddim_schedule(1000, k)
    for name, (cfg, shape) in WORKLOADS.items():
        eng = Engine(ModelConfig(**cfg), max_batch=n)
        eng.set_params(eng.init_params(seed=1, perturb=0.02))
        data = torch.from_numpy(np.random.default_rng(3).uniform(-1, 1, (n,) + shape).astype(np.float32)).cuda()
        x = data.clone()

        def encode():
            x.copy_(data)
            eng.ddim_encode_setup(betas, steps)
            eng.ddim_encode(x)

        def decode():
            x.copy_(data)
            eng.ddim_setup(betas, steps, 0.0, key=(0, 7))
            eng.ddim_sample(x)

        encode()
        decode()                                       # warm-up: module load, FiLM tables, graph capture
        t = {"encode": [], "ddim": []}
        launches = {}
        for _ in range(args.repeats):
            for key, fn in (("encode", encode), ("ddim", decode)):
                dt, nl = timed(fn, eng)
                t[key].append(1e3 * dt / k)
                launches[key] = nl / k
        emit(dict(part="per_step", workload=name, n=n, steps=k, encode_ms_per_step=min(t["encode"]),
                  ddim_ms_per_step=min(t["ddim"]), encode_spread=t["encode"], ddim_spread=t["ddim"],
                  encode_launches_per_step=launches["encode"], ddim_launches_per_step=launches["ddim"]))
        del eng, data, x
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


def _errors(gen, real):
    goals = np.roll(real, 1, axis=0)
    out = {}
    for name, got, want in (("start", gen[0], real), ("goal", gen[-1], goals)):
        d = np.asarray(got, np.float64) - np.asarray(want, np.float64)
        out[f"{name}_mse"] = float(np.mean(d * d))
        out[f"{name}_max_abs"] = float(np.max(np.abs(d)))
    return out


def interpolation(args, emit):
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
        for k in (None,) + KS:
            name = "stochastic" if k is None else f"ddim{k}"
            extra = (["--sampling=ddpm"] if k is None else
                     ["--sampling=ddim", "--interpolate_encoder=ddim", f"--ddim_steps={k}", "--ddim_eta=0"])
            t0 = time.perf_counter()
            r = subprocess.run([sys.executable, "-m", "smd_b200.sample_ncsn", f"--flagfile={cfg}", "--sample_size=1000",
                                "--interpolate", f"--sampling_dir={name}", *extra], capture_output=True, text=True,
                               env=env, cwd=ROOT)
            seconds = time.perf_counter() - t0
            if r.returncode != 0:
                raise SystemExit(r.stderr[-3000:])
            out = os.path.join(tmp, "run", name, "ncsn")
            with open(os.path.join(out, "generated.pkl"), "rb") as f:
                gen = np.asarray(pickle.load(f), np.float32)
            with open(os.path.join(out, "real.pkl"), "rb") as f:
                real = np.asarray(pickle.load(f), np.float32)
            rec = dict(part="interpolate", encoder="stochastic" if k is None else "ddim", steps=1000 if k is None else k,
                       n=1000, seconds=seconds, written_units=_errors(gen, real))
            if k is not None:
                with open(os.path.join(out, "reconstruction.json")) as f:
                    rec["normalised_units"] = json.load(f)
            emit(rec)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--chain_steps", type=int, default=100, help="steps timed per chain in the per-step part")
    ap.add_argument("--train_steps", type=int, default=400)
    ap.add_argument("--parts", default="per_step,interpolate")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ddim_encode_bench needs a CUDA device")
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
    if "interpolate" in parts:
        interpolation(args, emit)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
