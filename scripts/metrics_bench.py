"""Times the latent-space metrics: smd_latent_stats on its own and metrics.latent_metrics end to end (stats, n x m
fp64 singular values, host combination) at n = m in {1000, 3000} and d in {1344, 16384, 65536} (32 x 42 sliced mel
latents, 32 x 512 unsliced, 128 x 512 unsliced), and the host route of metrics.py (scipy sqrtm, O(d^3)) where its
d x d covariances fit: d = 1344 only.  Inputs are uniform in [-1, 1] with a shifted, scaled second set.  Prints one
JSON line with the card's name and power limit read in the same run.

    python scripts/metrics_bench.py [--repeats 5] [--no-cpu]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _time(fn, repeats):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(repeats):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / repeats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--no-cpu", action="store_true")
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from smd_b200 import lib as L, metrics
    lib = L.load_library()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    out = {"card": card, "runs": []}
    gen = torch.Generator(device="cuda").manual_seed(0)
    for n in (1000, 3000):
        for d in (1344, 16384, 65536):
            x = torch.rand((n, d), device="cuda", generator=gen) * 2 - 1
            y = 0.8 * (torch.rand((n, d), device="cuda", generator=gen) * 2 - 1) + 0.1
            ws = torch.empty(lib.smd_latent_stats_workspace_bytes(n, n, d), dtype=torch.uint8, device="cuda")
            stats = torch.empty(9, dtype=torch.float64, device="cuda")
            cross = torch.empty((n, n), dtype=torch.float32, device="cuda")
            st = torch.cuda.current_stream().cuda_stream

            def call():
                L.check(lib.smd_latent_stats(x.data_ptr(), n, y.data_ptr(), n, d, 1.0, 2, 1.0, 0.0, ws.data_ptr(),
                                             ws.numel(), stats.data_ptr(), cross.data_ptr(), st))

            rows = (2 * n + 2 + 127) // 128 * 128
            gemm_flop = 3 * 2 * rows * rows * ((d + 63) // 64 * 64)     # the three bf16 passes of the Gram product
            stats_ms = _time(call, args.repeats)
            metrics.latent_metrics(x, y)                                # warm-up: the solver's first call sets up
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.repeats):
                gpu = metrics.latent_metrics(x, y)
            torch.cuda.synchronize()
            e2e_ms = (time.perf_counter() - t0) * 1e3 / args.repeats
            run = {"n": n, "m": n, "d": d, "workspace_bytes": ws.numel(), "gram_gemm_tflop": gemm_flop / 1e12,
                   "latent_stats_ms": stats_ms, "latent_stats_tflops": gemm_flop / stats_ms / 1e9,
                   "latent_metrics_ms": e2e_ms, "gpu": gpu}
            if d == 1344 and not args.no_cpu:
                xh, yh = x.double().cpu().numpy(), y.double().cpu().numpy()
                t0 = time.perf_counter()
                cpu = {"frechet_distance": metrics.frechet_distance(xh, yh), "mmd_rbf": metrics.mmd_rbf(xh, yh),
                       "mmd_polynomial": metrics.mmd_polynomial(xh, yh)}
                run["cpu_metrics_ms"] = (time.perf_counter() - t0) * 1e3
                run["cpu"] = cpu
            out["runs"].append(run)
            print(json.dumps(run), file=sys.stderr, flush=True)
            del x, y, ws, cross
            torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
