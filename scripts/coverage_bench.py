"""Times one smd_latent_coverage call (improved precision / recall, realism, PRD and NDB histograms from one Gram
product) with device events at n = m in {1000, 3000, 8192} and d in {1344, 16384} (32 x 42 sliced mel latents and 32 x
512 unsliced), with the defaults of metrics.py (k = 3; PRD 20 clusters x 10 runs; NDB 50 bins; 10 restarts; at most
300 Lloyd iterations).  Reports the Lloyd iterations the fits ran (the most of any restart) and the Gram bytes one
iteration reads (the S(p, C) pass reads the fit's N x N block of G once per fit), and the host functions of
metrics.py where they finish (d = 1344, n = 1000).  Inputs are uniform in [-1, 1] with a shifted, scaled second set.
Prints one JSON line with the card's name and power limit read in the same run.

    python scripts/coverage_bench.py [--repeats 2] [--no-cpu] [--max-n 8192]
"""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--max-n", type=int, default=8192)
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from smd_b200 import metrics
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    cfg = metrics.COVERAGE_DEFAULTS
    out = {"card": card, "config": cfg, "runs": []}
    gen = torch.Generator(device="cuda").manual_seed(0)
    metrics.latent_coverage(torch.rand((64, 64), device="cuda"), torch.rand((64, 64), device="cuda"))   # module load
    torch.cuda.synchronize()
    for n in (1000, 3000, 8192):
        if n > args.max_n:
            continue
        for d in (1344, 16384):
            x = torch.rand((n, d), device="cuda", generator=gen) * 2 - 1
            y = 0.8 * (torch.rand((n, d), device="cuda", generator=gen) * 2 - 1) + 0.1
            times = []
            for _ in range(args.repeats):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                counts, realism, prd_hist, ndb_hist, iters = metrics.latent_coverage(x, y)
                b.record()
                torch.cuda.synchronize()
                times.append(a.elapsed_time(b))
            it = iters.cpu().tolist()
            f_prd, f_ndb = cfg["prd_runs"] * cfg["restarts"], cfg["restarts"]
            run = {"n": n, "m": n, "d": d, "coverage_ms": times, "lloyd_iterations": {"prd": it[0], "ndb": it[1]},
                   "gram_bytes_per_iteration": {"prd": f_prd * (2 * n) ** 2 * 4, "ndb": f_ndb * n ** 2 * 4},
                   "gpu": metrics.combine_coverage(counts.cpu().numpy(), realism.cpu().numpy(),
                                                   prd_hist.cpu().numpy(), ndb_hist.cpu().numpy(), n, n)}
            if d == 1344 and n == 1000 and not args.no_cpu:
                xh, yh = x.double().cpu().numpy(), y.double().cpu().numpy()
                t0 = time.perf_counter()
                recall, precision = metrics.prd_f_beta_score(metrics.precision_recall_distribution(xh, yh))
                ip, ir = metrics.precision_recall(xh, yh)
                cpu = {"precision": precision, "recall": recall, "improved_precision": ip, "improved_recall": ir,
                       "ipr_realism": float(np.mean(metrics.realism_scores(xh, yh))), "ndb": metrics.ndb_score(xh, yh)}
                run["cpu_ms"] = (time.perf_counter() - t0) * 1e3
                run["cpu"] = cpu
            out["runs"].append(run)
            print(json.dumps(run), file=sys.stderr, flush=True)
            del x, y
            torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
