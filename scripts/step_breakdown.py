"""Phase breakdown of one train step from a CUPTI timeline written by scripts/timeline.py (eager or graph replay):
prologue, trunk forward, tail forward, tail backward, trunk backward, optimizer.
Phases are cut on the main (dX) stream at well-defined kernels; the other two streams overlap and are reported as
busy time.  Usage: python scripts/step_breakdown.py <timeline.json written by scripts/timeline.py>"""
import json
import sys
from collections import defaultdict


def main():
    rows = json.load(open(sys.argv[1]))
    # one step = from a q_sample_kernel to the next one
    starts = [i for i, r in enumerate(rows) if r["name"].startswith("smd::q_sample_kernel") or "q_sample_kernel" in r["name"]]
    if len(starts) < 2:
        raise SystemExit("need at least two steps in the timeline")
    a, b = starts[-2], starts[-1]
    step = rows[a:b]
    t0 = step[0]["ts"]
    end = lambda r: r["ts"] + r["dur"] - t0

    def first(pred, lo=0):
        for i in range(lo, len(step)):
            if pred(step[i]):
                return i
        return None

    i_embed = first(lambda r: "embed" in r["name"] and "bwd" not in r["name"])
    i_post = first(lambda r: "ln_film_act_kernel" in r["name"])                               # first tail kernel
    i_loss = first(lambda r: "ddpm_loss_bwd_kernel" in r["name"])
    i_trunk_bwd = first(lambda r: "ln128_bwd_kernel" in r["name"], i_loss)                    # post_ln backward
    i_embed_bwd = first(lambda r: "embed_bwd_kernel" in r["name"])
    i_sumsq = first(lambda r: "sumsq_kernel" in r["name"])
    cuts = [("prologue (memsets, q_sample, embed)", 0.0, end(step[i_embed])),
            ("trunk forward", end(step[i_embed]), step[i_post]["ts"] - t0),
            ("tail forward + loss", step[i_post]["ts"] - t0, end(step[i_loss])),
            ("tail backward", end(step[i_loss]), step[i_trunk_bwd]["ts"] - t0),
            ("trunk backward", step[i_trunk_bwd]["ts"] - t0, end(step[i_embed_bwd])),
            ("remaining weight-gradient GEMMs", end(step[i_embed_bwd]), step[i_sumsq]["ts"] - t0),
            ("clip + Adam + repack", step[i_sumsq]["ts"] - t0, max(end(r) for r in step))]
    busy = defaultdict(float)
    for r in step:
        busy[r["stream"]] += r["dur"]
    total = max(end(r) for r in step)
    out = {"step_us": round(total, 1), "launches": len(step),
           "phases_us": {n: round(hi - lo, 1) for n, lo, hi in cuts},
           "stream_busy_us": {str(k): round(v, 1) for k, v in busy.items()}}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
