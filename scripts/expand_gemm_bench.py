"""Times the trunk's three K = 128, N = 2048 GEMMs with their production epilogues -- FFN up (bias + tanh-GELU to bf16
with the bf16 pre-activation), its adjoint dX2 (x gelu'(pre-activation) to bf16) and the post dense (bias, fp32 out,
row-statistics partials) -- at 4096 tokens (the train step at batch 128) and 32 000 tokens (the sampler at 1000
samples), on the 128 x 128 route and on the route gemm_kind selects (gemm_bf16_wgmma_expand_kernel), alternating the
two in one process, and checks that every output of the pair is bit-identical.  The 128 x 128 route is reached through
the C ABI hook by handing A over MN-major ([K][tokens]), a layout the expand kernel does not take; its tiles,
epilogue and K loop are those the train step ran on that route.
Usage: python scripts/expand_gemm_bench.py [--iters N] [--rounds R]"""
import argparse
import ctypes
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from smd_b200 import lib as L  # noqa: E402

K, N = 128, 2048
OPS = ["ffn_up", "dx2", "post"]
# the outputs each kind runs without, besides the full production set
DROPS = {"ffn_up": [(), ("pre",)], "dx2": [()], "post": [(), ("stats",), ("bias", "stats")]}


def bytes_moved(op, M, drop=()):
    """HBM bytes the launch has to move: A, W, the outputs, and for dX2 the pre-activation it reads"""
    a, w = M * K * 2, K * N * 2
    out = {"ffn_up": (1 if "pre" in drop else 2) * M * N * 2, "dx2": 2 * M * N * 2,
           "post": M * N * 4 + (0 if "stats" in drop else M * N // 128 * 3 * 8)}[op]
    return a + w + out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    lib = L.load_library()
    stream = torch.cuda.current_stream()
    print(json.dumps({"device": torch.cuda.get_device_name()}))
    for M in (4096, 32000):
        for op in OPS:
            for drop in DROPS[op]:
                run_case(lib, stream, args, M, op, drop)


def run_case(lib, stream, args, M, op, drop):
    p = lambda t: None if t is None else t.data_ptr()
    gen = torch.Generator(device="cpu").manual_seed(M + len(op))
    X = (torch.randn(M, K, generator=gen) * 0.5).to(torch.bfloat16).cuda()
    Xt = X.t().contiguous()
    if op == "dx2":
        W = (torch.randn(N, K, generator=gen) * (0.5 / math.sqrt(K / 64))).to(torch.bfloat16).cuda()
        b_mn, bias = 0, None
        gg = torch.randn(M, N, generator=gen).to(torch.bfloat16).cuda()
    else:
        W = (torch.randn(K, N, generator=gen) * (0.5 / math.sqrt(K / 64))).to(torch.bfloat16).cuda()
        b_mn, bias, gg = 1, torch.randn(N, generator=gen).cuda(), None
    if "bias" in drop:
        bias = None
    outs = {}
    for route in ("128x128", "expand"):
        o = {}
        if op == "post":
            o["f32"] = torch.empty(M, N, device="cuda")
            if "stats" not in drop:
                o["stats"] = torch.zeros(M, 2, device="cuda")
                o["part"] = torch.empty(M, N // 128 * 3, 2, device="cuda")
        else:
            o["bf16"] = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
            if op == "ffn_up" and "pre" not in drop:
                o["pre"] = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
        outs[route] = o
    nslots = ctypes.c_int(0)

    def run(route):
        a, a_mn = (Xt, 1) if route == "128x128" else (X, 0)
        o = outs[route]
        L.check(lib.smd_gemm_bf16_epi(a.data_ptr(), W.data_ptr(), M, N, K, a_mn, b_mn, p(bias),
                                      1 if op == "ffn_up" else 0, p(o.get("f32")), p(o.get("bf16")),
                                      p(o.get("pre")), p(gg), p(o.get("stats")), p(o.get("part")),
                                      ctypes.byref(nslots), stream.cuda_stream))

    times = {"128x128": [], "expand": []}
    for route in times:
        for _ in range(10):
            run(route)
    for _ in range(args.rounds):
        for route in times:
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            for _ in range(args.iters):
                run(route)
            ev1.record()
            torch.cuda.synchronize()
            times[route].append(ev0.elapsed_time(ev1) * 1e3 / args.iters)
    same = all(torch.equal(outs["128x128"][k].view(torch.int16 if v.dtype == torch.bfloat16 else torch.int32),
                           v.view(torch.int16 if v.dtype == torch.bfloat16 else torch.int32))
               for k, v in outs["expand"].items() if k != "stats")
    old, new = min(times["128x128"]), min(times["expand"])
    moved = bytes_moved(op, M, drop)
    floor = moved / 3.35e12 * 1e6
    print(json.dumps({"op": op, "tokens": M, "without": list(drop), "us_128x128": round(old, 2),
                      "us_expand": round(new, 2), "speedup": round(old / new, 2), "hbm_floor_us": round(floor, 1),
                      "expand_TBps": round(moved / new * 1e-6, 2),
                      "spread_us": {k: [round(t, 2) for t in v] for k, v in times.items()},
                      "bitwise_equal": bool(same)}))

if __name__ == "__main__":
    main()
