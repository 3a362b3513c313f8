"""Times the trunk GEMMs with N = 128 output columns (base config: 128-wide trunk, mlp_dims 2048) at 4096 tokens (the
train step at batch 128) and 32 000 tokens (the sampler's unfused trunk at S = 128 / TransformerMDN), on the 128 x 128
route and on the route gemm_kind selects for the op (the swapped-operand gemm_bf16_wgmma_swap_kernel, except for the
fp32 kinds once their 128 x 128 tiles take more than one round), in one process, and checks that each pair of fp32
outputs agrees.  The 128 x 128 route is reached through the C ABI hook by handing over the token operand
MN-major ([K][tokens]), a layout the swapped route does not take; its tiles, epilogue and K loop are the train step's.
Usage: python scripts/trunk_gemm_bench.py [--iters N]"""
import argparse
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from smd_b200 import lib as L  # noqa: E402

N = 128
# (name, K, weight read MN-major, LayerNorm epilogue): forward ops read the (in, out) weight, dX ops the plain one
OPS = [("op_o (attention out-projection + LN)", 128, 1, True),
       ("op_ffn2 (FFN down + LN)", 2048, 1, True),
       ("dXpost (post dense dX)", 2048, 0, False),
       ("dX1 (FFN up dX)", 2048, 0, False),
       ("dXo (out-projection dX)", 128, 0, False),
       ("dXqkv (QKV dX)", 384, 0, False)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    lib = L.load_library()
    stream = torch.cuda.current_stream()
    print(json.dumps({"device": torch.cuda.get_device_name()}))
    for M in (4096, 32000):
        for name, K, b_mn, ln in OPS:
            gen = torch.Generator(device="cpu").manual_seed(K + M)
            X = (torch.randn(M, K, generator=gen) * 0.5).to(torch.bfloat16).cuda()
            Xt = X.t().contiguous()
            Wt = (torch.randn(N, K, generator=gen) * (0.5 / math.sqrt(K / 64))).to(torch.bfloat16)
            W = (Wt.t().contiguous() if b_mn else Wt).cuda()
            bias = torch.randn(N, generator=gen).cuda() if ln else None
            res = torch.randn(M, N, generator=gen).cuda() if ln else None
            gam = torch.ones(N, device="cuda") if ln else None
            bet = torch.zeros(N, device="cuda") if ln else None
            outs = {}
            p = lambda t: None if t is None else t.data_ptr()

            def run(a, a_mn, o32, o16):
                L.check(lib.smd_gemm_bf16(a.data_ptr(), W.data_ptr(), M, N, K, a_mn, b_mn, 0, 1, p(bias), p(res), 0,
                                          o32.data_ptr(), p(o16), None, p(gam), p(bet), stream.cuda_stream))

            times = {}
            for route, a, a_mn in (("128x128", Xt, 1), ("swap", X, 0)):
                o32 = torch.empty(M, N, device="cuda")
                o16 = torch.empty(M, N, dtype=torch.bfloat16, device="cuda") if ln else None
                for _ in range(10):
                    run(a, a_mn, o32, o16)
                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ev0.record()
                for _ in range(args.iters):
                    run(a, a_mn, o32, o16)
                ev1.record()
                torch.cuda.synchronize()
                times[route] = ev0.elapsed_time(ev1) * 1e3 / args.iters
                outs[route] = o32
            rel = float((outs["swap"].double() - outs["128x128"].double()).norm() / outs["128x128"].double().norm())
            flop = 2.0 * M * N * K
            print(json.dumps({"op": name, "tokens": M, "K": K, "us_128x128": round(times["128x128"], 2),
                              "us_swap": round(times["swap"], 2), "speedup": round(times["128x128"] / times["swap"], 2),
                              "tflops_swap": round(flop / times["swap"] * 1e-6, 1), "rel_l2": f"{rel:.2e}",
                              "agree": rel <= 1e-5}))


if __name__ == "__main__":
    main()
