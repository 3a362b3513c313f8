"""Times the res-block GEMM shapes alone (CUDA events, L2 flushed before every launch, like bench.py's dominant-GEMM
figure), each with the epilogue the train step launches it with:

  res-a  bias + bf16 + row stats            (kEpiAct)     A K-major activations, B the (in, out) weight MN-major
  res-b  bias + residual + f32 + row stats  (kEpiF32Res)  same operands
  dX     bf16 only                          (kEpiAct)     both K-major
  dW     f32                                (kEpiF32)     both MN-major, the reduction runs over the tokens
  dom    bias + f32 + row stats             (kEpiF32)     bench.py's dominant GEMM, both K-major

Every case has a no-output twin (`"epi": "none"`): the same operands with every epilogue pointer null, so the same
mainloop and accumulator staging run without any epilogue traffic.  The gap between a case and its twin is the time
the tensor cores spend waiting on the epilogue.  torch.matmul (cuBLAS) on the same bf16 operands is the yardstick of
what this card reaches on the shape.

Each result line is JSON; `sha` is a hash of the GEMM's fp32 / bf16 outputs (not of the row statistics, whose atomics
make the last bits order dependent), so two libraries can be compared bit for bit.

  python scripts/gemm_l2_probe.py [--root TREE] [--out FILE] [--iters N] [--tokens 4096 32000] [--bn 128 256]

--bn 256 asks for the wide layout (128 x 256 tiles), which every case here gets; its `sha` must equal the BN = 128
line's of the same case.

--root imports smd_b200 (and its libsmd.so) from another checkout of this repository, e.g. a build of the parent
commit, so that two builds are timed by the same script.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import subprocess
import sys

import torch


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=10).stdout.strip().splitlines()
        return out[0] if out else None
    except Exception:
        return None


# name -> (a_mn, b_mn, outputs); outputs among bias, res, f32, bf16, stats
CASES = {
    "res-a": (0, 1, ("bias", "bf16", "stats")),
    "res-b": (0, 1, ("bias", "res", "f32", "stats")),
    "dX": (0, 0, ("bf16",)),
    "dW": (1, 1, ("f32",)),
    "dom": (0, 0, ("bias", "f32", "stats")),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--tokens", type=int, nargs="+", default=[4096, 32000])
    ap.add_argument("--bn", type=int, nargs="+", default=[128, 256])
    ap.add_argument("--cases", nargs="+", default=list(CASES))
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    from smd_b200 import lib as L
    lib = L.load_library()
    if not torch.cuda.is_available():
        raise SystemExit("gemm_l2_probe.py needs a CUDA device")
    dev = torch.device("cuda")
    st = torch.cuda.current_stream().cuda_stream
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    lines = [{"gpu": gpu_info(), "root": os.path.abspath(args.root)}]
    print(json.dumps(lines[0]), flush=True)

    def timed(fn):
        total = 0.0
        for i in range(args.iters + 3):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            if i >= 3:
                total += e0.elapsed_time(e1)
        return total / args.iters * 1e3  # us

    gen = torch.Generator(device=dev)
    p = lambda t: None if t is None else t.data_ptr()
    for tokens in args.tokens:
        for name in args.cases:
            a_mn, b_mn, outs = CASES[name]
            # dW reduces over the tokens: [2048 in][tokens] x [tokens][2048 out]
            M, N, K = (2048, 2048, tokens) if name == "dW" else (tokens, 2048, 2048)
            gen.manual_seed(M * 7 + N + K + a_mn)
            A = torch.randn(*((K, M) if a_mn else (M, K)), device=dev, generator=gen).to(torch.bfloat16)
            B = torch.randn(*((K, N) if b_mn else (N, K)), device=dev, generator=gen).to(torch.bfloat16)
            bias = torch.randn(N, device=dev, generator=gen) if "bias" in outs else None
            res = torch.randn(M, N, device=dev, generator=gen) if "res" in outs else None
            o32 = torch.empty(M, N, device=dev) if "f32" in outs else None
            o16 = torch.empty(M, N, device=dev, dtype=torch.bfloat16) if "bf16" in outs else None
            stats = torch.zeros(M, 2, device=dev) if "stats" in outs else None
            flop = 2.0 * M * N * K
            for BN in args.bn:
                for epi in ("full", "none"):
                    full = epi == "full"
                    ptrs = [p(t) if full else None for t in (bias, res, o32, o16, stats)]
                    call = lambda: L.check(lib.smd_gemm_bf16(A.data_ptr(), B.data_ptr(), M, N, K, a_mn, b_mn, BN, 1,
                                                             ptrs[0], ptrs[1], 0, ptrs[2], ptrs[3], ptrs[4], None, None,
                                                             st))
                    us = timed(call)
                    rec = {"case": name, "epi": epi, "M": M, "N": N, "K": K, "a_mn": a_mn, "b_mn": b_mn, "BN": BN,
                           "us": us, "tflops": flop / us / 1e6}
                    if full:
                        if stats is not None:
                            stats.zero_()
                        call()
                        torch.cuda.synchronize()
                        h = hashlib.sha256()
                        for t in (o32, o16):
                            if t is not None:
                                h.update(t.view(torch.uint8).cpu().numpy().tobytes())
                        rec["sha"] = h.hexdigest()[:16]
                        if stats is not None:
                            rec["stats_sum"] = [float(v) for v in stats.double().sum(0).cpu()]
                    print(json.dumps(rec), flush=True)
                    lines.append(rec)
            At = A.t() if a_mn else A          # [M][K] view
            Bt = B if b_mn else B.t()          # [K][N] view
            us = timed(lambda: torch.matmul(At, Bt))
            rec = {"case": name, "M": M, "N": N, "K": K, "impl": "torch.matmul (cuBLAS, bf16 out)", "us": us,
                   "tflops": flop / us / 1e6}
            print(json.dumps(rec), flush=True)
            lines.append(rec)
            del A, B, bias, res, o32, o16, stats
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
