"""Times the res-block GEMM shapes alone (CUDA events, L2 flushed before every launch, like bench.py's dominant-GEMM
figure) to show whether the kernel is bound by operand traffic from L2 or by the tensor cores:

  * BN = 128 and BN = 64: BN = 64 moves about 1.5x the operand bytes from L2 into the SMs.  (The kernel issues
    m64n128 wgmma whatever BN is, so BN = 64 also issues twice the tensor-core instructions: the comparison bounds
    the cost of the operand traffic rather than isolating it);
  * torch.matmul (cuBLAS) on the same bf16 operands, as the yardstick of what this card reaches on the shape.

Each result line is JSON; `sha` is a hash of the GEMM's fp32 output, so two libraries can be compared bit for bit.

  python scripts/gemm_l2_probe.py [--root TREE] [--out FILE] [--iters N]

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=20)
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

    # (name, M, N, K, a_mn, b_mn, epilogue): the res-block GEMMs of the train step / sampler at batch 128 (4096 tokens)
    # and 1000 samples (32000 tokens).  fwd: A K-major activations, B the (in, out) weight read MN-major; dX: both
    # K-major; dW: both MN-major (reduction over tokens).
    cases = [
        ("fwd", 4096, 2048, 2048, 0, 1, "bias_f32_stats"),
        ("dX", 4096, 2048, 2048, 0, 0, "bias_f32_stats"),
        ("dW", 2048, 2048, 4096, 1, 1, "f32"),
        ("fwd", 32000, 2048, 2048, 0, 1, "bias_f32_stats"),
        ("dX", 32000, 2048, 2048, 0, 0, "bias_f32_stats"),
    ]
    gen = torch.Generator(device=dev)
    for name, M, N, K, a_mn, b_mn, kind in cases:
        gen.manual_seed(M * 7 + N + K + a_mn)
        A = torch.randn(*((K, M) if a_mn else (M, K)), device=dev, generator=gen).to(torch.bfloat16)
        B = torch.randn(*((K, N) if b_mn else (N, K)), device=dev, generator=gen).to(torch.bfloat16)
        bias = torch.randn(N, device=dev, generator=gen) if kind != "f32" else None
        out = torch.empty(M, N, device=dev)
        stats = torch.zeros(M, 2, device=dev) if kind != "f32" else None
        p = lambda t: None if t is None else t.data_ptr()
        flop = 2.0 * M * N * K

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

        for BN in (128, 64):
            call = lambda: L.check(lib.smd_gemm_bf16(A.data_ptr(), B.data_ptr(), M, N, K, a_mn, b_mn, BN, 1, p(bias),
                                                     None, 0, out.data_ptr(), None, p(stats), None, None, st))
            us = timed(call)
            if stats is not None:
                stats.zero_()
            call()
            torch.cuda.synchronize()
            sha = hashlib.sha256(out.cpu().numpy().tobytes()).hexdigest()[:16]
            rec = {"case": name, "M": M, "N": N, "K": K, "a_mn": a_mn, "b_mn": b_mn, "BN": BN, "us": us,
                   "tflops": flop / us / 1e6, "sha": sha}
            print(json.dumps(rec), flush=True)
            lines.append(rec)
        At = A.t() if a_mn else A          # [M][K] view
        Bt = B if b_mn else B.t()          # [K][N] view
        us = timed(lambda: torch.matmul(At, Bt))
        rec = {"case": name, "M": M, "N": N, "K": K, "impl": "torch.matmul (cuBLAS, bf16 out)", "us": us,
               "tflops": flop / us / 1e6}
        print(json.dumps(rec), flush=True)
        lines.append(rec)
        del A, B, out
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
