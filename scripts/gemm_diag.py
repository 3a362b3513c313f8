"""Diagnostic sweep of the wgmma GEMM on a GPU: every case runs in its own process (a trap or fault cannot
poison the next) and prints error structure, not just pass/fail.  Usage: python scripts/gemm_diag.py"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def one(cfg):
    import torch
    from smd_b200 import lib as L
    lib = L.load_library()
    M, N, K = cfg["M"], cfg["N"], cfg["K"]
    g = torch.Generator().manual_seed(1)
    A = (torch.randn(M, K, generator=g)).to(torch.bfloat16)
    B = (torch.randn(N, K, generator=g)).to(torch.bfloat16)
    if cfg.get("kmask") is not None:          # keep only one 16-wide k slice non-zero
        j = cfg["kmask"]
        m = torch.zeros(K)
        m[16 * j:16 * j + 16] = 1
        A = (A.float() * m).to(torch.bfloat16)
    ref = A.float() @ B.float().t()
    Ad = (A.t().contiguous() if cfg["a_mn"] else A).cuda()
    Bd = (B.t().contiguous() if cfg["b_mn"] else B).cuda()
    out = torch.full((M, N), float("nan"), device="cuda")
    rc = lib.smd_gemm_bf16(Ad.data_ptr(), Bd.data_ptr(), M, N, K, cfg["a_mn"], cfg["b_mn"], cfg.get("BN", 0),
                           cfg["cg"], None, None, 0, out.data_ptr(), None, None, None, None,
                           torch.cuda.current_stream().cuda_stream)
    if rc != 0:
        print("  rc", rc, lib.smd_last_error().decode())
        return
    torch.cuda.synchronize()
    got = out.cpu()
    nan = int(torch.isnan(got).sum())
    d = (torch.nan_to_num(got) - ref)
    rel = float(d.norm() / ref.norm())
    print(f"  rel-L2 {rel:.3e} max-abs {float(d.abs().max()):.3e} nan {nan}/{got.numel()}")
    if rel > 1e-4:
        bad = d.abs() > 1e-2 * (1 + ref.abs())
        print("  bad frac", float(bad.float().mean()))
        rb = bad.float().reshape(M // 8 if M % 8 == 0 else -1, 8, N).mean((0, 2)) if M % 8 == 0 else None
        print("  bad by row%8", None if rb is None else [round(float(v), 3) for v in rb])
        cbk = 16
        cb = bad.float().reshape(M, N // cbk, cbk).mean((0, 2)) if N % cbk == 0 else None
        print("  bad by col block16 (first 16)", None if cb is None else [round(float(v), 2) for v in cb[:16]])
        rb32 = bad.float().reshape(M // 32, 32, N).mean((1, 2)) if M % 32 == 0 else None
        print("  bad by row block32 (first 16)", None if rb32 is None else [round(float(v), 2) for v in rb32[:16]])
        print("  got[0,:6]", [round(float(v), 3) for v in got[0, :6]], "ref", [round(float(v), 3) for v in ref[0, :6]])
        print("  got[1,:6]", [round(float(v), 3) for v in got[1, :6]], "ref", [round(float(v), 3) for v in ref[1, :6]])
        # is it a scaled / partial-K result?
        ratio = (torch.nan_to_num(got) * ref).sum() / (ref * ref).sum()
        print("  projection got.ref/ref.ref", float(ratio))


CASES = []
for cg in (1, 2):
    CASES += [dict(M=128 * cg, N=64, K=16 * 4, a_mn=0, b_mn=0, cg=cg, BN=64, kmask=0),
              dict(M=128 * cg, N=64, K=64, a_mn=0, b_mn=0, cg=cg, BN=64, kmask=1),
              dict(M=128 * cg, N=64, K=64, a_mn=0, b_mn=0, cg=cg, BN=64),
              dict(M=128 * cg, N=256, K=64, a_mn=0, b_mn=0, cg=cg),
              dict(M=256, N=256, K=256, a_mn=0, b_mn=0, cg=cg),
              dict(M=1024, N=2048, K=2048, a_mn=0, b_mn=0, cg=cg),
              dict(M=128 * cg, N=128, K=64, a_mn=1, b_mn=1, cg=cg, BN=128, kmask=0),
              dict(M=128 * cg, N=128, K=64, a_mn=1, b_mn=1, cg=cg, BN=128, kmask=2),
              dict(M=128 * cg, N=128, K=64, a_mn=1, b_mn=1, cg=cg, BN=128),
              dict(M=256, N=256, K=256, a_mn=1, b_mn=0, cg=cg),
              dict(M=256, N=256, K=256, a_mn=0, b_mn=1, cg=cg),
              dict(M=2048, N=2048, K=4096, a_mn=1, b_mn=1, cg=cg)]

if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--one":
        one(json.loads(sys.argv[2]))
        sys.exit(0)
    for c in CASES:
        print("case", json.dumps(c), flush=True)
        try:
            r = subprocess.run([sys.executable, __file__, "--one", json.dumps(c)], capture_output=True, text=True,
                               timeout=180)
            print(r.stdout, end="")
            if r.returncode != 0:
                print("  EXIT", r.returncode, r.stderr[-600:])
        except subprocess.TimeoutExpired:
            print("  TIMEOUT")
