"""Per-kernel SASS mnemonic counts of libsmd.so (cuobjdump -sass): the evidence that the hot kernels use wgmma (HGMMA),
TMA (UTMALDG), mbarriers (SYNCS), mma.sync (HMMA), programmatic dependent launch and per-warpgroup register budgets
(USETMAXREG), and which of them touch local memory (STL / LDL: register spills).
Usage: python scripts/sass_mnemonics.py"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "symbolic-music-diffusion_b200", "libsmd.so")
KEYS = ["HGMMA", "HGMMA.64x256x16", "HGMMA.64x32x16", "UTMALDG", "UTMASTG", "SYNCS", "HMMA", "MUFU.TANH", "LDGSTS", "UBLKCP", "ACQBULK", "RED", "ATOM",
        "USETMAXREG", "STL", "LDL"]


def main():
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    names = {}
    cur = None
    counts = collections.defaultdict(collections.Counter)
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            # the same template instantiation is emitted by several translation units: count the first copy only
            cur = m.group(1) if m.group(1) not in counts else None
            if cur is not None:
                counts[cur]["_seen"] = 1
            continue
        if cur is None:
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
        if not m:
            continue
        op = m.group(1)
        if op.startswith("HGMMA"):   # the mnemonic match stops at the shape's lower-case x: read the whole token
            op = line[m.start(1):].split()[0]
        for k in KEYS:
            if op == k or op.startswith(k + ".") or (k == "MUFU.TANH" and op.startswith("MUFU.TANH")):
                counts[cur][k] += 1
    dem = subprocess.run(["c++filt"] + list(counts.keys()), capture_output=True, text=True).stdout.splitlines()
    for mangled, d in zip(list(counts.keys()), dem):
        d = re.sub(r"^void ", "", d)
        d = re.sub(r"\(.*$", "", d).replace("smd::", "")
        names[mangled] = d
    print("# SASS mnemonics per kernel (cuobjdump -sass libsmd.so, sm_90a): wgmma = HGMMA;")
    print("# TMA = UTMALDG; mbarrier = SYNCS; mma.sync = HMMA;")
    print("# cp.async = LDGSTS; programmatic dependent launch = ACQBULK; setmaxnreg = USETMAXREG; spills = STL / LDL")
    seen = set()
    for mangled in sorted(counts, key=lambda k: names[k]):
        n = names[mangled]
        if n in seen:
            continue
        seen.add(n)
        c = counts[mangled]
        if not any(c[k] for k in KEYS):
            continue
        print(f"{n:72s} " + "  ".join(f"{k}={c[k]}" for k in KEYS if c[k]))


if __name__ == "__main__":
    main()
