"""Count the Hopper-specific SASS mnemonics per kernel of libpanfusion_b200.so (cuobjdump, no GPU needed):
wgmma.mma_async -> HGMMA, wgmma.fence / commit / wait -> WARPGROUP.*, TMA -> UTMALDG/UTMASTG/UBLKCP, mbarrier -> SYNCS.
Usage: python scripts/sass_evidence.py"""
import collections
import re
import subprocess
import sys
from pathlib import Path

LIB = Path(__file__).resolve().parent.parent / "panfusion_b200" / "lib" / "libpanfusion_b200.so"
PAT = re.compile(r"\b(HGMMA[A-Z0-9_.]*|WARPGROUP[A-Z0-9_.]*|UTMALDG[A-Z0-9_.]*|UTMASTG[A-Z0-9_.]*|UBLKCP[A-Z0-9_.]*|"
                 r"SYNCS[A-Z0-9_.]*|UTMAPF[A-Z0-9_.]*|UTMACMDFLUSH[A-Z0-9_.]*|MUFU\.EX2[A-Z0-9_.]*)")
out = subprocess.run(["cuobjdump", "-sass", str(LIB)], capture_output=True, text=True, check=True).stdout
kernels, cur = collections.OrderedDict(), None
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip().split("(")[0]
        kernels[cur] = collections.Counter()
        continue
    if cur:
        for op in PAT.findall(line):
            kernels[cur][op.split(".")[0] if not op.startswith("MUFU") else "MUFU.EX2"] += 1
print(f"# SASS evidence for {LIB.name} (sm_90a): Hopper tensor-core / TMA mnemonics per kernel")
for k, c in kernels.items():
    if any(n.startswith(("HGMMA", "UTMA", "UBLKCP")) for n in c):
        print(f"{k}\n    " + ", ".join(f"{n}={v}" for n, v in sorted(c.items())))
