"""Opcode histogram of every compiled translation unit (cuobjdump -sass of whisper-burn_b200/build/*.o): which kernels
really contain wgmma / TMA / bulk-copy instructions.  python scripts/sass_opcodes.py"""
import collections
import re
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
KEY = ["HGMMA", "WARPGROUP", "UTMALDG", "UTMASTG", "UBLKCP", "SYNCS", "HMMA", "LDSM", "LDGSTS",
       "FFMA", "HFMA2", "MUFU", "UCGABAR_ARV", "BAR", "ATOMS", "RED", "LDG", "LDS", "STS", "SHFL"]
print("# SASS opcode counts per translation unit (sm_90a), from cuobjdump -sass; wgmma.mma_async = HGMMA, wgmma fence / wait = WARPGROUP,")
print("# TMA tensor load = UTMALDG, 1-D bulk copy = UBLKCP, mbarrier = SYNCS, mma.sync = HMMA, ldmatrix = LDSM")
print(f"{'unit':16s} " + " ".join(f"{k:>8s}" for k in KEY))
for obj in sorted((ROOT / "whisper-burn_b200" / "build").glob("*.o")):
    out = subprocess.run(["cuobjdump", "-sass", str(obj)], capture_output=True, text=True).stdout
    ops = collections.Counter()
    for m in re.finditer(r"^\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", out, flags=re.M):
        ops[m.group(1)] += 1
    if not ops:
        continue
    row = [sum(v for k2, v in ops.items() if k2 == k or k2.startswith(k + ".") or (k in ("BAR", "RED", "LDG", "LDS", "STS") and k2 == k)) for k in KEY]
    print(f"{obj.stem:16s} " + " ".join(f"{v:8d}" for v in row))
