"""Static SASS instruction counts of the kernels on the measured path (cuobjdump needs no GPU).

    python tools/dev/sass_mnemonics.py > profiles/r02_sass_mnemonics.txt
"""
import collections
import re
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
LIB = ROOT / "gaussian_splatting_b200" / "libgsr_b200.so"
KEEP = ("12k_render_fwdILb1EE", "12k_render_bwdILb1EE", "12k_render_fwdILb0EE", "12k_render_bwdILb0EE",
        "k_preprocess_fwdILi16ELb1", "k_preprocess_bwdILi16ELb1", "k_emit_pairs_fused", "k_tile_ranges",
        "k_camera_centre", "k_adamILb0", "k_adamILb1", "k_densify_apply", "k_densify_accumulate")
SHOW = ("FFMA", "FMUL", "FADD", "UBLKCP", "LDGSTS", "SYNCS", "ARRIVES", "REDG.F32x4", "REDG", "ATOMG", "ATOMS", "BAR",
        "MUFU", "SHFL", "REDUX", "F2F", "DADD", "DMUL", "DFMA")

text = subprocess.run(["cuobjdump", "-sass", str(LIB)], check=True, capture_output=True, text=True).stdout
cur, counts = None, collections.OrderedDict()
for line in text.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = m.group(1)
        counts[cur] = collections.Counter()
        continue
    m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.x]+)", line)
    if m and cur:
        op = m.group(1)
        counts[cur][op.split(".")[0]] += 1
        counts[cur]["total"] += 1
        if op.startswith("REDG") and "F32x4" in op:
            counts[cur]["REDG.F32x4"] += 1

print("cuobjdump -sass gaussian_splatting_b200/libgsr_b200.so — static instruction counts of the kernels on the measured path")
print("(UBLKCP = cp.async.bulk 1-D TMA copy, LDGSTS = cp.async, SYNCS / ARRIVES = mbarrier,")
print(" REDG.F32x4 = red.global.add.v4.f32; ILb1EE = with contribution masks, ILb0EE = without)\n")
for name, c in counts.items():
    if not any(k in name for k in KEEP):
        continue
    cells = "  ".join(f"{k}={c[k]}" for k in SHOW if c[k])
    print(f"{name[:72]:72s} total {c['total']:5d}  {cells}")
