"""Instruction counts of the loops of a kernel in an object file (cuobjdump -sass):
    python tools/dev/sass_loops.py gaussian_splatting_b200/_build/gsr_render.o k_render_bwdILb1
    python tools/dev/sass_loops.py --inner gaussian_splatting_b200/_build/gsr_render.o k_render_bwdILb1EE
Default: every backward branch (loop) with its body length and an opcode histogram of the largest loops.
--inner: the innermost loops instead (the tile walks), in address order.  A compare-and-swap retry loop (how sm_90
compiles a shared-memory float atomicAdd) does not make the loop around it an outer loop; it is counted as a
"spin" loop inside it."""
import collections
import re
import subprocess
import sys


def opcode(t):
    return re.sub(r"^@!?U?P\w+\s+", "", t).split()[0]


def main():
    args = sys.argv[1:]
    inner = "--inner" in args
    obj, pat = [a for a in args if a != "--inner"]
    txt = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
    funcs = re.split(r"\n\s+Function : ", txt)
    for f in funcs[1:]:
        name = f.split("\n", 1)[0]
        if pat not in name:
            continue
        ins = []
        for line in f.splitlines():
            m = re.match(r"\s+/\*([0-9a-f]{4,5})\*/\s+(.*?);", line)
            if m:
                ins.append((int(m.group(1), 16), m.group(2).strip()))
        addr_idx = {a: i for i, (a, _) in enumerate(ins)}
        print(name, "total", len(ins))
        loops = []  # (first index, last index) of every backward branch's body
        for i, (a, t) in enumerate(ins):
            m = re.search(r"BRA(?:\.\w+)*\s+(?:\w+,\s*)?0x([0-9a-f]+)", t)
            if m:
                tgt = int(m.group(1), 16)
                if tgt <= a and tgt in addr_idx:
                    loops.append((addr_idx[tgt], i))

        def hist(lo, hi):
            return collections.Counter(opcode(t).split(".")[0] for _, t in ins[lo:hi + 1])

        if not inner:
            for lo, hi in sorted(loops, key=lambda l: l[1] - l[0], reverse=True)[:8]:
                h = hist(lo, hi)
                print(f"  loop {ins[lo][0]:#06x}..{ins[hi][0]:#06x}: {hi - lo + 1} instr  "
                      + " ".join(f"{k}:{v}" for k, v in h.most_common(14)))
            continue
        def inside(lo, hi):
            return [l for l in loops if l != (lo, hi) and lo <= l[0] and l[1] <= hi]

        spin = {l for l in loops if not inside(*l) and any(".CAS" in opcode(t) for _, t in ins[l[0]:l[1] + 1])}
        for lo, hi in sorted(loops):
            if (lo, hi) in spin:
                continue
            nested = inside(lo, hi)
            if any(l not in spin for l in nested):
                continue
            h = hist(lo, hi)
            ops = [opcode(t) for _, t in ins[lo:hi + 1]]
            atoms = [o for o in ops if o.startswith("ATOMS")]
            print(f"  inner loop {ins[lo][0]:#06x}..{ins[hi][0]:#06x}: {hi - lo + 1} instr, "
                  f"LDL {h['LDL']} STL {h['STL']}, {len(nested)} spin loops, shared atomics {atoms}")
            print("    " + " ".join(f"{k}:{v}" for k, v in h.most_common(16)))


if __name__ == "__main__":
    main()
