"""md5 of the SASS instruction listing of libgsr_b200.so (comments / line tables do not enter it).

    python tools/dev/sass_digest.py [path/to/libgsr_b200.so]
    python tools/dev/sass_digest.py --per-kernel [path/to/libgsr_b200.so]       one "digest instructions name" per kernel
    python tools/dev/sass_digest.py --compare OLD.so NEW.so                        kernels changed / removed / added
    python tools/dev/sass_digest.py --json OUT.json [path/to/libgsr_b200.so]      per-kernel digests + nvcc release

Used to show that the library built from the committed sources is, instruction for instruction, the one a GPU run
measured (profiles/README.md names the digest of the round's last GPU call), and that a change leaves the SASS of every
existing kernel byte-identical (--compare; encodings included)."""
import hashlib
import re
import shutil
import subprocess
import sys
from pathlib import Path

DEFAULT = Path(__file__).resolve().parents[2] / "gaussian_splatting_b200" / "libgsr_b200.so"


def _tool(name):
    return shutil.which(name) or f"/usr/local/cuda/bin/{name}"


def sass(lib):
    return subprocess.run([_tool("cuobjdump"), "-sass", str(lib)], check=True, capture_output=True, text=True).stdout


def per_kernel(lib):
    """{mangled kernel name: (md5 of its instruction lines, instruction count)}"""
    out, cur, lines = {}, None, []
    for line in sass(lib).splitlines() + ["Function : <end>"]:
        m = re.search(r"Function : (\S+)", line)
        if m:
            if cur is not None:
                out[cur] = (hashlib.md5("".join(lines).encode()).hexdigest(), len(lines))
            cur, lines = m.group(1), []
        elif cur is not None and re.match(r"\s+/\*[0-9a-f]{4}\*/", line):
            lines.append(line + "\n")
    out.pop("<end>", None)
    return out


def main(argv):
    if argv[:1] == ["--per-kernel"]:
        for name, (d, n) in sorted(per_kernel(argv[1] if len(argv) > 1 else DEFAULT).items()):
            print(d, n, name)
        return 0
    if argv[:1] == ["--json"]:
        import json

        ver = subprocess.run([_tool("nvcc"), "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
        kernels = {k: d for k, (d, n) in sorted(per_kernel(argv[2] if len(argv) > 2 else DEFAULT).items())}
        Path(argv[1]).write_text(json.dumps(dict(nvcc=ver, kernels=kernels), indent=0) + "\n")
        return 0
    if argv[:1] == ["--compare"]:
        old, new = per_kernel(argv[1]), per_kernel(argv[2])
        changed = sorted(k for k in old if k in new and old[k] != new[k])
        removed, added = sorted(set(old) - set(new)), sorted(set(new) - set(old))
        print(f"{len(old)} kernels before, {len(new)} after: {len(old) - len(changed) - len(removed)} identical, "
              f"{len(changed)} changed, {len(removed)} removed, {len(added)} added")
        for tag, names in (("changed", changed), ("removed", removed), ("added", added)):
            for k in names:
                print(tag, k)
        return 1 if changed or removed else 0
    lib = Path(argv[0]) if argv else DEFAULT
    text = sass(lib)
    lines = [l + "\n" for l in text.splitlines() if re.match(r"\s+/\*[0-9a-f]{4}\*/", l)]
    print(hashlib.md5("".join(lines).encode()).hexdigest(), len(lines), "instructions", lib)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
