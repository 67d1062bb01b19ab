"""Per-kernel SASS comparison of two builds of libepp_engine.so (no GPU needed): which kernels compile to the same
instructions.  A change confined to the pool kernels must leave every per-request kernel identical.

    python tools/sass_compare.py OLD.so NEW.so
"""
from __future__ import annotations

import re
import subprocess
import sys


def kernels(lib: str) -> dict:
    """Kernel name -> SASS lines.  Anonymous-namespace hashes and the source-file identifiers (which depend on the
    build directory) are dropped."""
    out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    fs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = re.sub(r"_GLOBAL__N__[0-9a-f]+_(\d+)_(\w+?)_cu_[0-9a-f]+", r"_GLOBAL__N_\2", m.group(1))
            fs[cur] = []
        elif cur is not None and "identifier =" not in line:
            fs[cur].append(" ".join(line.split()))     # the column padding follows the widest line of the whole module
    return fs


def main(old: str, new: str) -> int:
    a, b = kernels(old), kernels(new)
    same, changed = 0, []
    for n in sorted(set(a) | set(b)):
        if n not in a or n not in b:
            print(("removed: " if n in a else "added:   ") + n)
        elif a[n] == b[n]:
            same += 1
        else:
            changed.append(n)
            print("changed: " + n)
    print(f"identical: {same}  changed: {len(changed)}")
    return 1 if changed else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1], sys.argv[2]))
