"""Compare the SASS of two libbgs.so builds kernel by kernel (cuobjdump -sass; runs without a GPU).

    python scripts/sass_diff.py old/libbgs.so new/libbgs.so

Prints the kernels only one build has and every kernel present in both whose instruction text differs (addresses and
encodings are ignored, so only a change of code counts).  Exit status 1 when a shared kernel differs.
"""
from __future__ import annotations

import re
import subprocess
import sys

CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"


def kernels(lib: str) -> dict[str, list[str]]:
    text = subprocess.run([CUOBJDUMP, "-sass", lib], check=True, capture_output=True, text=True).stdout
    out, name = {}, None
    for line in text.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            out[name] = []
            continue
        m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
        if name is not None and m:
            out[name].append(m.group(1).strip())
    return out


def main():
    old, new = kernels(sys.argv[1]), kernels(sys.argv[2])
    for k in sorted(set(old) - set(new)):
        print(f"only in {sys.argv[1]}: {k}")
    for k in sorted(set(new) - set(old)):
        print(f"only in {sys.argv[2]}: {k} ({len(new[k])} instructions)")
    changed = [k for k in sorted(set(old) & set(new)) if old[k] != new[k]]
    for k in changed:
        print(f"changed: {k}")
    print(f"{len(set(old) & set(new))} kernels in both, {len(changed)} changed")
    sys.exit(1 if changed else 0)


if __name__ == "__main__":
    main()
