"""Compare the SASS of two libbgs.so builds kernel by kernel (cuobjdump -sass; runs without a GPU).

    python scripts/sass_diff.py old/libbgs.so new/libbgs.so
    python scripts/sass_diff.py --ignore-params --rename 'raster_mixed_kernel<(\\(int\\)\\d), (\\(bool\\)\\d)>' \\
        'raster_kernel<\\1, (bool)0, \\2, (bool)0, bgs::OneView>' old/libbgs.so new/libbgs.so

Kernels are paired by demangled name without the parameter list.  --rename PATTERN REPLACEMENT (repeatable) rewrites the
old build's names with re.sub before pairing, so kernels renamed between the builds pair up; each new kernel may pair with
one old kernel only.  --ignore-params compares kernel-parameter constant-bank operands (c[0x0][...]) as equal, so a kernel
whose parameters moved pairs as unchanged when nothing else differs.

Prints the kernels only one build has, every pair whose instruction text differs (addresses and encodings are ignored, so
only a change of code counts) with its differing instructions, and each pair's REG / STACK / SHARED / LOCAL from
cuobjdump --dump-resource-usage, marked when they differ.  Exit status 1 when a pair differs in code or resources.
"""
from __future__ import annotations

import argparse
import re
import subprocess
import sys

CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"
CUFILT = "/usr/local/cuda/bin/cu++filt"
RESOURCES = ("REG", "STACK", "SHARED", "LOCAL")
PARAM = re.compile(r"c\[0x0\]\[0x[0-9a-f]+\]")


def demangle(names: list[str]) -> dict[str, str]:
    """mangled -> demangled name without its return type and parameter list"""
    out = subprocess.run([CUFILT], input="\n".join(names), check=True, capture_output=True, text=True).stdout.splitlines()
    short = {}
    for m, d in zip(names, out):
        depth, end = 0, len(d)
        for i, ch in enumerate(d):   # the parameter list: the first '(' outside the template arguments
            if ch == "<":
                depth += 1
            elif ch == ">":
                depth -= 1
            elif ch == "(" and depth == 0:
                end = i
                break
        short[m] = re.sub(r"^void ", "", d[:end])
    return short


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


def resources(lib: str) -> dict[str, dict[str, int]]:
    text = subprocess.run([CUOBJDUMP, "--dump-resource-usage", lib], check=True, capture_output=True, text=True).stdout
    out, name = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        if name is not None and "REG:" in line:
            out[name] = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", line) if k in RESOURCES}
            name = None
    return out


def load(lib: str, renames: list[tuple[str, str]]):
    sass, res = kernels(lib), resources(lib)
    names = demangle(sorted(sass))
    out = {}
    for m, d in names.items():
        for pat, rep in renames:
            d = re.sub(pat, rep, d)
        if d in out:
            sys.exit(f"{lib}: two kernels pair as {d}")
        out[d] = (sass[m], res.get(m, {}))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--rename", nargs=2, action="append", default=[], metavar=("PATTERN", "REPLACEMENT"))
    ap.add_argument("--ignore-params", action="store_true")
    args = ap.parse_args()
    old, new = load(args.old, [tuple(r) for r in args.rename]), load(args.new, [])
    norm = (lambda ins: [PARAM.sub("c[0x0][param]", i) for i in ins]) if args.ignore_params else (lambda ins: ins)
    for k in sorted(set(old) - set(new)):
        print(f"only in {args.old}: {k}")
    for k in sorted(set(new) - set(old)):
        print(f"only in {args.new}: {k} ({len(new[k][0])} instructions)")
    changed = 0
    for k in sorted(set(old) & set(new)):
        (so, ro), (sn, rn) = old[k], new[k]
        a, b = norm(so), norm(sn)
        res = " ".join(f"{r}:{ro.get(r)}" + ("" if ro.get(r) == rn.get(r) else f"->{rn.get(r)}") for r in RESOURCES)
        if a == b and ro == rn:
            print(f"same: {k} [{res}]")
            continue
        changed += 1
        print(f"changed: {k} [{res}]")
        if len(a) != len(b):
            print(f"    {len(a)} -> {len(b)} instructions")
        else:
            for i, (x, y) in enumerate(zip(a, b)):
                if x != y:
                    print(f"    {i:5d}: {x}  ->  {y}")
    print(f"{len(set(old) & set(new))} kernels in both, {changed} changed")
    sys.exit(1 if changed else 0)


if __name__ == "__main__":
    main()
