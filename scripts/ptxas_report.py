"""Registers, stack frame and spills of every kernel in one CUDA source, as ptxas reports them for sm_90a.

    python scripts/ptxas_report.py [source.cu ...] [--filter k_optimize]

Compiles with the flags of dpo_b200/build.py into a temporary directory (no GPU needed; the in-tree build is not
touched) and prints one row per kernel entry, demangled.  Compare the table before and after a change to a hot kernel:
a stack frame or spill bytes in a persistent kernel cost every phase it runs.
"""
from __future__ import annotations

import argparse
import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from dpo_b200 import build  # noqa: E402


def demangle(names):
    cxxfilt = shutil.which("c++filt")
    if not cxxfilt or not names:
        return list(names)
    res = subprocess.run([cxxfilt], input="\n".join(names), capture_output=True, text=True)
    out = res.stdout.splitlines()
    return out if len(out) == len(names) else list(names)


def report(src: str):
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [build.NVCC] + build.FLAGS + ["-c", src, "-o", os.path.join(tmp, "k.o")]
        res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{res.stderr}")
    rows, cur = [], None
    for line in res.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = {"name": m.group(1), "regs": 0, "stack": 0, "spill_st": 0, "spill_ld": 0}
            rows.append(cur)
            continue
        if cur is None:
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            cur["stack"], cur["spill_st"], cur["spill_ld"] = map(int, m.groups())
        m = re.search(r"Used (\d+) registers", line)
        if m:
            cur["regs"] = int(m.group(1))
    for r, name in zip(rows, demangle([r["name"] for r in rows])):
        r["name"] = name
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("sources", nargs="*", default=[os.path.join(build.CSRC, "dpgo_kernels.cu")])
    ap.add_argument("--filter", default="k_optimize", help="substring of the demangled kernel name ('' = all)")
    args = ap.parse_args()
    print(f"| kernel | registers | stack (B) | spill stores (B) | spill loads (B) |")
    print(f"|---|---|---|---|---|")
    for src in args.sources:
        for r in report(src):
            if args.filter in r["name"]:
                print(f"| `{r['name']}` | {r['regs']} | {r['stack']} | {r['spill_st']} | {r['spill_ld']} |")


if __name__ == "__main__":
    main()
