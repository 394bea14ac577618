"""Compare the SASS of two builds of the CUDA library kernel by kernel, and print the resources of the kernels the second one
adds: the check that a change left every existing kernel's instructions as they were.

    python tools/sass_compare.py <before.so> <after.so> [--ptxas-log build.log]

Build the `before` library from the parent commit (`git stash; python wheeledlab_b200/build.py; cp ...`).  Addresses are
stripped; opcodes, operands and encodings are compared.  `--ptxas-log`: the output of `nvcc -Xptxas -v` for the `after`
build (`python wheeledlab_b200/build.py` prints it), from which registers, shared memory and spills of the new kernels are
listed.  Needs cuobjdump, no GPU.  Exit code 1 if an existing kernel changed or disappeared."""
from __future__ import annotations

import argparse
import re
import subprocess
import sys

CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"


def sass(lib: str) -> dict:
    out = subprocess.run([CUOBJDUMP, "-sass", lib], capture_output=True, text=True, check=True).stdout
    fns, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            fns[cur] = []
        elif cur and re.match(r"\s+/\*[0-9a-f]{4}\*/", line):
            fns[cur].append(re.sub(r"^\s*/\*[0-9a-f]{4}\*/", "", line).strip())
    return fns


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("before")
    ap.add_argument("after")
    ap.add_argument("--ptxas-log", default=None)
    a = ap.parse_args()
    old, new = sass(a.before), sass(a.after)
    changed = [k for k in old if k not in new or old[k] != new[k]]
    added = [k for k in new if k not in old]
    print(f"{len(old)} kernels before, {len(new)} after; {len(old) - len(changed)} identical instruction for instruction")
    for k in changed:
        print("CHANGED" if k in new else "REMOVED", k)
    for k in added:
        print("new", k, f"({len(new[k])} instructions)")
    if a.ptxas_log:
        log = open(a.ptxas_log).read()
        for name, spills, used in re.findall(r"Compiling entry function '(\S+)' for 'sm_90a'\n(?:ptxas info\s*:.*\n)*?ptxas info\s*: Function "
                                             r"properties for \S+\n\s*(.*)\nptxas info\s*: Used (.*)\n", log):
            if name in added:
                print(f"  {name}: {used}; {spills}")
    sys.exit(1 if changed else 0)


if __name__ == "__main__":
    main()
