#!/usr/bin/env python
"""Static report on the integrator sub-step loop of every wl_step_duo_kernel and wl_step_duo_deep_kernel instantiation (CPU
only: nvcc + cuobjdump).

    python tools/substep_sass.py [--src DIR | --cubin FILE] [--json OUT]

Compiles csrc/wl_api.cu with the library's flags to a cubin (or reads --cubin), finds in each duo kernel the innermost
loop that holds the force / torque butterfly (SHFL.BFLY), and prints per pass: instruction count, opcode mix, the
control flow inside the loop (BSSY / BSYNC, BRA, BRA.DIV), and a latency-weighted longest dependent chain over two
consecutive passes.  `--src` compiles another tree (a checkout of the parent commit, for an A/B of the static figures).

The chain is an estimate from the instruction stream alone: every instruction of the body is taken as executed (predicated
ones depend on their predicate and on the old value of what they write), branches cost nothing, a register written before
the loop is ready at cycle 0, and each instruction's result is ready LATENCY cycles after its last operand.  LATENCY is a
rough Hopper table, not a measurement: fixed-latency ALU ops 4 cycles; conversions and rounding (F2I, I2F, FRND) 12;
MUFU (rcp / rsqrt / sin ...) 18; SHFL 24; LDS 28; LDC 12; global loads 400."""
from __future__ import annotations

import argparse
import json
import re
import shutil
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent

LATENCY = {"F2I": 12, "I2F": 12, "FRND": 12, "F2F": 12, "MUFU": 18, "SHFL": 24, "LDS": 28, "LDC": 12, "LDG": 400, "LD": 400}
DEFAULT_LATENCY = 4
NO_DEST = {"ST", "STS", "STG", "STL", "BRA", "BSSY", "BSYNC", "BAR", "EXIT", "NOP", "WARPSYNC", "RET", "CALL", "MEMBAR",
           "RED", "CCTL", "BREAK", "JMP", "DEPBAR", "ERRBAR", "PREEXIT", "ACQBULK", "YIELD"}

_LINE = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(@!?U?P[0-9T]\s+)?([A-Z][A-Z0-9_.]*)\s*(.*?)\s*;")
_REG = re.compile(r"(?<![\w.])(U?R\d+|U?P\d)(?![\w])")
_KERNEL = re.compile(r"_Z18wl_step_duo_kernelILi(\d)ELj(\d+)E")
_DEEP_KERNEL = re.compile(r"_Z23wl_step_duo_deep_kernelILj(\d+)E")
DEEP = "deep"                                               # the FAN field of a wl_step_duo_deep_kernel<K> key


def _build_module():
    import importlib.util
    spec = importlib.util.spec_from_file_location("_wl_build", ROOT / "wheeledlab_b200" / "build.py")
    b = importlib.util.module_from_spec(spec); spec.loader.exec_module(b)
    return b


def tools():
    """(nvcc, cuobjdump) or None when either is missing"""
    nvcc = shutil.which(_build_module().NVCC)
    if nvcc is None:
        return None
    cuobjdump = shutil.which("cuobjdump", path=str(Path(nvcc).parent)) or shutil.which("cuobjdump")
    return (nvcc, cuobjdump) if cuobjdump else None


def compile_cubin(src_root: Path, out: Path) -> Path:
    b = _build_module()
    flags = [f for f in b.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC")]
    cmd = [b.NVCC, *flags, "-cubin", "-o", str(out), str(src_root / "wheeledlab_b200" / "csrc" / "wl_api.cu")]
    subprocess.run(cmd, check=True, cwd=str(src_root))
    return out


def kernel_name(fan, k) -> str:
    return f"wl_step_duo_deep_kernel<0x{k:08x}>" if fan == DEEP else f"wl_step_duo_kernel<{fan}, 0x{k:08x}>"


def sorted_kernels(sass: dict):
    """the items of kernel_sass(), wl_step_duo_kernel instantiations first"""
    return sorted(sass.items(), key=lambda kv: (kv[0][0] == DEEP, str(kv[0][0]), kv[0][1]))


def kernel_sass(cubin: Path):
    """{(FAN, K): [(addr, pred, opcode, operands)]} for every duo kernel in the cubin; FAN = DEEP for
    wl_step_duo_deep_kernel<K>"""
    txt = subprocess.run([tools()[1], "-sass", str(cubin)], check=True, capture_output=True, text=True).stdout
    out, cur = {}, None
    for line in txt.splitlines():
        if "Function :" in line:
            m, d = _KERNEL.search(line), _DEEP_KERNEL.search(line)
            cur = (int(m.group(1)), int(m.group(2))) if m else (DEEP, int(d.group(1))) if d else None
            if cur is not None:
                out[cur] = []
            continue
        if cur is None:
            continue
        m = _LINE.search(line)
        if m:
            out[cur].append((int(m.group(1), 16), (m.group(2) or "").strip(), m.group(3), m.group(4)))
    return out


def find_loop(ins):
    """(first, last) index of the innermost backward branch's body that contains the SHFL.BFLY butterfly"""
    addr = [a for a, *_ in ins]
    idx = {a: k for k, a in enumerate(addr)}
    bfly = [k for k, (_, _, op, _) in enumerate(ins) if op.startswith("SHFL.BFLY")]
    best = None
    for k, (a, _, op, ops) in enumerate(ins):
        if op.split(".")[0] != "BRA" or op.startswith("BRA.DIV"):
            continue
        m = re.search(r"0x([0-9a-f]+)", ops)
        if not m:
            continue
        tgt = int(m.group(1), 16)
        if tgt >= a or tgt not in idx:
            continue
        lo = idx[tgt]
        if any(lo <= s <= k for s in bfly) and (best is None or k - lo < best[1] - best[0]):
            best = (lo, k)
    return best


def _regs(tok: str, width: int):
    out = []
    for r in _REG.findall(tok):
        out.append(r)
        if width > 1 and r[0] in "RU" and not r.startswith(("P", "UP")):
            pre = "UR" if r.startswith("UR") else "R"
            n = int(r[len(pre):])
            out += [f"{pre}{n + d}" for d in range(1, width)]
    return out


def dest_src(pred: str, op: str, operands: str):
    base = op.split(".")[0]
    width = 4 if ".128" in op else 2 if ".64" in op else 1
    toks = [t.strip() for t in operands.split(",")] if operands else []
    dst, src = [], []
    if base not in NO_DEST and toks:
        nd = 2 if (len(toks) > 1 and re.fullmatch(r"!?U?P(\d|T)", toks[0])) or \
                  (len(toks) > 1 and re.fullmatch(r"U?P(\d|T)", toks[1]) and base in ("IADD3", "IMAD", "LEA", "IADD")) else 1
        dst = [r for t in toks[:nd] for r in _regs(t, width if base.startswith("LD") or width > 1 else 1)]
        toks = toks[nd:]
    for t in toks:
        src += _regs(t, width if base.startswith("ST") or base in ("DADD", "DMUL", "DFMA") else 1)
    if pred:
        src.append(pred.lstrip("@!"))
        src += dst                                          # a predicated write keeps the old value otherwise
    return dst, src


def chain(body, passes: int = 2) -> int:
    ready, longest = {}, 0
    for _ in range(passes):
        for _, pred, op, operands in body:
            base = op.split(".")[0]
            if base in ("BRA", "BSSY", "BSYNC", "NOP"):
                continue
            dst, src = dest_src(pred, op, operands)
            t = max([ready.get(r, 0) for r in src], default=0) + LATENCY.get(base, DEFAULT_LATENCY)
            for r in dst:
                ready[r] = t
            longest = max(longest, t)
    return longest


def report(cubin: Path):
    rows = []
    for (fan, k), ins in sorted_kernels(kernel_sass(cubin)):
        loop = find_loop(ins)
        row = {"kernel": kernel_name(fan, k), "fan": fan, "spec": k}
        if loop is None:
            row["error"] = "no sub-step loop found"
            rows.append(row); continue
        body = ins[loop[0]:loop[1] + 1]
        mix = {}
        for _, _, op, _ in body:
            mix[op.split(".")[0]] = mix.get(op.split(".")[0], 0) + 1
        row.update({
            "loop": f"0x{body[0][0]:04x}-0x{body[-1][0]:04x}",
            "instructions_per_pass": len(body),
            "bssy": sum(op == "BSSY" for _, _, op, _ in body),
            "bsync": sum(op == "BSYNC" for _, _, op, _ in body),
            "bra": sum(op.split(".")[0] == "BRA" and not op.startswith("BRA.DIV") for _, _, op, _ in body),
            "bra_div": sum(op.startswith("BRA.DIV") for _, _, op, _ in body),
            "chain_two_passes": chain(body, 2),
            "mix": dict(sorted(mix.items(), key=lambda kv: -kv[1])),
        })
        rows.append(row)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--src", default=str(ROOT), help="tree to compile (default: this checkout)")
    ap.add_argument("--cubin", default=None, help="read this cubin instead of compiling")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    with tempfile.TemporaryDirectory(prefix="wl_sass_") as td:
        cubin = Path(args.cubin) if args.cubin else compile_cubin(Path(args.src).resolve(), Path(td) / "wl_api.cubin")
        rows = report(cubin)
    for r in rows:
        if "error" in r:
            print(f"{r['kernel']}: {r['error']}"); continue
        print(f"{r['kernel']}  loop {r['loop']}: {r['instructions_per_pass']} instructions per pass, BSSY {r['bssy']} / BSYNC "
              f"{r['bsync']} / BRA {r['bra']} / BRA.DIV {r['bra_div']}, chain over two passes {r['chain_two_passes']} cycles")
        print("    " + ", ".join(f"{k} {v}" for k, v in r["mix"].items()))
    if args.json:
        Path(args.json).write_text(json.dumps(rows, indent=1) + "\n")


if __name__ == "__main__":
    main()
