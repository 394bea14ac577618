#!/usr/bin/env python
"""Static report on the segments of the duo kernels (wl_step_duo_kernel, wl_step_duo_deep_kernel) outside their sub-step
loop (CPU only: nvcc + cuobjdump).

    python tools/phase_sass.py [--src DIR | --cubin FILE] [--json OUT]

Splits each duo instantiation's SASS at its named barriers, in code order: the env warp from entry to `bar.sync 1`, the sub-step
loop region up to `bar.arrive 2`, and from there to the env warp's exit; the aux warp from that exit to `bar.arrive 1`, and from
`bar.sync 2` to its exit.  Per segment: instructions, BSSY (divergent regions), CALL (slow-path calls), BRA.  The out-of-line
slow-path bodies after the last exit are not counted.  `--src` compiles another tree (the parent commit, for an A/B)."""
from __future__ import annotations

import argparse
import json
import tempfile
from pathlib import Path

import substep_sass as ss

SEGMENTS = ("env: entry -> bar.sync 1", "env: bar.sync 1 -> bar.arrive 2", "env: bar.arrive 2 -> exit",
            "aux: start -> bar.arrive 1", "aux: bar.sync 2 -> exit")


def _is(ins, op, bar=None):
    _, pred, o, ops = ins
    if not o.startswith(op):
        return False
    return bar is None or ops.split(",")[0].strip() == hex(bar)


def segments(ins):
    """{segment: (first, last) index} of one duo kernel"""
    k = lambda pred, start=0: next(j for j in range(start, len(ins)) if pred(ins[j]))
    sync1 = k(lambda x: _is(x, "BAR.SYNC", 1))
    arv2 = k(lambda x: _is(x, "BAR.ARV", 2), sync1)
    env_exit = k(lambda x: x[2] == "EXIT" and not x[1], arv2)
    arv1 = k(lambda x: _is(x, "BAR.ARV", 1), env_exit)
    sync2 = k(lambda x: _is(x, "BAR.SYNC", 2), arv1)
    aux_exit = k(lambda x: x[2] == "EXIT" and not x[1], sync2)
    return dict(zip(SEGMENTS, ((0, sync1), (sync1, arv2), (arv2, env_exit), (env_exit + 1, arv1), (sync2, aux_exit))))


def report(cubin: Path):
    rows = []
    for (fan, key), ins in ss.sorted_kernels(ss.kernel_sass(cubin)):
        row = {"kernel": ss.kernel_name(fan, key), "fan": fan, "spec": key}
        for name, (a, b) in segments(ins).items():
            body = ins[a:b + 1]
            row[name] = {"instructions": len(body), "bssy": sum(o == "BSSY" for _, _, o, _ in body),
                         "call": sum(o.startswith("CALL") for _, _, o, _ in body),
                         "bra": sum(o.split(".")[0] == "BRA" for _, _, o, _ in body)}
        rows.append(row)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--src", default=str(ss.ROOT), help="tree to compile (default: this checkout)")
    ap.add_argument("--cubin", default=None, help="read this cubin instead of compiling")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    with tempfile.TemporaryDirectory(prefix="wl_sass_") as td:
        cubin = Path(args.cubin) if args.cubin else ss.compile_cubin(Path(args.src).resolve(), Path(td) / "wl_api.cubin")
        rows = report(cubin)
    for r in rows:
        print(r["kernel"])
        for name in SEGMENTS:
            s = r[name]
            print(f"    {name:34s} {s['instructions']:5d} instructions, BSSY {s['bssy']:2d}, CALL {s['call']}, BRA {s['bra']:2d}")
    if args.json:
        Path(args.json).write_text(json.dumps(rows, indent=1) + "\n")


if __name__ == "__main__":
    main()
