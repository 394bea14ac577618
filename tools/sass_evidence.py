#!/usr/bin/env python
"""Per kernel of the built library, the static instruction count and the SASS mnemonics that prove
which hardware paths are used (TMA, bulk copies, mbarriers, named barriers, fire-and-forget atomics, IEEE slow paths).

    python tools/sass_evidence.py > sass_evidence.txt
"""
import collections
import re
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
LIB = ROOT / "wheeledlab_b200" / "libwheeledlab_b200.so"
KEYS = ["INSTR", "UTMALDG", "UBLKCP", "SYNCS", "BAR.ARV", "BAR.SYNC", "REDG", "ATOMG", "MUFU.RCP", "MUFU.RSQ", "FCHK", "SHFL", "STRONG.SYS",
        "PREEXIT", "ACQBULK", "CCTL.E.PF2"]


def main():
    sass = subprocess.run(["cuobjdump", "-sass", str(LIB)], capture_output=True, text=True).stdout
    rows, name, proofs = collections.defaultdict(collections.Counter), None, []
    for ln, line in enumerate(sass.split("\n")):
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip().split("(")[0]
            continue
        m = re.match(r"\s+/\*([0-9a-f]{4,5})\*/\s+(.*?);", line)
        if not m or name is None:
            continue
        rows[name]["INSTR"] += 1
        for k in KEYS[1:]:
            if k in m.group(2):
                rows[name][k] += 1
        if "UTMALDG" in m.group(2) or "UBLKCP" in m.group(2) or ("STG" in m.group(2) and "STRONG.SYS" in m.group(2)):
            proofs.append(f"{name}: /*{m.group(1)}*/ {m.group(2).strip()}")
    print("# cuobjdump -sass wheeledlab_b200/libwheeledlab_b200.so (sm_90a): static instruction count per kernel and the mnemonics that prove the")
    print("# hardware paths used.  UTMALDG.2D = cp.async.bulk.tensor.2d (TMA tile of the height-field, wl_scan_kernel<true>); UBLKCP = cp.async.bulk")
    print("# 1-D (policy weight blob, wl_act_step_quad_kernel); SYNCS = mbarrier arrive / expect_tx / try_wait; BAR.ARV + BAR.SYNC = named barriers")
    print("# of the env-warp / aux-warp hand-off (wl_step_duo_kernel); REDG = fire-and-forget reductions of the episode log (no ticket, no fence);")
    print("# ATOMG = the K-step rollout's last-CTA ticket; FCHK = range check of an IEEE division with slow-path call (the integrator sub-step uses")
    print("# fdiv_norm / fsqrt_norm instead).  No wgmma anywhere: there is no dense contraction on this path (tensor cores unused by design).")
    print("# STG...STRONG.SYS = multimem.st.relaxed.sys (wl_step_duo_kernel: output rows stored once to the NVSwitch multicast alias of the symmetric")
    print("# rollout buffers, replicated by the switch into every rank's copy; wl_set_multicast_fanout); in the other kernels STRONG.SYS marks the")
    print("# system-scope loads/stores of the peer-memory all-reduce (wl_dp_adam_kernel) and of the flag protocols.")
    print("# PREEXIT = griddepcontrol.launch_dependents and ACQBULK = griddepcontrol.wait (programmatic dependent launch); CCTL.E.PF2 =")
    print("# prefetch.global.L2 (wl_step_duo_kernel: the lines of its first loads, requested before the wait).")
    print("kernel | " + " | ".join(KEYS))
    for n in sorted(rows):
        print(n[:64] + " | " + " | ".join(str(rows[n].get(k, 0)) for k in KEYS))
    print("\n# instruction sites:")
    for p in proofs:
        print(p)


if __name__ == "__main__":
    main()
