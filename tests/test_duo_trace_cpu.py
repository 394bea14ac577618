"""The residency report of the duo kernel's phase trace (tools/duo_trace.py residency()), on hand-made records: which CTAs
of a launch entered late, how long they ran, and how the CTAs of consecutive launches shared an SM."""
import importlib.util
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
_spec = importlib.util.spec_from_file_location("duo_trace", ROOT / "tools" / "duo_trace.py")
tr = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(tr)
ENTRY, LAST = tr.TR.index("entry"), tr.TR.index("last store")


def _records(ctas):
    """ctas: (launch, cta, smid, entry ns, last store ns); one env warp and one aux warp per CTA, the aux warp stores last"""
    recs = np.zeros(2 * len(ctas), dtype=tr.record_dtype())
    for k, (launch, cta, sm, entry, last) in enumerate(ctas):
        for role in (0, 1):
            r = recs[2 * k + role]
            r["st"], r["t"], r["cta"], r["smid"], r["role"] = 1, launch, cta, sm, role
            r["ts"][ENTRY] = entry + 32 * role
            r["ts"][LAST] = last - 64 * (1 - role)
    return recs


def test_late_ctas_and_sm_sharing():
    ctas = [(0, 0, 0, 1000, 6000), (0, 1, 0, 1100, 6100), (0, 2, 1, 1200, 6200), (0, 3, 1, 3000, 7000),   # CTA 3 late
            (1, 0, 0, 6500, 11000), (1, 1, 1, 6600, 11100), (1, 2, 1, 7100, 11200), (1, 3, 1, 6700, 11300)]
    recs = _records(ctas)
    launches = [list(range(0, 8)), list(range(8, 16))]
    out = tr.residency(recs, launches)
    late = [v for k, v in out.items() if k.startswith("env CTAs entering")]
    assert late == [0.25, [0.125, 0.25]]               # 1/4 and 0/4: the upper median, 1 of 8 CTAs, the most in one launch
    assert out["CTA last store - CTA entry, late CTAs (ns, median)"] == 4000
    assert out["CTA last store - CTA entry, other CTAs (ns, median)"] == 5000
    assert out["launches whose last store is a late CTA's"] == 1
    assert out["SMs by CTAs of launch k + launch k+1 (mean SMs per launch pair)"] == {"2+1": 1.0, "2+3": 1.0}
    # SM 0: CTAs 0, 1 of launch 0 end before CTA 0 of launch 1 enters -> 2 at once; SM 1: CTA 3 of launch 0 still runs
    # when CTAs 1 and 3 of launch 1 enter, and ends before CTA 2 does -> 3 at once
    assert out["SMs by most CTAs of launches k and k+1 resident at once (mean SMs per launch pair)"] == {"2": 1.0, "3": 1.0}


def test_summarize_includes_the_residency_rows():
    ctas = [(0, c, c % 2, 1000 + 10 * c, 6000 + 10 * c) for c in range(4)] + \
           [(1, c, c % 2, 5000 + 10 * c, 10000 + 10 * c) for c in range(4)]
    out = tr.summarize(_records(ctas), "t", 2)
    assert out["launches"] == 2
    assert out["launches whose last store is a late CTA's"] == 0
    assert out["SMs by CTAs of launch k + launch k+1 (mean SMs per launch pair)"] == {"2+2": 2.0}
