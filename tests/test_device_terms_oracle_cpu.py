"""The oracle's twin of the device terms (oracle/wl_oracle.c: term_value, dterms_env, dterms_log; DESIGN.md 6l) against the
reference's own functions (tests/golden/device_terms.npz, make_golden.py) and against the fp64 oracle, without a GPU.

* Discrete outcomes: on every golden state and parameter set the fp32 oracle takes the reference's branch (value zero or
  not, a clamp at its cap or not) and its indicator terms equal the reference's values exactly.  The designed states sit on
  every threshold and one fp32 ulp either side (tests/golden/make_golden.py), so a comparison turned from ``>`` into ``>=``
  or a cell lookup one cell off shows here.
* Continuous outputs: |fp32 oracle - fp64 oracle| and |golden - fp64 oracle| are within a written-out rounding bound
  (below).  The reference forms v_b with the quaternion formula and its angles with libm; the oracle (and the kernel) with
  the rotation matrix and the deterministic polynomials.  Both are fp32 evaluations of the same function, so both lie
  within the bound of the fp64 value.
* The fp64 oracle takes the reference's branches on the random states.  The designed states are left out of that check:
  at one fp32 ulp from a threshold the fp64 evaluation legitimately lands on the other side.
"""
from __future__ import annotations

import numpy as np
import pytest

import oracle_lib as O
import device_terms_golden as D

G = D.G
U = 2.0 ** -24
NR = int(G["n_random"])
CAPS = {"forward_vel": np.float32(1.2), "forward_wheel_spin": np.float32(200.0)}
INDICATORS = ("low_vel_penalty", "is_traversable", "low_speed_penalty", "off_track", "roll_over", "bool_is_not_traversable")
ANGLE_TERMS = ("steep_penalty", "upright_penalty")


@pytest.fixture(scope="module")
def cfg():
    return D.config().cfg


def _vals(cfg, name, params, kind="f32", t=0, st=None):
    st = D.state() if st is None else st
    o = O.device_terms(cfg, D.table(name, params, cfg), st, np.zeros(st.shape[1], np.uint8), t, vis_map=G["map"], kind=kind)
    return o


def _bound(name, ref):
    """A rounding bound on |fp32 evaluation - exact value| per state.  Every fp32 operation rounds with relative error <= u;
    the inputs enter v_b = R(q)^T v and w_b through at most 9 roundings each, with |R| <= |q|^2 per entry (|q| <= 3 here),
    a sum of 4 wheel speeds through 3, a sqrt or a square through 2 more and the terms' own few operations; 64 u of the
    magnitudes involved covers every chain with room.  The angle terms add the polynomial atan / asin (<= 2e-7 absolute,
    cephes) and the libm angle of the reference, each scaled by 57.3 degrees per radian for upright_penalty."""
    q2 = np.sum(G["quat"].astype(np.float64) ** 2, axis=1)
    mag = (1.0 + np.abs(ref) + q2 * (np.abs(G["vel_w"]).sum(1) + np.abs(G["ang_w"]).sum(1)) + np.abs(G["omega"]).sum(1)
           + np.abs(G["pos"]).sum(1))
    e = 64 * U * mag * (1.0 + mag if name in ("yaw_change_onElev", "vel_rew_trav") else 1.0)
    if name in ANGLE_TERMS:
        e = e + (1e-6 + 64 * U * np.abs(ref)) * (57.3 if name == "upright_penalty" else 1.0)
    if name == "upright_penalty":         # arccos amplifies r22's rounding by 1 / sqrt(1 - r22^2)
        q = G["quat"].astype(np.float64)
        r22 = 1.0 - 2.0 * (q[:, 1] ** 2 + q[:, 2] ** 2) / np.maximum(q2, 1e-30)
        e = e + 57.3 * 16 * U / np.sqrt(np.maximum(1.0 - r22 ** 2, 1e-300))
    return e


def _branch(name, v):
    b = v != 0
    if name in CAPS:
        b = b | (v.astype(np.float32) == CAPS[name]) * 2
    return b


@pytest.mark.parametrize("name", D.STATE_FUNCS)
def test_fp32_oracle_takes_the_references_branch_on_every_golden_state(cfg, name):
    for j, ps in enumerate(G["p_" + name]):
        ref = G["f_" + name][j]
        v = _vals(cfg, name, ps)["vals"][:, 0]
        bad = np.nonzero(_branch(name, v) != _branch(name, ref))[0]
        assert bad.size == 0, f"{name}{tuple(ps)}: branch differs at states {bad[:8].tolist()}"
        if name in INDICATORS:
            assert np.array_equal(v.astype(np.float32), ref), f"{name}{tuple(ps)}"


@pytest.mark.parametrize("name", [n for n in D.STATE_FUNCS if n not in INDICATORS])
def test_continuous_values_within_the_rounding_bound_of_fp64(cfg, name):
    worst = 0.0
    for j, ps in enumerate(G["p_" + name]):
        ref = G["f_" + name][j].astype(np.float64)
        v32 = _vals(cfg, name, ps)["vals"][:, 0]
        v64 = _vals(cfg, name, ps, kind="f64")["vals"][:, 0]
        same = (_branch(name, v64) == _branch(name, ref)) & (_branch(name, v64) == _branch(name, v32))
        if name in ("is_traversable_speed_scaled", "vel_rew_trav"):      # and the same cell (a cell edge is a branch too)
            same &= _vals(cfg, "is_traversable", [], kind="f64")["vals"][:, 0] == G["f_is_traversable"][0]
        e = _bound(name, v64)
        for got in (v32, ref):
            err = np.abs(got - v64)[same]
            assert (err <= e[same]).all(), f"{name}{tuple(ps)}: max |err| / bound {np.max(err / e[same]):.3g}"
            worst = max(worst, float(np.max(err / e[same])))
    print(f"{name}: largest |err| / bound {worst:.3g}")


@pytest.mark.parametrize("name", D.STATE_FUNCS)
def test_fp64_oracle_takes_the_references_branch_on_random_states(cfg, name):
    for j, ps in enumerate(G["p_" + name]):
        ref = G["f_" + name][j][:NR]
        v = _vals(cfg, name, ps, kind="f64")["vals"][:NR, 0]
        bad = np.nonzero(_branch(name, v) != _branch(name, ref))[0]
        assert bad.size == 0, f"{name}{tuple(ps)}: branch differs at random states {bad[:8].tolist()}"


def test_bool_is_not_traversable_either_side_of_the_switch(cfg):
    for kind in ("f32", "f64"):
        for c, ref in zip(G["t_bool_is_not_traversable"], G["f_bool_is_not_traversable"]):
            v = _vals(cfg, "bool_is_not_traversable", [], kind=kind, t=int(c))["vals"][:, 0]
            if kind == "f32":
                assert np.array_equal(v.astype(np.float32), ref), f"counter {c}"
            else:
                assert np.array_equal(v[:NR].astype(np.float32), ref[:NR]), f"counter {c}"
    assert G["f_bool_is_not_traversable"][0].sum() == 0 and G["f_bool_is_not_traversable"][1].sum() > 0


def test_elevation_continuity_sequences(cfg):
    """Three calls per sequence on the same envs (first call, no change, rise, fall, z on the threshold and one ulp either
    side); the previous elevation is unset before each sequence (the reference's function attribute deleted)."""
    zs = G["cont_z"]
    m = zs.shape[1]
    for j, ps in enumerate(G["p_elevation_continuity"]):
        prev = None
        for k in range(zs.shape[0]):
            pos = np.zeros((m, 3), np.float32); pos[:, 2] = zs[k]
            o = O.device_terms(cfg_n(m), D.table("elevation_continuity", ps, cfg), D.state(pos=pos), np.zeros(m, np.uint8), 0,
                               vis_map=G["map"], prev=prev)
            prev = o["prev"]
            assert np.array_equal(o["vals"][:, 0].astype(np.float32), G["f_elevation_continuity"][j, k]), f"threshold {ps}, call {k}"
    assert (G["f_elevation_continuity"][:, 0] == 0).all()


def cfg_n(n):
    return D.config(n).cfg


@pytest.mark.parametrize("n", [1, 127, 128, 129, 4097, 33 * 128 + 1, 9000])
def test_episode_log_is_the_fixed_order_sum_within_its_bound(n):
    """Episode_* of one step against an fp64 sum of the same per-env episode sums.  A sum of m fp32 values in any tree order
    is within (ceil(log2 m) + 1) u sum|x| of the exact sum; the count column is exact.  The lane-strided pass over more than
    32 CTAs is exercised from n > 4096."""
    c = cfg_n(n)
    rng = np.random.default_rng(n)
    st = np.zeros((D.NUM_GROUPS, n, 4), np.float32)
    st[D.G_QUAT, :, 0] = 1.0
    st[D.G_LINVEL, :, 0] = rng.uniform(-2, 2, n).astype(np.float32)
    st[D.G_LINVEL, :, 2] = rng.uniform(-1, 1, n).astype(np.float32)
    done = (rng.random(n) < 0.7).astype(np.uint8)
    sums = np.zeros((8, n)); sums[0] = rng.uniform(-5, 5, n).astype(np.float32); sums[1] = rng.uniform(0, 3, n).astype(np.float32)
    terms = [(1, 0, 1.0 / D.step_dt(c), []), (4, 0, 2.0, []), (14, 1, 0.0, [0.5])]
    o = O.device_terms(c, terms, st, done, 0, vis_map=G["map"], sums=sums.copy())
    vals = o["vals"]
    scale = np.array([np.float32(1.0 / D.step_dt(c) * D.step_dt(c)), np.float32(2.0 * D.step_dt(c))], np.float64)
    ep = np.stack([sums[0] + np.float32(vals[:, 0] * scale[0]), sums[1] + np.float32(vals[:, 1] * scale[1])], 1)
    fired = (o["fired"] >> 2) & 1
    d = (done != 0) | (fired != 0)
    cnt = d.sum()
    levels = int(np.ceil(np.log2(max(n, 2)))) + 8
    L = float(c.episode_length_s)
    for k in range(2):
        exact = ep[d, k].sum() / max(cnt, 1) / L
        bound = ((levels + 3) * U * np.abs(ep[d, k]).sum()) / max(cnt, 1) / L + 3 * U * abs(exact) + 1e-30
        assert abs(o["term_log"][k] - exact) <= bound, (k, o["term_log"][k], exact, bound)
    assert o["term_log"][2] == float(((done != 0) | (fired != 0))[fired != 0].sum())
    assert (o["term_log"][3:] == 0).all()
    # the per-episode sums: zeroed for the done envs, carried for the others
    assert np.array_equal(o["sums"][0][~d], np.float32(ep[~d, 0]).astype(np.float64))
    assert (o["sums"][:2, d] == 0).all()
