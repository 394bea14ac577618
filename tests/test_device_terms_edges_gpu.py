"""Device terms on the GPU against the oracle's twin (DESIGN.md 6l), bit for bit:

* placed states: the handle's own wl_terms_kernel + wl_terms_log_kernel (wl_test_device_terms) on every golden state of
  tests/golden/device_terms.npz (thresholds exactly and one ulp either side, Euler-angle and r22 edges, off_track and cell
  edges), one term per table, weight 1 / step_dt so that the reward is the term's value;
* the test entry on the pre-reset state wl_step_stage_a leaves equals wl_step_terms;
* trajectories: obs, reward, done masks, fired bits, term_log and state against wlo_step_terms every step;
* the Episode_* log over more than 32 CTAs against an fp64 sum of the kernel's own per-env contributions."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import wheeledlab_b200 as wl                                   # noqa: E402
from wheeledlab_b200 import _lib                               # noqa: E402
from wheeledlab_b200.sim import WheeledSim                     # noqa: E402

import device_terms_golden as D                                # noqa: E402
import oracle_lib as O                                         # noqa: E402
from test_device_terms_gpu import SET_DRIFT, SET_ELEV_A, SET_ELEV_B, SET_VISUAL, _desc, _task   # noqa: E402

G = D.G


def _bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def _kernel(sim, st, done, t, rew=None):
    """wl_test_device_terms on a host state [16, N, 4]: (reward, fired bits, term_log) as numpy."""
    n = sim.num_envs
    d_st = torch.from_numpy(np.ascontiguousarray(st, np.float32)).cuda()
    d_done = torch.from_numpy(np.ascontiguousarray(done, np.uint8)).cuda()
    d_rew = torch.zeros(n, device="cuda") if rew is None else rew.clone()
    d_tl = torch.full((8,), 7.0, device="cuda")
    _lib.check(_lib.lib.wl_test_device_terms(sim._h, C.c_void_p(d_st.data_ptr()), C.c_void_p(d_done.data_ptr()),
                                             C.c_void_p(d_rew.data_ptr()), C.c_void_p(d_tl.data_ptr()), int(t), None),
               "wl_test_device_terms")
    torch.cuda.synchronize()
    return d_rew.cpu().numpy(), sim.device_term_masks.cpu().numpy().copy(), d_tl.cpu().numpy()


@pytest.fixture(scope="module")
def golden_sim():
    spec = D.config()
    return spec, WheeledSim(spec, "cuda:0")


@pytest.mark.parametrize("name", D.STATE_FUNCS)
@pytest.mark.parametrize("role", [D.ROLE_REWARD, D.ROLE_TERMINATION])
def test_placed_golden_states_equal_the_oracle_bit_for_bit(golden_sim, name, role):
    spec, sim = golden_sim
    st = D.state()
    for done_all in (1, 0):
        done = np.full(D.N, done_all, np.uint8)
        for ps in G["p_" + name]:
            terms = D.table(name, ps, spec.cfg, role)
            sim.set_device_terms(terms)
            rew, fired, tl = _kernel(sim, st, done, 0)
            o = O.device_terms(spec.cfg, terms, st, done, 0, vis_map=G["map"])
            tag = f"{name}{tuple(ps)} role {role} done {done_all}"
            assert np.array_equal(_bits(rew), _bits(o["rew"])), tag
            assert np.array_equal(fired, o["fired"]), tag
            assert np.array_equal(_bits(tl), _bits(o["term_log"])), tag
            if role == D.ROLE_REWARD:          # the reward is the value: the reference's branch on every state
                ref = G["f_" + name][list(map(tuple, G["p_" + name])).index(tuple(ps))]
                assert np.array_equal(rew != 0, ref != 0), tag
            else:
                assert np.array_equal(fired & 1, (G["f_" + name][list(map(tuple, G["p_" + name])).index(tuple(ps))] != 0)), tag


def test_placed_bool_is_not_traversable_and_elevation_continuity(golden_sim):
    spec, sim = golden_sim
    st = D.state()
    done = np.ones(D.N, np.uint8)
    for role in (D.ROLE_REWARD, D.ROLE_TIME_OUT):
        terms = D.table("bool_is_not_traversable", [], spec.cfg, role)
        sim.set_device_terms(terms)
        for c, ref in zip(G["t_bool_is_not_traversable"], G["f_bool_is_not_traversable"]):
            rew, fired, tl = _kernel(sim, st, done, int(c))
            o = O.device_terms(spec.cfg, terms, st, done, int(c), vis_map=G["map"])
            assert np.array_equal(_bits(rew), _bits(o["rew"])) and np.array_equal(fired, o["fired"]), c
            assert np.array_equal(_bits(tl), _bits(o["term_log"])), c
            assert np.array_equal((rew if role == D.ROLE_REWARD else fired).astype(np.float32), ref), c
    zs = G["cont_z"]
    m = zs.shape[1]
    cs = D.config(m)
    small = WheeledSim(cs, "cuda:0")
    for j, ps in enumerate(G["p_elevation_continuity"]):
        terms = D.table("elevation_continuity", ps, cs.cfg)
        small.set_device_terms(terms)                 # previous elevations unset before each sequence
        prev = None
        for k in range(zs.shape[0]):
            pos = np.zeros((m, 3), np.float32); pos[:, 2] = zs[k]
            rew, _, _ = _kernel(small, D.state(pos=pos), np.zeros(m, np.uint8), 0)
            o = O.device_terms(cs.cfg, terms, D.state(pos=pos), np.zeros(m, np.uint8), 0, vis_map=G["map"], prev=prev)
            prev = o["prev"]
            assert np.array_equal(_bits(rew), _bits(o["rew"])), (ps, k)
            assert np.array_equal(rew, G["f_elevation_continuity"][j, k]), (ps, k)


@pytest.mark.parametrize("kind,terms", [("elevation", SET_ELEV_A), ("visual", SET_VISUAL)])
def test_test_entry_on_the_stage_a_state_equals_wl_step_terms(kind, terms):
    n = 300
    table = [_desc(key, role, w, p) for _, _, key, role, w, p in terms]
    a, b = WheeledSim(_task(kind, n), "cuda:0"), WheeledSim(_task(kind, n), "cuda:0")
    for s in (a, b):
        s.set_device_terms(table); s.startup(); s.reset(None, 0)
    base = 1000 * int(a.cfg.max_episode_length) - 3 if kind == "visual" else 0
    gen = torch.Generator(device="cuda").manual_seed(3)
    for t in range(base, base + 12):
        act = (torch.rand((n, 2), generator=gen, device="cuda") * 2 - 1).contiguous()
        b.groups.copy_(a.groups)
        rew_b = torch.empty(n, device="cuda"); tbits = torch.empty(n, dtype=torch.uint8, device="cuda")
        _lib.check(_lib.lib.wl_step_stage_a(b._h, C.c_void_p(act.data_ptr()), C.c_void_p(rew_b.data_ptr()),
                                            C.c_void_p(tbits.data_ptr()), t, None), "stage a")
        torch.cuda.synchronize()
        rew2, fired2, tl2 = _kernel(b, b.groups.cpu().numpy(), tbits.cpu().numpy(), t, rew=rew_b)
        tl = torch.zeros(8, device="cuda")
        _, rew, _, _ = a.step_terms(act, t, term_log=tl)
        torch.cuda.synchronize()
        assert np.array_equal(_bits(rew.cpu().numpy()), _bits(rew2)), t
        assert np.array_equal(a.device_term_masks.cpu().numpy(), fired2), t
        assert np.array_equal(_bits(tl.cpu().numpy()), _bits(tl2)), t


TRAJ = [(k, n, s) for k, s in (("elevation", SET_ELEV_A), ("elevation", SET_ELEV_B), ("visual", SET_VISUAL), ("drift", SET_DRIFT))
        for n in (1, 31, 33, 4096)] + [("drift", 4224, SET_DRIFT), ("drift", 4225, SET_DRIFT), ("visual", 8965, SET_VISUAL)]


@pytest.mark.parametrize("kind,n,terms", TRAJ, ids=[f"{k}-{n}-{i % 4 if i < 16 else 'x'}" for i, (k, n, _) in enumerate(TRAJ)])
def test_trajectories_equal_wlo_step_terms_bit_for_bit(kind, n, terms):
    """Every step: obs, reward, done masks, fired bits, term_log, and the state every 10 steps.  Elevation at small N runs
    past every env's time-out; Visual starts 30 steps before bool_is_not_traversable's switch at 1000 episodes."""
    spec = _task(kind, n)
    table = [_desc(key, role, w, p) for _, _, key, role, w, p in terms]
    sim = WheeledSim(spec, "cuda:0")
    orc = O.Oracle(spec.cfg, heightfield=getattr(spec, "heightfield", None), threads=8)
    sim.set_device_terms(table); orc.set_device_terms(table)
    sim.startup(); orc.startup()
    sim.reset(None, 0); orc.reset(None, 0)
    L = int(spec.cfg.max_episode_length)
    steps = (L + 10) if (kind == "elevation" and n <= 64) else (60 if kind == "elevation" else min(L + 10, 80))
    base = 1000 * L - 30 if kind == "visual" else 0
    tl = torch.zeros(8, device="cuda")
    dones = 0
    for k in range(steps):
        t = base + k
        act = sim.synth_actions(t)
        obs, rew, term, trunc = sim.step_terms(act, t, term_log=tl)
        o_obs, o_rew, o_term, o_trunc, o_fired, o_tl = orc.step_terms(act.cpu().numpy(), t)
        torch.cuda.synchronize()
        assert np.array_equal(_bits(rew.cpu().numpy()), _bits(o_rew)), f"reward, step {t}"
        assert np.array_equal(term.cpu().numpy(), o_term) and np.array_equal(trunc.cpu().numpy(), o_trunc), f"dones, step {t}"
        assert np.array_equal(sim.device_term_masks.cpu().numpy(), o_fired), f"fired, step {t}"
        assert np.array_equal(_bits(tl.cpu().numpy()), _bits(o_tl)), f"term_log, step {t}"
        assert np.array_equal(_bits(obs.cpu().numpy()), _bits(o_obs)), f"obs, step {t}"
        dones += int(o_term.sum() + o_trunc.sum())
        if k % 10 == 9 or k == steps - 1:
            assert np.array_equal(_bits(sim.groups.cpu().numpy()[:9]), _bits(orc.export_state()[:9])), f"state, step {t}"
    assert dones > 0 or n < 32


@pytest.mark.parametrize("n", [4097, 4224 + 1, 8965])
def test_episode_log_over_more_than_32_ctas_against_fp64(n):
    """Episode_* of the kernel against an fp64 sum of the kernel's own per-env contributions (every env done: its
    contribution is its reward).  Bound: a tree of m fp32 values is within (ceil(log2 m) + 1) u sum|x| of the exact sum,
    plus the two divisions."""
    spec = D.config(n)
    sim = WheeledSim(spec, "cuda:0")
    rng = np.random.default_rng(n)
    st = np.zeros((D.NUM_GROUPS, n, 4), np.float32)
    st[D.G_QUAT, :, 0] = 1.0
    st[D.G_LINVEL, :, 0] = rng.uniform(-3, 3, n)
    st[D.G_LINVEL, :, 2] = rng.uniform(-1, 1, n)
    dt = D.step_dt(spec.cfg)
    terms = [(1, D.ROLE_REWARD, 1.0 / dt, []), (4, D.ROLE_REWARD, 1.0 / dt, []), (10, D.ROLE_TERMINATION, 0.0, [0.5])]
    sim.set_device_terms(terms)
    done = np.ones(n, np.uint8)
    rew_a, _, _ = _kernel(sim, st, done, 0)
    sim.set_device_terms(terms[:1])
    r1, _, tl1 = _kernel(sim, st, done, 0)
    sim.set_device_terms(terms[1:2])
    r2, _, tl2 = _kernel(sim, st, done, 0)
    sim.set_device_terms(terms)
    _, fired, tl = _kernel(sim, st, done, 0)
    L = float(spec.cfg.episode_length_s)
    lv = int(np.ceil(np.log2(n))) + 1 + 5          # the tree over 128, the lane-strided pass, the butterfly
    for k, x in ((0, r1), (1, r2)):
        exact = x.astype(np.float64).sum() / n / L
        bound = lv * 2 ** -24 * np.abs(x.astype(np.float64)).sum() / n / L + 3 * 2 ** -24 * abs(exact)
        assert abs(float(tl[k]) - exact) <= bound, (k, float(tl[k]), exact, bound)
        assert tl[k] != 0
    assert tl[2] == float(((fired >> 2) & 1).sum()) > 0
    assert np.array_equal(_bits(tl[:2]), _bits([tl1[0], tl2[0]]))
