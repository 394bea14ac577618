"""Device terms (wl_set_device_terms / wl_step_terms, DESIGN.md 6l) on the GPU: each library function against the same
function registered as a Python term through env.staged_step, the no-term and weight-0 baselines against wl_step bit for
bit, captured graphs on device counters against the eager host-counter sequence, elevation_continuity's state, and the
refusals."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import wheeledlab_b200 as wl                                   # noqa: E402
from wheeledlab_b200 import device_terms as dtm                # noqa: E402
from wheeledlab_b200._lib import WlError                       # noqa: E402
from wheeledlab_b200.env import ManagerBasedRLEnv              # noqa: E402
from wheeledlab_b200.sim import WheeledSim                     # noqa: E402


# ---- the library's functions restated as Python terms over the env's state (torch fp32, the reference's expressions) ----
def _vb(env):
    return env.scene["robot"].data.root_lin_vel_b


def _euler(q):
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    roll = torch.atan2(2.0 * (w * x + y * z), 1 - 2 * (x * x + y * y))
    sp = 2.0 * (w * y - z * x)
    pitch = torch.where(sp.abs() >= 1, torch.copysign(torch.full_like(sp, math.pi / 2), sp), torch.asin(sp))
    return roll % (2 * math.pi), pitch % (2 * math.pi)


def _trav(env):
    c, p = env.spec.cfg, env.sim.root_pos_w
    xi = ((p[:, 0] + c.vis_width / 2 + c.vis_row_spacing / 2) / c.vis_row_spacing).to(torch.int64).clamp(0, c.vis_rows - 1)
    yi = ((p[:, 1] + c.vis_height / 2 + c.vis_col_spacing / 2) / c.vis_col_spacing).to(torch.int64).clamp(0, c.vis_cols - 1)
    m = torch.as_tensor(env.spec.traversability, device=p.device).reshape(-1)
    return m[yi * c.vis_cols + xi]


def forward_vel(env):
    return torch.clamp(_vb(env)[:, 0], max=1.2)


def forward_wheel_spin(env):
    return torch.clamp(env.sim.wheel_vel.sum(-1), max=200)


def change_in_elevation(env):
    vz = env.sim.root_lin_vel_w[:, 2]
    return torch.where(vz > 0, vz, torch.zeros_like(vz))


def ascending(env):
    return torch.clamp(env.sim.root_lin_vel_w[:, 2], min=0.0)


def steep_penalty(env, thresh_pitch):
    return torch.clamp(_euler(env.sim.root_quat_w)[1] - thresh_pitch, min=0)


def make_elevation_continuity():
    def elevation_continuity(env, threshold_elev):
        z = env.sim.root_pos_w[:, 2] - 0.19
        if not hasattr(elevation_continuity, "prev"):
            elevation_continuity.prev = z.clone()
        d = z - elevation_continuity.prev
        on = z > threshold_elev
        r = torch.where(on & (d > 0), 50 * d, torch.zeros_like(z)) + torch.where(on & (d < 0), -50 * d, torch.zeros_like(z))
        elevation_continuity.prev = z.clone()
        return r
    return elevation_continuity


def yaw_change_onElev(env, threshold_yaw, threshold_z):
    z = env.sim.root_pos_w[:, 2] - 0.19
    wz = env.scene["robot"].data.root_ang_vel_b[:, 2]
    return torch.where((z > threshold_z) & (abs(wz) > threshold_yaw), 2 * abs(wz) ** 2, torch.zeros_like(wz))


def upright_penalty(env, thresh_deg):
    q = env.sim.root_quat_w
    two_s = 2.0 / (q * q).sum(-1)
    r22 = 1 - two_s * (q[:, 1] * q[:, 1] + q[:, 2] * q[:, 2])
    deg = torch.rad2deg(torch.arccos(r22))
    return torch.where(deg > thresh_deg, deg - thresh_deg, 0.0)


def roll_on_elev(env, z_start, roll_rate_thresh):
    wx = env.scene["robot"].data.root_ang_vel_b[:, 0]
    z = env.sim.root_pos_w[:, 2] - 0.19
    return torch.where((z > z_start) & (abs(wx) > roll_rate_thresh), abs(wx) * 2.0, torch.zeros_like(wx))


def low_vel_penalty(env, min_vel=0.1):
    return torch.where(_vb(env)[:, 0] < min_vel, 1.0, 0.0)


def is_traversable(env):
    return torch.where(_trav(env) != 0, 1.0, 0.0)


def is_traversable_speed_scaled(env):
    return is_traversable(env) * _vb(env)[:, 0]


def vel_rew_trav(env, speed_target_on_trav=1.0, speed_target_on_non_trav=2.0):
    tgt = torch.where(_trav(env) != 0, speed_target_on_trav, speed_target_on_non_trav).to(torch.float32)
    sd = -((torch.norm(_vb(env), dim=-1) - tgt) ** 2) + tgt ** 2
    return torch.where(sd > 0.0, sd, 0.0)


def low_speed_penalty(env, low_speed_thresh=0.3):
    return torch.where(torch.norm(_vb(env), dim=-1) < low_speed_thresh, 1.0, 0.0)


def off_track(env, straight, corner_out_radius):
    p = env.sim.root_pos_w
    x, y = p[:, 0], p[:, 1]
    r2 = corner_out_radius ** 2
    return torch.where(torch.abs(y) < straight, torch.where(torch.abs(x) > corner_out_radius, 1, 0),
                       torch.where(y > 0, torch.where((y - straight) ** 2 + x ** 2 > r2, 1, 0),
                                   torch.where((y + straight) ** 2 + x ** 2 > r2, 1, 0)))


def bool_is_not_traversable(env):
    if env.common_step_counter // env.max_episode_length < 1000:
        return torch.zeros(env.num_envs, device=env.device) == 1
    return _trav(env) == 0


def roll_over(env):
    roll = _euler(env.sim.root_quat_w)[0] - torch.pi
    return torch.logical_and(roll < torch.pi / 2, roll > -torch.pi / 2)


E, V = dtm.ELEVATION, dtm.VISUAL
# (name, python function, library entry, role, weight or time_out, params)
SET_ELEV_A = [
    ("fv", forward_vel, (E, "forward_vel"), "reward", 1.0, {}),
    ("spin", forward_wheel_spin, (E, "forward_wheel_spin"), "reward", 0.01, {}),
    ("dz", change_in_elevation, (E, "change_in_elevation"), "reward", 2.0, {}),
    ("asc", ascending, (E, "ascending"), "reward", 3.0, {}),
    ("steep", steep_penalty, (E, "steep_penalty"), "reward", -1.0, {"thresh_pitch": 0.3}),
    ("cont", "continuity", (E, "elevation_continuity"), "reward", 1.0, {"threshold_elev": 0.05}),
    ("yaw", yaw_change_onElev, (E, "yaw_change_onElev"), "reward", -0.1, {"threshold_yaw": 0.5, "threshold_z": 0.05}),
    ("up", upright_penalty, (E, "upright_penalty"), "reward", -0.01, {"thresh_deg": 10.0}),
]
SET_ELEV_B = [
    ("roll", roll_on_elev, (E, "roll_on_elev"), "reward", -1.0, {"z_start": 0.05, "roll_rate_thresh": 0.3}),
    ("lowv", low_vel_penalty, (E, "low_vel_penalty"), "reward", -1.0, {}),
    ("lows", low_speed_penalty, (V, "low_speed_penalty"), "reward", -0.5, {"low_speed_thresh": 0.3}),
    ("track", off_track, (V, "off_track"), "reward", -1.0, {"straight": 5.0, "corner_out_radius": 15.3}),
    ("flip", roll_over, (V, "roll_over"), "termination", False, {}),
    ("tilt", upright_penalty, (E, "upright_penalty"), "termination", True, {"thresh_deg": 40.0}),
]
SET_VISUAL = [
    ("trav", is_traversable, (V, "is_traversable"), "reward", 1.0, {}),
    ("travv", is_traversable_speed_scaled, (V, "is_traversable_speed_scaled"), "reward", 2.0, {}),
    ("velt", vel_rew_trav, (V, "vel_rew_trav"), "reward", 1.0, {"speed_target_on_trav": 1.5}),
    ("fv", forward_vel, (E, "forward_vel"), "reward", 0.5, {}),
    ("nottrav", bool_is_not_traversable, (V, "bool_is_not_traversable"), "termination", False, {}),
    ("track", off_track, (V, "off_track"), "termination", True, {"straight": 20.0, "corner_out_radius": 60.0}),
]
SET_DRIFT = [
    ("fv", forward_vel, (E, "forward_vel"), "reward", 1.0, {}),
    ("steep", steep_penalty, (E, "steep_penalty"), "reward", -1.0, {"thresh_pitch": 0.05}),
    ("lows", low_speed_penalty, (V, "low_speed_penalty"), "reward", -0.5, {}),
    ("track", off_track, (V, "off_track"), "termination", False, {"straight": 2.0, "corner_out_radius": 4.0}),
]


def _task(kind, n, seed=3):
    if kind == "elevation":
        return wl.elevation_task(num_envs=n, seed=seed)
    if kind == "visual":
        return wl.visual_task(num_envs=n, seed=seed)
    if kind == "visual_cam":
        return wl.visual_task(num_envs=n, seed=seed, camera="aug")
    return wl.drift_task(num_envs=n, seed=seed)


def _device_env(kind, n, terms, seed=3):
    env = ManagerBasedRLEnv(_task(kind, n, seed))
    for name, _, key, role, w, params in terms:
        tk = dtm.resolve(key[1], key[0])
        if role == "reward":
            env.add_device_reward_term(name, tk, w, params)
        else:
            env.add_device_termination_term(name, tk, w, params)
    return env


def _python_env(kind, n, terms, seed=3):
    env = ManagerBasedRLEnv(_task(kind, n, seed))
    cont = make_elevation_continuity()
    for name, fn, _, role, w, params in terms:
        fn = cont if fn == "continuity" else fn
        if role == "reward":
            env.add_reward_term(name, fn, w, params)
        else:
            env.add_termination_term(name, fn, w, params)
    return env


def _desc(key, role, w, params):
    """A wl_term_desc row (kind, role, weight, params) of a table entry."""
    tk = dtm.resolve(key[1], key[0])
    r = dtm.ROLE_REWARD if role == "reward" else (dtm.ROLE_TIME_OUT if w else dtm.ROLE_TERMINATION)
    return (tk.kind, r, w if role == "reward" else 0.0, dtm.param_values(tk, params))


def _actions(n, t, gen):
    return (torch.rand((n, 2), generator=gen, device="cuda") * 2 - 1).contiguous()


@pytest.mark.parametrize("kind,n,terms", [("elevation", 4096, SET_ELEV_A), ("elevation", 4096, SET_ELEV_B),
                                          ("visual", 512, SET_VISUAL), ("visual_cam", 512, SET_VISUAL),
                                          ("drift", 4096, SET_DRIFT), ("elevation", 33, SET_ELEV_B), ("drift", 31, SET_DRIFT)])
def test_device_terms_equal_the_same_functions_as_python_terms(kind, n, terms):
    """Rewards within 2e-5 of the larger of |reward| and sum |weight| * step_dt (the Python side forms v_b with the
    quaternion formula, the kernel with the rotation matrix; sums of 4 in another order), done masks and states equal.  A
    thresholded value may flip at a float tie: such env-steps are counted and bounded.  Elevation runs past the time-out
    of every env at step 200, so elevation_continuity's previous elevation is checked across resets; Visual starts 30 steps
    before bool_is_not_traversable's switch at 1000 episodes."""
    steps = 210 if kind == "elevation" else 150
    dev, py = _device_env(kind, n, terms), _python_env(kind, n, terms)
    if kind.startswith("visual"):
        dev.common_step_counter = py.common_step_counter = 1000 * dev.max_episode_length - 30
    dev.reset(); py.reset()
    gen = torch.Generator(device="cuda").manual_seed(5)
    ties, log_ties, checked, dones = 0, 0, 0, 0
    scale = sum(abs(w) for _, _, _, r, w, _ in terms if r == "reward") * dev.step_dt
    for t in range(steps):
        a = _actions(n, t, gen)
        _, r_d, te_d, tr_d, ex_d = dev.step(a)
        _, r_p, te_p, tr_p, ex_p = py.step(a)
        assert torch.equal(te_d, te_p) and torch.equal(tr_d, tr_p), f"done masks differ at step {t}"
        assert torch.equal(dev.sim.groups[:9], py.sim.groups[:9]), f"states differ at step {t}"
        dones += int((te_d | tr_d).sum())
        tol = 2e-5 * torch.maximum(torch.maximum(r_p.abs(), r_d.abs()), torch.full_like(r_p, scale))
        ties += int(((r_d - r_p).abs() > tol).sum())
        checked += n
        for k in dev.device_log_names:
            x, y = ex_d["log"][k].float(), ex_p["log"][k].float()
            log_ties += int(not torch.allclose(x, y, rtol=1e-4, atol=1e-5 * max(scale, 1.0)))
    assert ties <= max(2, checked // 2000), f"{ties} reward mismatches in {checked} env-steps"
    assert log_ties <= max(1, steps // 50), f"{log_ties} episode-log mismatches"
    assert dones > 0 or n < 64


@pytest.mark.parametrize("kind,n", [("elevation", 1024), ("drift", 4096), ("visual", 512), ("elevation", 1), ("drift", 4097)])
def test_no_terms_and_weight_zero_terms_equal_wl_step(kind, n):
    a, b, c = (WheeledSim(_task(kind, n), "cuda:0") for _ in range(3))
    c.set_device_terms([(1, dtm.ROLE_REWARD, 0.0, []), (4, dtm.ROLE_REWARD, 0.0, [])])
    for s in (a, b, c):
        s.startup(); s.reset(None, 0)
    gen = torch.Generator(device="cuda").manual_seed(2)
    logs = [torch.zeros(16, device="cuda") for _ in range(3)]
    tl = torch.full((8,), 7.0, device="cuda")
    for t in range(300):
        act = _actions(n, t, gen)
        ra = a.step(act, t, log=logs[0])
        rb = b.step_terms(act, t, log=logs[1], term_log=tl)
        rc = c.step_terms(act, t, log=logs[2])
        for x, y, z in zip(ra, rb, rc):
            assert torch.equal(x, y) and torch.equal(x, z), f"step {t}"
    for s in (a, b, c):
        s.flush_log()
    # the episode-log row: counts exact; its sums are float atomics across warps (in wl_step too), so their order and
    # last bits may vary from run to run
    for lg in logs[1:]:
        assert torch.equal(logs[0][8:], lg[8:]) and torch.allclose(logs[0], lg, rtol=1e-5, atol=1e-6)
    assert torch.equal(a.groups, b.groups) and torch.equal(a.groups, c.groups)
    assert torch.equal(tl, torch.full((8,), 7.0, device="cuda"))      # no terms: wl_step itself, the row is not written


@pytest.mark.parametrize("kind,base,terms", [("elevation", 50 * 200 - 6, SET_ELEV_A[:5] + SET_ELEV_B[4:]),
                                             ("visual", 1000 * 50 - 6, SET_VISUAL)])
def test_captured_device_counter_graph_equals_eager_host_counters(kind, base, terms):
    """K = 4 calls on WL_DEVICE_COUNTER_PLUS(k) + wl_advance_counter(K), captured once and replayed 3 times, equal 12 eager
    host-counter calls bit for bit (obs, reward, dones, term_log, state; the built-in log rows' counts), across a curriculum boundary (Elevation:
    episode 50) and bool_is_not_traversable's switch at 1000 episodes (Visual)."""
    n, K, R = 512, 4, 3
    table = [_desc(key, role, w, p) for _, _, key, role, w, p in terms]
    a, b = WheeledSim(_task(kind, n), "cuda:0"), WheeledSim(_task(kind, n), "cuda:0")
    for s in (a, b):
        s.set_device_terms(table); s.startup(); s.reset(None, 0)
    gen = torch.Generator(device="cuda").manual_seed(9)
    acts = [_actions(n, k, gen) for k in range(K * R)]
    first = a.step_terms(acts[0], base - 1)
    b.step_terms(acts[0], base - 1)
    outs = [tuple(torch.empty_like(x) for x in first) for _ in range(K)]
    logs, tls = torch.zeros((K, 16), device="cuda"), torch.zeros((K, 8), device="cuda")
    ref = []
    for t in range(K * R):
        o = a.step_terms(acts[t], base + t, log=(la := torch.zeros(16, device="cuda")), term_log=(ta := torch.zeros(8, device="cuda")))
        ref.append((tuple(x.clone() for x in o), la, ta))
    a.flush_log()
    stream = torch.cuda.Stream(); stream.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    acts_k = [torch.empty_like(acts[0]) for _ in range(K)]
    b.set_step_counter(base)
    with torch.cuda.stream(stream), torch.cuda.graph(g, stream=stream):
        for k in range(K):
            b.step_terms(acts_k[k], WheeledSim.device_counter_plus(k), out=outs[k], log=logs[k], term_log=tls[k])
        b.advance_counter(K)
    torch.cuda.current_stream().wait_stream(stream)
    b.set_step_counter(base)
    for r in range(R):
        for k in range(K):
            acts_k[k].copy_(acts[r * K + k])
        g.replay()
        torch.cuda.synchronize()
        for k in range(K):
            (o, la, ta) = ref[r * K + k]
            for x, y in zip(o, outs[k]):
                assert torch.equal(x, y), f"replay {r} step {k}"
            assert torch.equal(ta, tls[k]), f"term_log, replay {r} step {k}"
            if k < K - 1:      # built-in log row: counts exact, sums are float atomics across warps (order may vary)
                assert torch.equal(la[8:], logs[k][8:]) and torch.allclose(la, logs[k], rtol=1e-5, atol=1e-6), f"log row, replay {r} step {k}"
    b.note_device_counter(base + K * R)
    assert torch.equal(a.groups, b.groups) and torch.equal(a.rew_weight, b.rew_weight)


def test_elevation_continuity_state():
    """The first call sees no change (reward = the built-in reward bit for bit); each handle keeps its own previous
    elevation: a second handle whose first call comes later starts from no change there and then follows the first.
    (That the state survives env resets is checked against the Python function above, past every env's time-out.)"""
    n = 256
    desc = [_desc((E, "elevation_continuity"), "reward", 10.0, {"threshold_elev": -100.0})]   # every z is above it
    base, a, b = (WheeledSim(_task("elevation", n), "cuda:0") for _ in range(3))
    a.set_device_terms(desc); b.set_device_terms(desc)
    for s in (base, a, b):
        s.startup(); s.reset(None, 0)
    gen = torch.Generator(device="cuda").manual_seed(1)
    for t in range(40):
        act = _actions(n, t, gen)
        r0 = base.step(act, t)[1].clone()
        r1 = a.step_terms(act, t)[1].clone()
        r2 = b.step_terms(act, t)[1].clone() if t >= 20 else b.step(act, t)[1].clone()   # wl_step: no terms run
        if t == 0:
            assert torch.equal(r1, r0)
        else:
            assert not torch.equal(r1, r0)
        if t == 20:
            assert torch.equal(r2, r0)
        elif t > 20:
            assert torch.equal(r2, r1)


def test_refusals():
    s = WheeledSim(_task("elevation", 64), "cuda:0")
    with pytest.raises(WlError):                           # map term off the Visual task
        s.set_device_terms([(dtm.resolve("is_traversable", V).kind, 0, 1.0, [])])
    with pytest.raises(WlError):                           # more than 8
        s.set_device_terms([(1, 0, 1.0, [])] * 9)
    with pytest.raises(WlError):
        s.set_device_terms([(5, 0, 1.0, [float("nan")])])
    with pytest.raises(WlError):
        s.set_device_terms([(5, 0, float("inf"), [0.1])])
    with pytest.raises(WlError):
        s.set_device_terms([(99, 0, 1.0, [])])
    d = WheeledSim(wl.drift_task(num_envs=64, seed=1), "cuda:0")
    d.startup(); d.reset(None, 0)
    d.set_device_terms([(1, 0, 1.0, [])])
    buf = torch.zeros(64 * 1024, device="cuda")
    d.set_peer_fanout([16 * 1024])
    with pytest.raises(WlError, match="fan-out"):
        d.step_terms(torch.zeros((64, 2), device="cuda"), 0)
    d.set_peer_fanout([])
    del buf
    env = ManagerBasedRLEnv(_task("elevation", 64))
    env.add_device_reward_term("fv", dtm.resolve("forward_vel", E), 1.0)
    with pytest.raises(NotImplementedError, match="not both"):
        env.add_reward_term("py", forward_vel, 1.0)
    env2 = ManagerBasedRLEnv(_task("elevation", 64))
    env2.add_reward_term("py", forward_vel, 1.0)
    with pytest.raises(NotImplementedError, match="not both"):
        env2.add_device_reward_term("fv", dtm.resolve("forward_vel", E), 1.0)
    with pytest.raises(NotImplementedError, match="library"):
        env.add_device_reward_term("lam", lambda e: e.sim.root_pos_w[:, 2], 1.0)


def test_get_term_and_log_of_device_terminations():
    env = _device_env("elevation", 2048, SET_ELEV_B)
    env.reset()
    gen = torch.Generator(device="cuda").manual_seed(4)
    fired_any = False
    for t in range(120):
        _, _, te, tr, ex = env.step(_actions(2048, t, gen))
        m_flip, m_tilt = env.termination_manager.get_term("flip"), env.termination_manager.get_term("tilt")
        assert bool((m_flip & ~te).sum() == 0) and bool((m_tilt & ~tr).sum() == 0)
        assert int(ex["log"]["Episode_Termination/flip"].item()) == int(m_flip.sum())
        assert int(ex["log"]["Episode_Termination/tilt"].item()) == int(m_tilt.sum())
        fired_any |= bool(m_flip.any() | m_tilt.any())
        env.termination_manager.get_term("time_out")
    assert fired_any


def test_elevation_continuity_previous_elevation_survives_env_resets():
    """Every env terminates at every step (an always-firing off_track), so every step starts from a reset state: the
    reward still measures the change from the PRE-reset elevation of the step before, as the reference's function
    attribute does (the Python function keeps it too).  A kernel that reset it with the env would give no change."""
    n, steps = 1024, 12
    always = ("all", lambda e, **kw: torch.ones(e.num_envs, dtype=torch.bool, device=e.device), (V, "off_track"), "termination", False,
              {"straight": 1e6, "corner_out_radius": -1.0})
    terms = [("cont", "continuity", (E, "elevation_continuity"), "reward", 1.0, {"threshold_elev": -100.0}), always]
    dev, py = _device_env("elevation", n, terms), _python_env("elevation", n, terms)
    dev.reset(); py.reset()
    gen = torch.Generator(device="cuda").manual_seed(6)
    base = ManagerBasedRLEnv(_task("elevation", n)); base.reset()
    for t in range(steps):
        a = _actions(n, t, gen)
        _, r_d, te, _, _ = dev.step(a)
        _, r_p, _, _, _ = py.step(a)
        _, r_0, _, _, _ = base.step(a)
        assert bool(te.all())
        assert torch.allclose(r_d, r_p, rtol=1e-5, atol=1e-6), f"step {t}"
        if t == 0:
            assert torch.equal(r_d, r_0)
        else:                               # the change from the pre-reset elevation is large for every env
            assert bool(((r_d - r_0).abs() > 1e-3).float().mean() > 0.9), f"step {t}"


def test_get_term_of_a_built_in_term_is_its_own_mask_with_device_terms():
    """Drift records no per-term bits without device terms; with them, get_term of a built-in term is still that term's
    own mask, not the union with the device terms."""
    n = 512
    env = _device_env("drift", n, [("all", None, (V, "off_track"), "termination", False, {"straight": 1e6, "corner_out_radius": -1.0})])
    ref = ManagerBasedRLEnv(_task("drift", n))
    env.reset(); ref.reset()
    gen = torch.Generator(device="cuda").manual_seed(3)
    a = _actions(n, 0, gen)
    _, _, te, tr, _ = env.step(a)
    _, _, te_r, tr_r, _ = ref.step(a)
    tm = env.termination_manager
    assert bool(te.all()) and bool(tm.get_term("all").all())
    assert torch.equal(tm.get_term("out_of_bounds"), te_r) and torch.equal(tm.get_term("time_out"), tr_r)
    assert not bool(tm.get_term("out_of_bounds").all())
