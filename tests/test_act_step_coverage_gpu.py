"""The fused act step (wl_act_step_quad_kernel<TASK>: actor-critic, Gaussian draw and env step in one launch) against the
CPU oracle and an exact reference of its policy side, across the tasks, step specs, launch geometries and placements the
Drift-family act step runs.

Env side, every step, bit for bit: the oracle is stepped with the kernel's sampled actions and its obs, reward and done
masks must equal the kernel's; the episode-log counts exactly and its sums (float atomics) to rtol 1e-5; the full state and
the reward weights at the end.  The helpers come from test_duo_coverage_gpu.

Policy side, every step:
- The noise exactly: z0, z1 rebuilt per env from Philox (RNG_POLICY), u01 / u01_open, the oracle's det_log / det_sincos
  (bit-equal to the device's, test_oracle_cpu / test_gpu_parity) and fp32 sqrt and products (-fmad=false); then the action
  must be the correctly rounded fmaf(std, z, mean) bit for bit.
- Mean and value against an fp64 evaluation of the blob, with the PPO tests' criterion: per-tensor relative error within
  max(K x torch fp32's error, 1e-6) (K below).
- log_prob against the fp64 formula on the kernel's own action and mean, within a bound written out from the __logf error
  bound and the fp32 roundings of the kernel's expression.

Two policies: std (0.7, 1.3), and std (0.05, 3.0) with every weight scaled x3 (most pre-activations far from 0, many
negative; std outside [0.5, 2], where __logf's bound is relative)."""
import math
from fractions import Fraction

import numpy as np
import pytest

import oracle_lib as O
import test_duo_coverage_gpu as duo

torch = pytest.importorskip("torch")

DEV = "cuda:0"
RNG_POLICY = 9                                              # wl_device.cuh RNG stream of the policy noise
U24 = np.float32(5.9604644775390625e-08)                    # 2^-24 (u01 / u01_open)
TWO_PI_F = np.float32(6.28318530717958647692)
LOG_2PI_F = np.float32(1.8378770664093453)                  # the kernel's fp32 constant for 2 * 0.5 log(2 pi)
# The act step's ELU is __expf(x) - 1 (ex2.approx: ~2 ulp of exp(x), so ~2^-22 absolute near x = 0 where torch's expm1f
# is accurate to an ulp of the result); the PPO kernel's is expm1f.  K bounds the act step's mean / value error relative to
# torch fp32's own error against fp64.  Measured on an H100 SXM over this file's matrix (largest per-step ratio of a run,
# printed by each test): mean 7.06x (blind Visual, weights x3), value 4.27x, at N >= 31; 13.1x / 7.9x at N = 1, where
# torch fp32's error on two numbers is ~1e-8 and the 1e-6 floor decides.  K = 10 keeps ~40 % above the worst.
ELU_K = 10.0
FLOOR = 1e-6

POLICIES = {"std0.7_1.3": ((0.7, 1.3), 1.0), "std0.05_3.0_w3": ((0.05, 3.0), 3.0)}


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _policy(name, obs_dim, seed=0):
    from wheeledlab_b200.policy import pack_actor_critic
    std, scale = POLICIES[name]
    torch.manual_seed(seed)
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(obs_dim, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(),
                                         torch.nn.Linear(64, out)).to(DEV)
    actor, critic = mk(2), mk(1)
    with torch.no_grad():
        for p in list(actor.parameters()) + list(critic.parameters()):
            p.mul_(scale)
    return pack_actor_critic(actor, critic, torch.tensor(std), obs_dim, DEV)


def _forward(blob, obs_dim, obs, dtype):
    """(mean [N, 2], value [N]) of the blob's networks in `dtype` (torch ops: the fp32 form is torch fp32's error)."""
    from wheeledlab_b200.policy import actor_critic_state_dict
    sd = {k: v.to(dtype) for k, v in actor_critic_state_dict(blob, obs_dim).items()}
    outs = []
    for net in ("actor", "critic"):
        x = obs.to(dtype)
        for k in (0, 2, 4):
            x = torch.nn.functional.linear(x, sd[f"{net}.{k}.weight"], sd[f"{net}.{k}.bias"])
            if k < 4:
                x = torch.nn.functional.elu(x)
        outs.append(x)
    return outs[0], outs[1].squeeze(-1)


def _err(x, ref):
    return ((x.double() - ref.double()).norm() / ref.double().norm()).item()


# ---- the exact policy-side references ----------------------------------------------------------------------------------
def _noise(seed, offset, n, t):
    """box_muller(philox(seed, env_id_offset + i, t, RNG_POLICY, 0)) as the device computes it, in fp32."""
    r = O.philox(seed, offset, t, RNG_POLICY, 0, n)
    u1 = ((r[:, 0] >> 8) + 1).astype(np.float32) * U24     # u01_open
    u2 = (r[:, 1] >> 8).astype(np.float32) * U24           # u01
    rad = np.sqrt(np.float32(-2.0) * O.detmath(4, u1))     # det_log; IEEE sqrt
    ang = TWO_PI_F * u2
    return rad * O.detmath(1, ang), rad * O.detmath(0, ang)   # r cos, r sin


def _fma32(a, b, c):
    """fp32 fmaf(a, b, c), correctly rounded.  a*b is exact in fp64; the sum rounds once to fp64, and rounding that to fp32
    is wrong only where the fp64 value is exactly halfway between two floats: those are settled on exact rationals."""
    a, b, c = (np.asarray(x, np.float32) for x in (a, b, c))
    x = a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)
    f = x.astype(np.float32)
    fd = f.astype(np.float64)
    other = np.nextafter(f, np.where(x > fd, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
    tie = (x != fd) & (2.0 * x == fd + other.astype(np.float64))
    for i in np.flatnonzero(tie):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        mid = (Fraction(float(f[i])) + Fraction(float(other[i]))) / 2
        if exact == mid:                                    # a true tie: the even neighbour
            f[i] = f[i] if (f.view(np.uint32)[i] & 1) == 0 else other[i]
        elif (exact > mid) == (float(other[i]) > float(f[i])):
            f[i] = other[i]
    return f


def _ulp32(x):
    x = np.abs(np.asarray(x, np.float32))
    return (np.nextafter(x, np.float32(np.inf)) - x).astype(np.float64)


def _logf_bound(s):
    """CUDA __logf: max absolute error 2^-21.41 for x in [0.5, 2], otherwise max 3 ulp (CUDA C++ Programming Guide,
    intrinsic functions)."""
    s = np.float32(s)
    return 2.0 ** -21.41 if 0.5 <= s <= 2.0 else 3.0 * float(_ulp32(np.log(s)))


def _log_prob_tol(z0, z1, a, std):
    """|kernel log_prob - fp64 formula on the kernel's action and mean| bound per env:
    - __logf of each std (_logf_bound);
    - the kernel's fp32 expression -0.5f*(z0*z0 + z1*z1) - logf(s0) - logf(s1) - C: six rounded operations (the 0.5 is
      exact), each within 2^-24 of a partial result bounded by M = 0.5 (z0^2 + z1^2) + |log s0| + |log s1| + C, and C's own
      rounding, 2^-24 C;
    - the formula reads z back as (a - m) / s, and a = fmaf(s, z, m) rounded: |a - m - s z| <= 2^-24 |a|, so
      |0.5 ((a - m)/s)^2 - 0.5 z^2| <= |z| d / s + d^2 / (2 s^2) with d = 2^-24 |a|."""
    e = 2.0 ** -24
    s0, s1 = (float(np.float32(x)) for x in std)
    z0, z1 = z0.astype(np.float64), z1.astype(np.float64)
    C = float(LOG_2PI_F)
    M = 0.5 * (z0 * z0 + z1 * z1) + abs(math.log(s0)) + abs(math.log(s1)) + C
    tol = _logf_bound(s0) + _logf_bound(s1) + 6 * e * M + e * C
    for z, s, ak in ((z0, s0, a[:, 0]), (z1, s1, a[:, 1])):
        d = e * np.abs(ak.astype(np.float64))
        tol = tol + np.abs(z) * d / s + d * d / (2 * s * s)
    return tol


class Ratios:
    """Largest mean / value error of the act step relative to torch fp32's error over a run (printed; see ELU_K)."""

    def __init__(self):
        self.mean = self.value = 0.0

    def report(self, what):
        print(f"{what}: act-step err / torch-fp32 err: mean {self.mean:.3g}, value {self.value:.3g}")


def _check_policy(blob, std, obs_dim, seed, offset, obs_in, act, mean, lp, val, t, what, ratios):
    n = obs_in.shape[0]
    a, m, l = act.cpu().numpy(), mean.cpu().numpy(), lp.cpu().numpy()
    z0, z1 = _noise(seed, offset, n, t)
    s = np.asarray(std, np.float32)
    for k, z in ((0, z0), (1, z1)):
        want = _fma32(np.full(n, s[k]), z, m[:, k])
        bad = np.flatnonzero(_bits(a[:, k]) != _bits(want))
        assert bad.size == 0, f"{what}: action[{k}] is not fmaf(std, z, mean) at envs {bad[:8]} ({a[bad[:4], k]} vs {want[bad[:4]]})"
    with torch.no_grad():
        m64, v64 = _forward(blob, obs_dim, obs_in, torch.float64)
        m32, v32 = _forward(blob, obs_dim, obs_in, torch.float32)
    for name, got, ref, t32 in (("mean", mean, m64, m32), ("value", val, v64, v32)):
        ek, et = _err(got, ref), _err(t32, ref)
        setattr(ratios, name, max(getattr(ratios, name), ek / max(et, 1e-30)))
        assert ek <= max(ELU_K * et, FLOOR), f"{what}: {name} err {ek:.3g} vs torch fp32 {et:.3g} (K = {ELU_K})"
    a64, m64k, s64 = a.astype(np.float64), m.astype(np.float64), s.astype(np.float64)
    ref = (-0.5 * (((a64 - m64k) / s64) ** 2).sum(1) - np.log(s64).sum() - math.log(2 * math.pi))
    tol = _log_prob_tol(z0, z1, a, std)
    bad = np.flatnonzero(np.abs(l.astype(np.float64) - ref) > tol)
    assert bad.size == 0, f"{what}: log_prob off the fp64 formula at envs {bad[:8]}: {l[bad[:4]]} vs {ref[bad[:4]]} (tol {tol[bad[:4]]})"


# ---- harness ---------------------------------------------------------------------------------------------------------
def _act_run(spec, steps, policy, record=False, check_oracle=True):
    """`steps` act steps from obs = observe(0): each step's policy side against the references and its env side against the
    oracle (stepped with the kernel's actions).  Returns the per-step outputs when `record`."""
    import wheeledlab_b200 as wl
    from wheeledlab_b200.policy import act_step
    cfg = spec.cfg
    n, seed, offset = int(cfg.num_envs), int(cfg.seed), int(cfg.env_id_offset)
    sim = wl.WheeledSim(spec, DEV); sim.startup(); sim.reset(None, 0)
    orc = None
    if check_oracle:
        orc = O.Oracle(cfg, heightfield=spec.heightfield, threads=8); orc.startup(); orc.reset(None, 0)
    D = sim.obs_dim
    blob = _policy(policy, D)
    std = POLICIES[policy][0]
    f32 = lambda *s: torch.empty(s, dtype=torch.float32, device=DEV)
    u8 = lambda *s: torch.empty(s, dtype=torch.uint8, device=DEV)
    w0 = sim.rew_weight.cpu().numpy().copy()
    obs_in = sim.observe(0, 0)
    ratios, n_done, rec = Ratios(), 0, []
    what0 = f"{spec.name} n={n} {policy}"
    for t in range(steps):
        what = f"{what0} step {t}"
        act, mean, lp, val = f32(n, 2), f32(n, 2), f32(n), f32(n)
        out = (f32(n, D), f32(n), u8(n), u8(n))
        log = torch.zeros(16, device=DEV)
        act_step(sim, obs_in, blob, act, mean, lp, val, out, log, t)
        sim.flush_log()
        _check_policy(blob, std, D, seed, offset, obs_in, act, mean, lp, val, t, what, ratios)
        if orc is not None:
            n_done += duo._check_step(out, orc.step(act.cpu().numpy(), t), what)
            duo._check_log(log.cpu().numpy(), orc.log(), what)
        if record:
            rec.append([x.cpu().numpy() for x in (act, mean, lp, val) + out])
        obs_in = out[0]
    ratios.report(what0)
    if orc is not None:
        assert np.array_equal(_bits(sim.groups.cpu().numpy()), _bits(orc.export_state())), f"{what0}: final state differs"
        w = sim.rew_weight.cpu().numpy()
        assert np.array_equal(_bits(w), _bits(orc.weights())), f"{what0}: reward weights differ"
        if cfg.term_enable:
            assert n_done > 0, f"{what0}: trajectory too short to exercise the auto-reset"
        else:                                                  # (the lowered play cfg has no termination term at all)
            assert n_done == 0, f"{what0}: an env reset with every termination term off"
        if cfg.curr_n > 0 and steps > cfg.max_episode_length:
            assert not np.array_equal(w, w0), f"{what0}: the curriculum boundary did not move the weights"
    return rec


def _episode_run(spec, policy):
    """Episodes of the spec's own length plus 20 steps: every env reaches its time-out and the reset path runs."""
    _act_run(spec, int(spec.cfg.max_episode_length) + 20, policy)


# ---- tasks and step specs --------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("policy", list(POLICIES))
@pytest.mark.parametrize("name", duo.SPECIALISED)
def test_act_step_on_drift_family_tasks(name, policy):
    """drift (RWD), hound_4wd, f1tenth_drift and the lowered reference Drift / Drift-play / F1Tenth cfgs (the play cfg turns
    every termination term off: no env may reset)."""
    _need_gpu()
    _episode_run(duo._spec(name, 333), policy)


@pytest.mark.gpu
@pytest.mark.parametrize("policy", list(POLICIES))
@pytest.mark.parametrize("deviation", list(duo.DEVIATIONS))
@pytest.mark.parametrize("base", ["drift", "hound_4wd"])
def test_act_step_on_step_spec_deviations(base, deviation, policy):
    _need_gpu()
    _episode_run(duo._spec(base, 333, deviation=deviation), policy)


@pytest.mark.gpu
@pytest.mark.parametrize("policy", list(POLICIES))
@pytest.mark.parametrize("randomize", [False, True])
def test_act_step_on_blind_visual_task(randomize, policy):
    """wl_act_step_quad_kernel<WL_TASK_VISUAL>: visual_task without a camera observes 8 proprioceptive floats."""
    _need_gpu()
    import wheeledlab_b200 as wl
    spec = wl.visual_task(num_envs=333, seed=11, randomize=randomize)
    assert spec.obs_dim == 8
    _episode_run(spec, policy)


# ---- launch geometry -------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("policy", list(POLICIES))
@pytest.mark.parametrize("n", [1, 7, 31, 32, 33, 4095, 4097, 33793])
def test_act_step_launch_geometry(n, policy):
    """32 envs per CTA plus the janitor CTA: one partial CTA, exactly one CTA, one env over, ragged last CTAs, and a size
    past the duo kernel's largest.  25-step episodes (test_duo_coverage_gpu._geometry_spec) over 40 steps."""
    _need_gpu()
    _act_run(duo._geometry_spec(n), 40, policy)


# ---- placement -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("policy", list(POLICIES))
def test_act_step_outputs_do_not_depend_on_the_cta_slot(policy):
    """Shards of 333 and 667 envs (env_id_offset 0 and 333) against one run of 1000: every output of every step equal bit
    for bit, the policy side included (the shards' envs sit in other CTA slots and lanes)."""
    _need_gpu()

    def spec(n, offset):
        s = duo._geometry_spec(n)
        s.cfg.env_id_offset = offset
        return s

    full = _act_run(spec(1000, 0), 40, policy, record=True)
    parts = [(0, _act_run(spec(333, 0), 40, policy, record=True, check_oracle=False)),
             (333, _act_run(spec(667, 333), 40, policy, record=True, check_oracle=False))]
    names = ("actions", "mean", "log_prob", "value", "obs", "reward", "terminated", "truncated")
    for t in range(40):
        for lo, rec in parts:
            for k, name in enumerate(names):
                a, b = full[t][k][lo:lo + rec[t][k].shape[0]], rec[t][k]
                assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), f"step {t}: {name} of envs {lo}.. differs in the shard"


# ---- the device counter across episode boundaries --------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["drift", "hound_4wd"])
def test_rollout_graph_crosses_episode_boundaries_on_the_device_counter(name):
    """FusedPolicyRollout (T = 64 act steps on the device counter, one graph) replayed 9 times: steps 0..575 cross the
    curriculum boundaries at t = 250 and 500 inside replays.  The oracle replays slab.actions; every slab row, every
    roll.logs row and the reward weights after each replay must match, and the policy side of every row the references."""
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.policy import FusedPolicyRollout
    T, reps, policy = 64, 9, "std0.7_1.3"
    spec = duo._spec(name, 333)
    cfg = spec.cfg
    assert int(cfg.max_episode_length) == 250
    sim = wl.WheeledSim(spec, DEV); sim.startup(); sim.reset(None, 0)
    orc = O.Oracle(cfg, threads=8); orc.startup(); orc.reset(None, 0)
    blob = _policy(policy, 14)
    roll = FusedPolicyRollout(sim, blob, T).capture(0)
    w_prev, moved, n_done, ratios = sim.rew_weight.cpu().numpy().copy(), 0, 0, Ratios()
    for it in range(reps):
        slab = roll.run()
        sim.flush_log()
        torch.cuda.synchronize()
        for k in range(T):
            t = it * T + k
            what = f"{name} replay {it} row {k} (t={t})"
            _check_policy(blob, POLICIES[policy][0], 14, int(cfg.seed), 0, slab.obs_in[k], slab.actions[k], roll.pol.mean[k],
                          roll.pol.log_prob[k], roll.pol.values[k], t, what, ratios)
            got = (slab.obs[k], slab.rewards[k], slab.terminated[k], slab.truncated[k])
            n_done += duo._check_step(got, orc.step(slab.actions[k].cpu().numpy(), t), what)
            duo._check_log(roll.logs[k].cpu().numpy(), orc.log(), what)
        w = sim.rew_weight.cpu().numpy()
        assert np.array_equal(_bits(w), _bits(orc.weights())), f"{name}: reward weights differ after replay {it}"
        moved += int(not np.array_equal(w, w_prev))
        w_prev = w.copy()
    ratios.report(f"{name} rollout graph")
    assert moved == 2, f"{name}: the weights moved in {moved} replays, not at t = 250 and 500"
    assert n_done > 0
    assert np.array_equal(_bits(sim.groups.cpu().numpy()), _bits(orc.export_state())), f"{name}: final state differs"
