"""wl_policy_act (the wide ReLU actor-critic of the Elevation / Visual tasks) against exact references and the CPU oracle.

Policy side, every step, with the criteria of test_act_step_coverage_gpu:
- the noise rebuilt exactly from Philox, and the action equal to the correctly rounded fmaf(std, z, mean) bit for bit;
- mean and value against an fp64 evaluation of the blob within max(K x torch fp32's error, 1e-6) (RELU_K below);
- log_prob against the fp64 formula within the __logf-derived bound.
Env side (Elevation): the oracle is stepped with the kernel's actions; obs, reward and done masks bit for bit every step.

The policy kernel reads the width from the sim, so the widths it is run at here are the tasks' own: 8 (blind Visual),
14 (Drift), 689 (Elevation) and 3208 (Visual with the camera).  Its layer 1 (wide_layer1) is shared with the PPO forward
kernel, which test_ppo_wide_gpu runs at the odd widths 1, 3, 5, 31, 65."""
import numpy as np
import pytest

import oracle_lib as O
import test_act_step_coverage_gpu as ac
import test_duo_coverage_gpu as duo

torch = pytest.importorskip("torch")

DEV = "cuda:0"
# Mean / value error of wl_policy_act relative to torch fp32's own error against fp64.  ReLU is exact, so the kernel's
# error is only its FP32 FFMA sums (per 32-input chunk, then across chunks).  Measured on an H100 80GB HBM3 over this file
# (largest per-step ratio of a run, printed by each test): mean 1.32x, value 1.46x; K = 4 is the PPO tests' factor.
# Below 32 envs a step has too few numbers for a relative error (one value that cancels to near 0 gave 8x at N = 1), so
# there the criterion is applied to the whole run's [steps, N] tensors.
RELU_K = 4.0
POOL_BELOW = 32
FLOOR = 1e-6
STD = (0.7, 1.3)


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def relu_policy(obs_dim, std=STD, scale=1.0, seed=0):
    from wheeledlab_b200.policy import pack_actor_critic
    torch.manual_seed(seed)
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(obs_dim, 64), torch.nn.ReLU(), torch.nn.Linear(64, 64), torch.nn.ReLU(),
                                         torch.nn.Linear(64, out)).to(DEV)
    actor, critic = mk(2), mk(1)
    with torch.no_grad():
        for p in list(actor.parameters()) + list(critic.parameters()):
            p.mul_(scale)
    return pack_actor_critic(actor, critic, torch.tensor(std), obs_dim, DEV)


def _forward(blob, obs_dim, obs, dtype):
    from wheeledlab_b200.policy import actor_critic_state_dict
    sd = {k: v.to(dtype) for k, v in actor_critic_state_dict(blob, obs_dim).items()}
    outs = []
    for net in ("actor", "critic"):
        x = obs.to(dtype)
        for k in (0, 2, 4):
            x = torch.nn.functional.linear(x, sd[f"{net}.{k}.weight"], sd[f"{net}.{k}.bias"])
            if k < 4:
                x = torch.relu(x)
        outs.append(x)
    return outs[0], outs[1].squeeze(-1)


def _check_err(name, got, ref, t32, what, ratios):
    ek, et = ac._err(got, ref), ac._err(t32, ref)
    setattr(ratios, name, max(getattr(ratios, name), ek / max(et, 1e-30)))
    assert ek <= max(RELU_K * et, FLOOR), f"{what}: {name} err {ek:.3g} vs torch fp32 {et:.3g} (K = {RELU_K})"


def check_policy(blob, std, obs_dim, seed, offset, obs_in, act, mean, lp, val, t, what, ratios, pool=None):
    """pool: a list to collect (name, got, fp64, torch fp32) in instead of checking mean / value per step."""
    n = obs_in.shape[0]
    a, m, l = act.cpu().numpy(), mean.cpu().numpy(), lp.cpu().numpy()
    z0, z1 = ac._noise(seed, offset, n, t)
    s = np.asarray(std, np.float32)
    for k, z in ((0, z0), (1, z1)):
        want = ac._fma32(np.full(n, s[k]), z, m[:, k])
        bad = np.flatnonzero(ac._bits(a[:, k]) != ac._bits(want))
        assert bad.size == 0, f"{what}: action[{k}] is not fmaf(std, z, mean) at envs {bad[:8]}"
    with torch.no_grad():
        m64, v64 = _forward(blob, obs_dim, obs_in, torch.float64)
        m32, v32 = _forward(blob, obs_dim, obs_in, torch.float32)
    for name, got, ref, t32 in (("mean", mean, m64, m32), ("value", val, v64, v32)):
        if pool is None:
            _check_err(name, got, ref, t32, what, ratios)
        else:
            pool.append((name, got.clone(), ref, t32))
    a64, m64k, s64 = a.astype(np.float64), m.astype(np.float64), s.astype(np.float64)
    ref = (-0.5 * (((a64 - m64k) / s64) ** 2).sum(1) - np.log(s64).sum() - np.log(2 * np.pi))
    tol = ac._log_prob_tol(z0, z1, a, std)
    bad = np.flatnonzero(np.abs(l.astype(np.float64) - ref) > tol)
    assert bad.size == 0, f"{what}: log_prob off the fp64 formula at envs {bad[:8]}"


def _run(spec, steps, std=STD, scale=1.0, check_oracle=True, record=False, obs_fn=None):
    """`steps` of (wl_policy_act, wl_step) from observe(0); obs_fn(t, obs) may replace the policy input (synthetic rows)."""
    import wheeledlab_b200 as wl
    from wheeledlab_b200.policy import policy_act
    cfg = spec.cfg
    n, seed, offset = int(cfg.num_envs), int(cfg.seed), int(cfg.env_id_offset)
    sim = wl.WheeledSim(spec, DEV); sim.startup(); sim.reset(None, 0)
    orc = None
    if check_oracle:
        orc = O.Oracle(cfg, heightfield=spec.heightfield, threads=8); orc.startup(); orc.reset(None, 0)
    D = sim.obs_dim
    blob = relu_policy(D, std, scale)
    f32 = lambda *s: torch.empty(s, dtype=torch.float32, device=DEV)
    obs_in = sim.observe(0, 0)
    ratios, n_done, rec = ac.Ratios(), 0, []
    pool = [] if n < POOL_BELOW else None
    what0 = f"{spec.name} n={n} D={D}"
    for t in range(steps):
        what = f"{what0} step {t}"
        if obs_fn is not None:
            obs_in = obs_fn(t, obs_in)
        act, mean, lp, val = f32(n, 2), f32(n, 2), f32(n), f32(n)
        policy_act(sim, obs_in, blob, act, mean, lp, val, t)
        out = sim.step(act, t)
        check_policy(blob, std, D, seed, offset, obs_in, act, mean, lp, val, t, what, ratios, pool)
        if orc is not None:
            n_done += duo._check_step(out, orc.step(act.cpu().numpy(), t), what)
        if record:
            rec.append([x.cpu().numpy() for x in (act, mean, lp, val) + tuple(out)])
        obs_in = out[0]
    if pool is not None:
        for name in ("mean", "value"):
            got, ref, t32 = (torch.stack([p[k] for p in pool if p[0] == name]) for k in (1, 2, 3))
            _check_err(name, got, ref, t32, f"{what0}, all steps", ratios)
    ratios.report(what0)
    if orc is not None:
        assert n_done > 0, f"{what0}: trajectory too short to exercise the auto-reset"
    return rec


def _elevation(n, seed=5, offset=0):
    import wheeledlab_b200 as wl
    spec = wl.elevation_task(num_envs=n, seed=seed, env_id_offset=offset)
    spec.cfg.max_episode_length = 25                         # resets within the run
    return spec


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 33, 4096])
def test_policy_act_drives_elevation_against_the_oracle(n):
    _need_gpu()
    assert _elevation(8).obs_dim == 689
    _run(_elevation(n), 60)


@pytest.mark.gpu
def test_policy_act_with_large_weights_and_extreme_std():
    """std (0.05, 3.0) and every weight x3: most pre-activations far from 0 and many negative."""
    _need_gpu()
    _run(_elevation(333), 30, std=(0.05, 3.0), scale=3.0)


@pytest.mark.gpu
@pytest.mark.parametrize("task", ["blind_visual", "drift"])
def test_policy_act_on_narrow_tasks_with_synthetic_observations(task):
    """The Drift sim (14) and blind Visual (8) as noise keys, fed N(0, 2) synthetic rows: one partial K chunk."""
    _need_gpu()
    import wheeledlab_b200 as wl
    spec = wl.visual_task(num_envs=100, seed=3) if task == "blind_visual" else duo._geometry_spec(100)

    def obs_fn(t, obs):
        g = torch.Generator(device=DEV).manual_seed(t)
        return torch.randn(obs.shape, generator=g, device=DEV) * 2.0

    _run(spec, 5, check_oracle=False, obs_fn=obs_fn)


@pytest.mark.gpu
def test_policy_act_on_camera_visual():
    """Visual with the camera: obs_dim 3208 (101 K chunks), N = 64, against the oracle."""
    _need_gpu()
    import wheeledlab_b200 as wl
    spec = wl.visual_task(num_envs=64, seed=9, camera="aug")
    assert spec.obs_dim == 3208
    spec.cfg.max_episode_length = 10
    _run(spec, 15)


@pytest.mark.gpu
def test_policy_act_outputs_do_not_depend_on_the_cta_slot():
    """Elevation shards of 333 and 667 envs (env_id_offset 0 and 333) against one run of 1000: every output bit for bit."""
    _need_gpu()
    full = _run(_elevation(1000), 30, check_oracle=False, record=True)
    parts = [(0, _run(_elevation(333), 30, check_oracle=False, record=True)),
             (333, _run(_elevation(667, offset=333), 30, check_oracle=False, record=True))]
    names = ("actions", "mean", "log_prob", "value", "obs", "reward", "terminated", "truncated")
    for t in range(30):
        for lo, rec in parts:
            for k, name in enumerate(names):
                a, b = full[t][k][lo:lo + rec[t][k].shape[0]], rec[t][k]
                assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), f"step {t}: {name} of envs {lo}.. differs in the shard"


@pytest.mark.gpu
def test_relu_rollout_graph_equals_the_eager_sequence():
    """FusedPolicyRollout(activation="relu"), T = 16, captured once and replayed 4 times on the device counter, against the
    same 64 (wl_policy_act, wl_step) pairs issued eagerly from a second sim: every slab row bit for bit."""
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.policy import FusedPolicyRollout, policy_act
    T, reps, n = 16, 4, 258
    spec = _elevation(n, seed=21)
    blob = relu_policy(689)
    sim = wl.WheeledSim(spec, DEV); sim.startup(); sim.reset(None, 0)
    roll = FusedPolicyRollout(sim, blob, T, activation="relu").capture(0)
    ref = wl.WheeledSim(_elevation(n, seed=21), DEV); ref.startup(); ref.reset(None, 0)
    obs_in = ref.observe(0, 0)
    f32 = lambda *s: torch.empty(s, dtype=torch.float32, device=DEV)
    for it in range(reps):
        slab = roll.run()
        torch.cuda.synchronize()
        for k in range(T):
            t = it * T + k
            act, mean, lp, val = f32(n, 2), f32(n, 2), f32(n), f32(n)
            policy_act(ref, obs_in, blob, act, mean, lp, val, t)
            out = ref.step(act, t)
            pairs = ((slab.obs_in[k], obs_in), (slab.actions[k], act), (roll.pol.mean[k], mean), (roll.pol.log_prob[k], lp),
                     (roll.pol.values[k], val), (slab.obs[k], out[0]), (slab.rewards[k], out[1]), (slab.terminated[k], out[2]),
                     (slab.truncated[k], out[3]))
            for j, (g, w) in enumerate(pairs):
                assert torch.equal(g.view(torch.uint8), w.view(torch.uint8)), f"replay {it} row {k}: field {j} differs"
            obs_in = out[0]


@pytest.mark.gpu
def test_act_step_still_refuses_elevation_and_policy_act_checks_arguments():
    _need_gpu()
    import ctypes as C
    import wheeledlab_b200 as wl
    from wheeledlab_b200._lib import WlPolicyOut, lib
    sim = wl.WheeledSim(_elevation(32), DEV); sim.startup(); sim.reset(None, 0)
    x = torch.zeros(64, 689, device=DEV)
    po = WlPolicyOut(x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr())
    assert lib.wl_policy_act(sim._h, None, C.c_void_p(x.data_ptr()), po, 0, None) == -1
    assert lib.wl_policy_act(sim._h, C.c_void_p(x.data_ptr()), C.c_void_p(x.data_ptr() + 4), po, 0, None) == -1
    assert b"16-byte" in lib.wl_last_error()
