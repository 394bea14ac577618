"""Playing a trained policy: wl_actor_mean, wl_act_infer_step, FusedPolicyRollout(deterministic=True), the runner's
get_inference_policy and tools/play_policy.py.

The contract: what is played is what was trained.  For the same observation rows and blob, bit for bit:
- wl_actor_mean(ELU) equals the mean wl_act_step stores (drift, hound_4wd, f1tenth_drift, blind Visual);
- wl_actor_mean(ReLU) equals the mean wl_policy_act stores (Elevation 689, camera Visual 3208);
- the actions of wl_act_infer_step equal wl_actor_mean(ELU) of its obs_in.
Both under the two policies of test_act_step_coverage_gpu.  At the other widths wl_actor_mean is checked against an fp64
evaluation of the blob with the existing criteria (ELU_K, RELU_K relative to torch fp32's error, floor 1e-6; pooled over
steps below 32 rows).  The env side of wl_act_infer_step and of wl_actor_mean -> wl_step is bit-exact against the oracle
stepped with the kernel's actions, with the helpers of test_duo_coverage_gpu / test_elev_visual_coverage_gpu."""
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import oracle_lib as O
import test_act_step_coverage_gpu as ac
import test_duo_coverage_gpu as duo
import test_elev_visual_coverage_gpu as ev
import test_policy_wide_gpu as pw

torch = pytest.importorskip("torch")

DEV = "cuda:0"
ROOT = Path(__file__).resolve().parent.parent


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _eq(a, b, what):
    assert torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)), what


def _relu_blob(D, policy):
    std, scale = ac.POLICIES[policy]
    return pw.relu_policy(D, std=std, scale=scale)


def _actor64(blob, D, obs, activation, dtype):
    from wheeledlab_b200.policy import actor_critic_state_dict
    sd = {k: v.to(dtype) for k, v in actor_critic_state_dict(blob, D).items()}
    f = torch.nn.functional.elu if activation == "elu" else torch.relu
    x = obs.to(dtype)
    for k in (0, 2, 4):
        x = torch.nn.functional.linear(x, sd[f"actor.{k}.weight"], sd[f"actor.{k}.bias"])
        if k < 4:
            x = f(x)
    return x


# ---- 1. the contract -------------------------------------------------------------------------------------------------
def _narrow_spec(task, n):
    import wheeledlab_b200 as wl
    if task == "blind_visual":
        return wl.visual_task(num_envs=n, seed=11)
    spec = duo._spec(task, n, seed=3)
    spec.cfg.max_episode_length = 25
    return spec


@pytest.mark.gpu
@pytest.mark.parametrize("policy", list(ac.POLICIES))
@pytest.mark.parametrize("n", [1, 31, 33, 4096, 33793])
@pytest.mark.parametrize("task", ["drift", "hound_4wd", "f1tenth_drift", "blind_visual"])
def test_actor_mean_equals_act_step_mean_and_infer_step_actions(task, n, policy):
    """Two sims of one spec: wl_act_step on one, wl_act_infer_step on the other, 6 steps.  actor_mean of each step's obs_in
    must equal the act step's stored mean and the inference step's actions, bit for bit."""
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.policy import act_infer_step, act_step, actor_mean
    spec = _narrow_spec(task, n)
    sims = [wl.WheeledSim(_narrow_spec(task, n), DEV) for _ in range(2)]
    for s in sims:
        s.startup(); s.reset(None, 0)
    D = sims[0].obs_dim
    blob = ac._policy(policy, D)
    f32 = lambda *s: torch.empty(s, dtype=torch.float32, device=DEV)
    u8 = lambda *s: torch.empty(s, dtype=torch.uint8, device=DEV)
    obs_a, obs_b = sims[0].observe(0, 0), sims[1].observe(0, 0)
    for t in range(6):
        what = f"{spec.name} n={n} {policy} step {t}"
        act, mean, lp, val = f32(n, 2), f32(n, 2), f32(n), f32(n)
        out_a = (f32(n, D), f32(n), u8(n), u8(n))
        act_step(sims[0], obs_a, blob, act, mean, lp, val, out_a, None, t)
        _eq(actor_mean(blob, D, obs_a, "elu"), mean, f"{what}: actor_mean != wl_act_step's mean")
        act_b = f32(n, 2)
        out_b = (f32(n, D), f32(n), u8(n), u8(n))
        act_infer_step(sims[1], obs_b, blob, act_b, out_b, None, t)
        _eq(actor_mean(blob, D, obs_b, "elu"), act_b, f"{what}: wl_act_infer_step's actions != actor_mean of its obs_in")
        obs_a, obs_b = out_a[0], out_b[0]


@pytest.mark.gpu
@pytest.mark.parametrize("policy", list(ac.POLICIES))
@pytest.mark.parametrize("case", ["elevation1", "elevation33", "elevation1000", "visual64"])
def test_actor_mean_equals_policy_act_mean(case, policy):
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.policy import actor_mean, policy_act
    if case.startswith("elevation"):
        spec = pw._elevation(int(case[len("elevation"):]))
    else:
        spec = wl.visual_task(num_envs=64, seed=9, camera="aug")
    sim = wl.WheeledSim(spec, DEV); sim.startup(); sim.reset(None, 0)
    n, D = sim.num_envs, sim.obs_dim
    assert D in (689, 3208)
    blob = _relu_blob(D, policy)
    f32 = lambda *s: torch.empty(s, dtype=torch.float32, device=DEV)
    obs = sim.observe(0, 0)
    for t in range(4):
        act, mean, lp, val = f32(n, 2), f32(n, 2), f32(n), f32(n)
        policy_act(sim, obs, blob, act, mean, lp, val, t)
        _eq(actor_mean(blob, D, obs, "relu"), mean, f"{case} {policy} step {t}: actor_mean != wl_policy_act's mean")
        obs = sim.step(act, t)[0]


# ---- 2. accuracy at other widths -------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 5, 31, 33, 100, 1000])
@pytest.mark.parametrize("D", [1, 3, 5, 31, 37, 65, 100, 129, 4096])
def test_actor_mean_relu_accuracy_at_other_widths(D, n):
    _need_gpu()
    from wheeledlab_b200.policy import actor_mean
    for policy in ac.POLICIES:
        blob = _relu_blob(D, policy)
        got, r64, r32 = [], [], []
        for s in range(8 if n < pw.POOL_BELOW else 1):
            g = torch.Generator(device=DEV).manual_seed(s)
            obs = torch.randn((n, D), generator=g, device=DEV) * 2.0
            got.append(actor_mean(blob, D, obs, "relu"))
            r64.append(_actor64(blob, D, obs, "relu", torch.float64))
            r32.append(_actor64(blob, D, obs, "relu", torch.float32))
        ek, et = ac._err(torch.cat(got), torch.cat(r64)), ac._err(torch.cat(r32), torch.cat(r64))
        assert ek <= max(pw.RELU_K * et, pw.FLOOR), f"D={D} n={n} {policy}: err {ek:.3g} vs torch fp32 {et:.3g}"


@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 2, 3, 4, 5, 8, 13, 16])
def test_actor_mean_elu_accuracy_at_every_width(D):
    _need_gpu()
    from wheeledlab_b200.policy import actor_mean
    for policy in ac.POLICIES:
        blob = ac._policy(policy, D)
        obs = torch.randn((1000, D), generator=torch.Generator(device=DEV).manual_seed(D), device=DEV) * 2.0
        r64 = _actor64(blob, D, obs, "elu", torch.float64)
        ek, et = ac._err(actor_mean(blob, D, obs, "elu"), r64), ac._err(_actor64(blob, D, obs, "elu", torch.float32), r64)
        assert ek <= max(ac.ELU_K * et, ac.FLOOR), f"D={D} {policy}: err {ek:.3g} vs torch fp32 {et:.3g}"


@pytest.mark.gpu
def test_actor_mean_refuses_device_tensors_it_cannot_take():
    _need_gpu()
    from wheeledlab_b200.policy import actor_mean, blob_layout
    blob = torch.zeros(blob_layout(14)[1], device=DEV)
    obs = torch.zeros(8, 14, device=DEV)
    with pytest.raises(ValueError, match="obs"):
        actor_mean(blob, 14, obs.cpu())
    with pytest.raises(ValueError, match="obs"):
        actor_mean(blob, 14, obs.double())
    with pytest.raises(ValueError, match="obs"):
        actor_mean(blob, 14, torch.zeros(14, 8, device=DEV).t())
    with pytest.raises(ValueError, match="blob"):
        actor_mean(blob[:-4], 14, obs)
    with pytest.raises(ValueError, match="out"):
        actor_mean(blob, 14, obs, out=torch.zeros(8, 3, device=DEV))
    with pytest.raises(ValueError, match="activation"):
        actor_mean(blob, 14, obs, "tanh")


# ---- 3. the env side against the oracle ------------------------------------------------------------------------------
def _infer_run(spec, steps, policy, record=False, check_oracle=True):
    """`steps` wl_act_infer_steps from observe(0): actions equal actor_mean(obs_in); obs / reward / dones, the episode log
    and the final state against the oracle stepped with the kernel's actions."""
    import wheeledlab_b200 as wl
    from wheeledlab_b200.policy import act_infer_step, actor_mean
    cfg = spec.cfg
    n = int(cfg.num_envs)
    sim = wl.WheeledSim(spec, DEV); sim.startup(); sim.reset(None, 0)
    orc = None
    if check_oracle:
        orc = O.Oracle(cfg, heightfield=spec.heightfield, threads=8); orc.startup(); orc.reset(None, 0)
    D = sim.obs_dim
    blob = ac._policy(policy, D)
    f32 = lambda *s: torch.empty(s, dtype=torch.float32, device=DEV)
    u8 = lambda *s: torch.empty(s, dtype=torch.uint8, device=DEV)
    obs_in, n_done, rec = sim.observe(0, 0), 0, []
    what0 = f"{spec.name} n={n} {policy}"
    for t in range(steps):
        what = f"{what0} step {t}"
        act = f32(n, 2)
        out = (f32(n, D), f32(n), u8(n), u8(n))
        log = torch.zeros(16, device=DEV)
        act_infer_step(sim, obs_in, blob, act, out, log, t)
        sim.flush_log()
        _eq(actor_mean(blob, D, obs_in, "elu"), act, f"{what}: actions != actor_mean(obs_in)")
        if orc is not None:
            n_done += duo._check_step(out, orc.step(act.cpu().numpy(), t), what)
            duo._check_log(log.cpu().numpy(), orc.log(), what)
        if record:
            rec.append([x.cpu().numpy() for x in (act,) + out])
        obs_in = out[0]
    if orc is not None:
        assert np.array_equal(_bits(sim.groups.cpu().numpy()), _bits(orc.export_state())), f"{what0}: final state differs"
        assert np.array_equal(_bits(sim.rew_weight.cpu().numpy()), _bits(orc.weights())), f"{what0}: reward weights differ"
        if cfg.term_enable:
            assert n_done > 0, f"{what0}: trajectory too short to exercise the auto-reset"
        else:
            assert n_done == 0, f"{what0}: an env reset with every termination term off"
    return rec


@pytest.mark.gpu
@pytest.mark.parametrize("policy", list(ac.POLICIES))
@pytest.mark.parametrize("name", duo.SPECIALISED)
def test_infer_step_on_drift_family_tasks_and_reference_cfgs(name, policy):
    """drift, hound_4wd, f1tenth_drift and the lowered Drift / Drift-play / F1Tenth reference cfgs, one episode + 20 steps."""
    _need_gpu()
    spec = duo._spec(name, 333)
    _infer_run(spec, int(spec.cfg.max_episode_length) + 20, policy)


@pytest.mark.gpu
@pytest.mark.parametrize("deviation", list(duo.DEVIATIONS))
def test_infer_step_on_step_spec_deviations(deviation):
    _need_gpu()
    spec = duo._spec("drift", 333, deviation=deviation)
    spec.cfg.max_episode_length = 25
    _infer_run(spec, 40, "std0.05_3.0_w3")


@pytest.mark.gpu
def test_infer_step_outputs_do_not_depend_on_the_cta_slot():
    """Shards of 333 and 667 envs (env_id_offset 0 and 333) against one run of 1000: every output of every step equal."""
    _need_gpu()

    def spec(n, offset):
        s = duo._geometry_spec(n)
        s.cfg.env_id_offset = offset
        return s

    full = _infer_run(spec(1000, 0), 40, "std0.7_1.3", record=True)
    parts = [(0, _infer_run(spec(333, 0), 40, "std0.7_1.3", record=True, check_oracle=False)),
             (333, _infer_run(spec(667, 333), 40, "std0.7_1.3", record=True, check_oracle=False))]
    for t in range(40):
        for lo, rec in parts:
            for k, name in enumerate(("actions", "obs", "reward", "terminated", "truncated")):
                a, b = full[t][k][lo:lo + rec[t][k].shape[0]], rec[t][k]
                assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), f"step {t}: {name} of envs {lo}.. differs in the shard"


@pytest.mark.gpu
def test_deterministic_graph_crosses_episode_boundaries_on_the_device_counter():
    """FusedPolicyRollout(deterministic=True), T = 64, replayed 9 times: steps 0..575 cross the curriculum boundaries at
    t = 250 and 500.  The oracle replays slab.actions; every slab row and log row, and the weights after each replay."""
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.policy import FusedPolicyRollout, actor_mean
    T, reps = 64, 9
    spec = duo._spec("drift", 333)
    sim = wl.WheeledSim(spec, DEV); sim.startup(); sim.reset(None, 0)
    orc = O.Oracle(spec.cfg, threads=8); orc.startup(); orc.reset(None, 0)
    blob = ac._policy("std0.7_1.3", 14)
    roll = FusedPolicyRollout(sim, blob, T, deterministic=True).capture(0)
    assert not hasattr(roll.slab, "values") and roll.pol is None
    w_prev, moved, n_done = sim.rew_weight.cpu().numpy().copy(), 0, 0
    for it in range(reps):
        slab = roll.run()
        sim.flush_log()
        torch.cuda.synchronize()
        for k in range(T):
            t = it * T + k
            what = f"replay {it} row {k} (t={t})"
            _eq(actor_mean(blob, 14, slab.obs_in[k], "elu"), slab.actions[k], f"{what}: actions != actor_mean(obs_in)")
            got = (slab.obs[k], slab.rewards[k], slab.terminated[k], slab.truncated[k])
            n_done += duo._check_step(got, orc.step(slab.actions[k].cpu().numpy(), t), what)
            duo._check_log(roll.logs[k].cpu().numpy(), orc.log(), what)
        w = sim.rew_weight.cpu().numpy()
        assert np.array_equal(_bits(w), _bits(orc.weights())), f"reward weights differ after replay {it}"
        moved += int(not np.array_equal(w, w_prev))
        w_prev = w.copy()
    assert moved == 2 and n_done > 0
    assert np.array_equal(_bits(sim.groups.cpu().numpy()), _bits(orc.export_state()))


@pytest.mark.gpu
@pytest.mark.parametrize("name,n,steps", [("elevation", 333, 40), ("Isaac-MushrElevationRL-v0.play.ref", 333, 205),
                                          ("Isaac-MushrVisualRL-v0.play.ref", 64, 55)])
def test_actor_mean_then_step_matches_the_oracle_on_relu_tasks(name, n, steps):
    """wl_actor_mean -> wl_step, the deterministic ReLU step, against the oracle: obs, reward, dones and the episode log."""
    _need_gpu()
    from wheeledlab_b200.policy import actor_mean
    spec = pw._elevation(n) if name == "elevation" else ev._ref_spec(name, n)
    sim, orc = ev._pair(spec)
    D = sim.obs_dim
    blob = _relu_blob(D, "std0.7_1.3")
    obs, n_done = sim.observe(0, 0), 0
    for t in range(steps):
        what = f"{name} step {t}"
        act = actor_mean(blob, D, obs, "relu")
        log = torch.empty(16, device=DEV)
        out = sim.step(act, t, log=log)
        sim.flush_log()
        n_done += ev._check_step(spec, out, orc.step(act.cpu().numpy(), t), what)
        ev._check_log(spec, log, orc.log(), what)
        obs = out[0]
    ev._check_end(sim, orc, name)
    ev._check_resets(spec, n_done, name)


# ---- 4. the graph and the reference's loop ---------------------------------------------------------------------------
def _agent(activation, steps=16):
    from wheeledlab_b200.runs import agent_cfg
    return agent_cfg(activation, steps=steps)


@pytest.mark.gpu
@pytest.mark.parametrize("task,n", [("Isaac-MushrDriftRL-v0", 333), ("Isaac-MushrElevationRL-v0", 258)])
def test_deterministic_graph_equals_eager_sequence_and_the_reference_play_loop(task, n):
    """Two envs of one seed, a runner on each with the same weights.  Env A replays a deterministic graph (T = 16, 3 times);
    env B runs play_policy.py's loop as written, from the graph's first observation: actions = policy(obs);
    obs, ... = env.step(actions).  Every action and observation equal bit for bit."""
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    from wheeledlab_b200.policy import FusedPolicyRollout
    from wheeledlab_b200.runs import task_activation
    act = task_activation(task)
    envs = [wl.make(task, device=DEV, num_envs=n, seed=5) for _ in range(2)]
    torch.manual_seed(0)
    runner = FusedOnPolicyRunner(envs[0], _agent(act), device=DEV)
    runner_b = FusedOnPolicyRunner(envs[1], _agent(act), device=DEV)
    runner_b.blob.copy_(runner.blob)
    for e in envs:
        e.reset()
    T, reps = 16, 3
    roll = FusedPolicyRollout(envs[0].sim, runner.blob, T, activation=act, deterministic=True).capture(envs[0].common_step_counter)
    env = envs[1]
    policy = runner_b.get_inference_policy(device=env.unwrapped.device)
    obs = roll.obs0.clone()
    for it in range(reps):
        slab = roll.run()
        envs[0].common_step_counter += T
        for k in range(T):
            with torch.inference_mode():
                actions = policy(obs)
                obs_dict, _, _, _, _ = env.step(actions)
                obs = obs_dict["policy"]
            _eq(slab.actions[k], actions, f"{task} replay {it} step {k}: actions differ from the play loop")
            _eq(slab.obs[k], obs, f"{task} replay {it} step {k}: observations differ from the play loop")


# ---- 5. the runner ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_inference_policy_reads_the_live_blob_and_checks_the_device():
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    from wheeledlab_b200.policy import actor_mean
    env = wl.make("Isaac-MushrDriftRL-v0", device=DEV, num_envs=256, seed=1)
    torch.manual_seed(0)
    runner = FusedOnPolicyRunner(env, _agent("elu"), device=DEV)
    policy = runner.get_inference_policy()
    with pytest.raises(ValueError, match="device"):
        runner.get_inference_policy(device="cpu")
    obs = torch.randn(256, 14, device=DEV)
    before = policy(obs)
    assert before.shape == (256, 2) and policy(obs).data_ptr() != before.data_ptr()
    runner.learn(2)
    after = policy(obs)
    assert not torch.equal(before, after), "learn() did not reach the inference policy"
    _eq(after, actor_mean(runner.blob, 14, obs, "elu"), "the inference policy is not actor_mean of the runner's blob")
    out = torch.empty(256, 2, device=DEV)
    assert policy(obs, out=out) is out


def _play_args(**kw):
    sys.path.insert(0, str(ROOT / "tools"))
    import play_policy
    args = play_policy.parser().parse_args([])
    for k, v in kw.items():
        setattr(args, k, v)
    return play_policy, args


@pytest.mark.gpu
@pytest.mark.parametrize("source", ["runner", "torch_actor_critic"])
def test_checkpoints_play_within_the_fp64_criterion_of_the_torch_actor(source, tmp_path):
    """A checkpoint saved by the runner, and one built from a torch ActorCritic-shaped state dict (actor.0/2/4, critic.0/2/4,
    std), both play: the actions are the torch actor's within ELU_K x torch fp32's error of fp64, and the saved rollouts
    file loads with recording.load_rollouts as [steps, N, D] / [steps, N, 2]."""
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    from wheeledlab_b200.policy import actor_critic_state_dict
    from wheeledlab_b200.recording import load_rollouts, save_slab
    n, steps = 64, 12
    path = tmp_path / "model_3.pt"
    torch.manual_seed(3)
    if source == "runner":
        env = wl.make("Isaac-MushrDriftRL-v0", device=DEV, num_envs=n, seed=2)
        r = FusedOnPolicyRunner(env, _agent("elu", 8), device=DEV)
        r.learn(1)
        r.save(str(path))
        sd = actor_critic_state_dict(r.blob, 14)
        env.close()
    else:
        mk = lambda out: torch.nn.Sequential(torch.nn.Linear(14, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(),
                                             torch.nn.Linear(64, out))
        actor, critic = mk(2), mk(1)
        sd = {**{f"actor.{k}": v for k, v in actor.state_dict().items()}, **{f"critic.{k}": v for k, v in critic.state_dict().items()},
              "std": torch.full((2,), 0.8)}
        torch.save({"model_state_dict": sd, "iter": 3, "infos": None}, str(path))
    play_policy, args = _play_args(task="Isaac-MushrDriftRL-v0", policy_path=str(path), log_dir=str(tmp_path / "pb"), num_envs=n, seed=4)
    rcfg = play_policy.resolve(args)
    runner, roll, stats = play_policy.play(rcfg, steps)
    slab = roll.slab
    actor = torch.nn.Sequential(torch.nn.Linear(14, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(), torch.nn.Linear(64, 2))
    actor.load_state_dict({k[len("actor."):]: v.cpu() for k, v in sd.items() if k.startswith("actor.")})
    obs = slab.obs_in.reshape(-1, 14).cpu()
    with torch.no_grad():
        r64, r32 = actor.double()(obs.double()), actor.float()(obs)
    got = slab.actions.reshape(-1, 2).cpu()
    ek, et = ac._err(got, r64), ac._err(r32, r64)
    assert ek <= max(ac.ELU_K * et, ac.FLOOR), f"{source}: played actions err {ek:.3g} vs torch fp32 {et:.3g}"
    f = save_slab(rcfg["playback_dir"], "t", slab)
    data = load_rollouts(f)
    assert tuple(data["observations"].shape) == (steps, n, 14) and tuple(data["actions"].shape) == (steps, n, 2)


# ---- 6. the script ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_play_policy_script_writes_the_rollouts_of_the_in_process_graph(tmp_path):
    """A Drift run directory (64 envs: run.json + models/model_0.pt and model_1.pt) played for 20 steps by
    tools/play_policy.py in a subprocess: the rollouts file equals the in-process graph's bit for bit."""
    _need_gpu()
    import wheeledlab_b200 as wl
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    from wheeledlab_b200.recording import load_rollouts
    from wheeledlab_b200.runs import save_run_config
    run, n, steps = tmp_path / "run", 64, 20
    env = wl.make("Isaac-MushrDriftRL-v0", device=DEV, num_envs=n, seed=6)
    torch.manual_seed(6)
    agent = _agent("elu", 8)
    agent["save_interval"] = 1
    r = FusedOnPolicyRunner(env, agent, log_dir=str(run), device=DEV)
    save_run_config(str(run), "Isaac-MushrDriftRL-v0", n, 6, agent)
    r.learn(2)
    env.close()
    assert sorted(os.listdir(run / "models")) == ["model_0.pt", "model_1.pt"]
    cmd = [sys.executable, str(ROOT / "tools" / "play_policy.py"), "-p", str(run), "--steps", str(steps), "-sd", "--play-name", "t"]
    p = subprocess.run(cmd, capture_output=True, text=True, cwd=str(tmp_path), timeout=600)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "Saved episode data" in p.stdout and "Episodes finished" in p.stdout
    got = load_rollouts(str(run / "playback" / "t-rollouts.pt"))
    play_policy, args = _play_args(run_path=str(run))
    rcfg = play_policy.resolve(args)
    assert rcfg["policy_path"].endswith("model_1.pt") and rcfg["num_envs"] == n
    _, roll, _ = play_policy.play(rcfg, steps)
    _eq(got["observations"], roll.slab.obs.cpu(), "the script's observations differ from the in-process graph")
    _eq(got["actions"], roll.slab.actions.cpu(), "the script's actions differ from the in-process graph")
