"""The data-parallel PPO update refuses malformed calls before anything is launched: wl_ppo_update_dp's own checks through
the C-ABI with pointers that are never dereferenced, and the Python layers (update_local_ranks, FusedOnPolicyRunner's
data-parallel set-up) with the library replaced by a stub that fails the test if a launch is reached."""
import ctypes as C
from types import SimpleNamespace

import pytest
import torch


class _NoLaunch:
    """Stands in for the library: any call fails the test (an argument check is missing if one is reached)."""

    def __getattr__(self, name):
        def launch(*args, **kwargs):
            pytest.fail(f"{name} was reached: the call should have been refused before any launch")
        return launch


D = 14
FAKE = 1 << 20                                     # 256-byte aligned, never dereferenced


def _call(R=2, ex=None, n_local=2, ranks=(0, 1), activation=0, obs_dim=D, per_rank=None, null=None, batch_null=None, epochs=1):
    import wheeledlab_b200 as wl
    from wheeledlab_b200._lib import WlPpoBatch, WlPpoParams
    p = WlPpoParams(obs_dim, 4096, epochs, 4, 0.2, 1.0, 0.005, 1.0, 0.01, 1, 1, 0)
    ex = ex if ex is not None else [FAKE + (r << 16) for r in range(R)]
    exa = (C.c_void_p * max(1, len(ex)))(*ex)
    nl = max(1, n_local)
    arr = lambda k: (C.c_void_p * nl)(*[FAKE + (k << 12) + (l << 24) for l in range(nl)])
    arrays = {k: arr(i) for i, k in enumerate(("blob", "m", "v", "state", "ws"))}
    if per_rank is not None:
        arrays[per_rank] = (C.c_void_p * nl)(*([None] + [FAKE] * (nl - 1)))
    fields = [FAKE] * 8
    if batch_null is not None:
        fields[batch_null] = None
    batches = (WlPpoBatch * nl)(*[WlPpoBatch(*fields) for _ in range(nl)])
    rk = (C.c_int32 * max(1, len(ranks)))(*ranks)
    args = [C.byref(p), activation, R, exa, n_local, rk, batches, arrays["blob"], arrays["m"], arrays["v"], arrays["state"],
            arrays["ws"], 1 << 30, None]
    if null is not None:
        args[null] = None
    rc = wl.lib.wl_ppo_update_dp(*args)
    return rc, wl.lib.wl_last_error().decode()


REFUSALS = [
    ("n_ranks 0", dict(R=0, ex=[FAKE], n_local=1, ranks=(0,)), "n_ranks must be in 1..8"),
    ("n_ranks 9", dict(R=9), "n_ranks must be in 1..8"),
    ("null exchange array", dict(null=3), "null d_exchange"),
    ("null exchange buffer", dict(ex=[FAKE, None]), "exchange buffer 1 is null or not 256-byte aligned"),
    ("misaligned exchange buffer", dict(ex=[FAKE + 16, FAKE + (1 << 16)]), "exchange buffer 0 is null or not 256-byte aligned"),
    ("n_local 0", dict(n_local=0, ranks=(0,)), "n_local must be in 1..n_ranks"),
    ("n_local > n_ranks", dict(n_local=3, ranks=(0, 1, 1)), "n_local must be in 1..n_ranks"),
    ("null local ranks", dict(null=5), "local_ranks non-null"),
    ("local rank out of range", dict(ranks=(0, 2)), "local rank index 2 out of 0..n_ranks-1"),
    ("negative local rank", dict(ranks=(-1, 1)), "local rank index -1"),
    ("repeated local rank", dict(ranks=(1, 1)), "local rank 1 given twice"),
    ("null params", dict(null=0), "null params"),
    ("unknown activation", dict(activation=2), "activation must be"),
    ("null batches", dict(null=6), "null per-rank array"),
    ("null blob array", dict(null=7), "null per-rank array"),
    ("null workspace array", dict(null=11), "null per-rank array"),
    ("null blob of a rank", dict(per_rank="blob"), "null d_blob"),
    ("null state of a rank", dict(per_rank="state"), "null d_blob / d_adam_m / d_adam_v / d_state"),
    ("null batch array", dict(batch_null=7), "null array in batch"),
    ("no epochs", dict(epochs=0), "num_learning_epochs must be >= 1"),
]


@pytest.mark.parametrize("kw,match", [c[1:] for c in REFUSALS], ids=[c[0] for c in REFUSALS])
def test_update_dp_refuses_before_any_launch(kw, match):
    rc, msg = _call(**kw)
    assert rc != 0 and msg.startswith("wl_ppo_update_dp") and match in msg, msg


def test_update_dp_refuses_elu_beyond_obs_dim_16_and_host_exchange_buffers():
    rc, msg = _call(obs_dim=17)
    assert rc != 0 and "obs_dim > 16" in msg, msg
    host = torch.zeros(4096, dtype=torch.uint8)                         # 256-byte aligned host memory: not a device buffer
    rc, msg = _call(ex=[host.data_ptr() + (-host.data_ptr() % 256), FAKE])
    assert rc != 0 and "local exchange buffer 0 is not device memory" in msg, msg


def test_exchange_bytes_holds_a_header_and_two_reduced_rows():
    import wheeledlab_b200 as wl
    from wheeledlab_b200.policy import blob_layout
    for obs_dim in (1, 14, 689, 3208, 4096):
        rowlen = (blob_layout(obs_dim)[1] + 3 + 3) & ~3
        assert wl.lib.wl_ppo_dp_exchange_bytes(obs_dim) == 256 + 2 * ((4 * rowlen + 255) // 256 * 256)
    for bad in (0, -1, 4097):
        assert wl.lib.wl_ppo_dp_exchange_bytes(bad) == 0 and b"obs_dim" in wl.lib.wl_last_error()


def _replicas(R=2, activation="elu", obs_dim=D, cfg=None):
    from wheeledlab_b200.learner import FusedPPO, PPOConfig, PPOExchange
    from wheeledlab_b200.policy import pack_actor_critic
    torch.manual_seed(0)
    act = torch.nn.ELU if activation == "elu" else torch.nn.ReLU
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(obs_dim, 64), act(), torch.nn.Linear(64, 64), act(), torch.nn.Linear(64, out))
    blob = pack_actor_critic(mk(2), mk(1), torch.ones(2), obs_dim, "cpu")
    return [FusedPPO(blob.clone(), obs_dim, cfg or PPOConfig(), activation, exchange=ex) for ex in PPOExchange.local(R, obs_dim, "cpu")]


def _inputs(n=64):
    slab = SimpleNamespace(obs_in=torch.zeros(n, D), actions=torch.zeros(n, 2), values=torch.zeros(n), log_prob=torch.zeros(n),
                           mean=torch.zeros(n, 2))
    return slab, torch.zeros(n), torch.zeros(n), torch.arange(n)


def test_update_local_ranks_refuses_mismatched_replicas(monkeypatch):
    from wheeledlab_b200 import learner
    from wheeledlab_b200.learner import FusedPPO, PPOConfig
    a, b = _replicas()
    c, d = _replicas()
    lone = FusedPPO(a.blob.clone(), D, PPOConfig())
    x = _inputs()
    monkeypatch.setattr(learner, "lib", _NoLaunch())
    with pytest.raises(ValueError, match="one .* per replica"):
        learner.update_local_ranks([a, b], [x])
    with pytest.raises(ValueError, match="same rank buffers"):
        learner.update_local_ranks([a, d], [x, x])
    with pytest.raises(ValueError, match="same rank buffers"):
        learner.update_local_ranks([a, lone], [x, x])
    with pytest.raises(ValueError, match="same rank"):
        learner.update_local_ranks([a, a], [x, x])
    with pytest.raises(ValueError, match="updates all 2 ranks together"):
        learner.update_local_ranks([a], [x])
    with pytest.raises(ValueError, match="update_local_ranks"):
        a.update(*x)
    b.cfg = PPOConfig(num_mini_batches=2)
    with pytest.raises(ValueError, match="share the network, obs_dim and PPOConfig"):
        learner.update_local_ranks([a, b], [x, x])


AGENT = {"num_steps_per_env": 8, "save_interval": 1, "empirical_normalization": False,
         "policy": {"class_name": "ActorCritic", "activation": "elu", "actor_hidden_dims": [64, 64], "critic_hidden_dims": [64, 64],
                    "init_noise_std": 1.0},
         "algorithm": {"class_name": "PPO"}}


def _env(device="cuda:1", offset=64, n=64, **extra):
    return SimpleNamespace(sim=SimpleNamespace(device=device, num_envs=n, obs_dim=D, cfg=SimpleNamespace(env_id_offset=offset)), **extra)


def _runner(monkeypatch, env, agent=AGENT, device="cuda:1", world=2, rank=1, local=1, initialised=False, uuids=None):
    import torch.distributed as dist
    from wheeledlab_b200 import learner
    monkeypatch.setattr(learner, "lib", _NoLaunch())
    monkeypatch.setattr(dist, "init_process_group", lambda *a, **k: pytest.fail("init_process_group reached"))
    monkeypatch.setenv("WORLD_SIZE", str(world)); monkeypatch.setenv("RANK", str(rank)); monkeypatch.setenv("LOCAL_RANK", str(local))
    if initialised:
        monkeypatch.setattr(dist, "is_initialized", lambda: True)
        monkeypatch.setattr(dist, "get_world_size", lambda group=None: world)
        monkeypatch.setattr(dist, "get_rank", lambda group=None: rank)
        monkeypatch.setattr(dist, "all_gather_object", lambda out, obj, group=None: out.__setitem__(slice(None), uuids))
        monkeypatch.setattr(torch.cuda, "set_device", lambda d: None)
        monkeypatch.setattr(torch.cuda, "get_device_properties", lambda d: SimpleNamespace(uuid=uuids[rank]))
    return learner.FusedOnPolicyRunner(env, agent, device=device)


def test_runner_refuses_a_device_other_than_local_rank(monkeypatch):
    with pytest.raises(ValueError, match=r"not cuda:1 \(LOCAL_RANK\)"):
        _runner(monkeypatch, _env(device="cuda:0"), device="cuda:0")


def test_runner_refuses_an_env_shard_that_repeats_another_ranks_envs(monkeypatch):
    with pytest.raises(ValueError, match="the ranks would simulate the same envs"):
        _runner(monkeypatch, _env(offset=0))
    with pytest.raises(ValueError, match="env_id_offset 32, not rank \\* num_envs = 64"):
        _runner(monkeypatch, _env(offset=32))


def test_runner_refuses_two_ranks_on_one_gpu(monkeypatch):
    with pytest.raises(ValueError, match="two ranks share a GPU"):
        _runner(monkeypatch, _env(), initialised=True, uuids=["GPU-a", "GPU-a"])


def test_runner_refuses_more_ranks_than_the_exchange_holds(monkeypatch):
    with pytest.raises(NotImplementedError, match="at most 8 ranks"):
        _runner(monkeypatch, _env(), world=9)


def test_runner_refuses_empirical_normalisation_and_python_terms_in_data_parallel_runs(monkeypatch):
    with pytest.raises(NotImplementedError, match="empirical_normalization"):
        _runner(monkeypatch, _env(), agent={**AGENT, "empirical_normalization": True})
    with pytest.raises(NotImplementedError, match="host-side Python terms"):
        _runner(monkeypatch, _env(_py_rewards=[("r", None, 1.0, {})]))
