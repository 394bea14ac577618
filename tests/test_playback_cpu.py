"""Playback without a GPU: tools/play_policy.py's argument handling and checkpoint resolution, the run.json round trip,
and wl_actor_mean's refusals, which return before any device call."""
import ctypes as C
import json
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


def _play_policy():
    sys.path.insert(0, str(ROOT / "tools"))
    import play_policy
    return play_policy


def _resolve(argv):
    pp = _play_policy()
    return pp.resolve(pp.parser().parse_args(argv))


def _run_dir(tmp_path, its, run_json=True):
    from wheeledlab_b200.runs import agent_cfg, save_run_config
    run = tmp_path / "run"
    (run / "models").mkdir(parents=True)
    for it in its:
        (run / "models" / f"model_{it}.pt").write_bytes(b"")
    (run / "models" / "notes.txt").write_text("")
    if run_json:
        save_run_config(str(run), "Isaac-MushrElevationRL-v0", 1024, 7, agent_cfg("relu", 24, 10))
    return run


@pytest.mark.parametrize("argv", [[], ["--task", "Isaac-MushrDriftRL-v0"], ["--policy-path", "model_1.pt"]])
def test_without_a_run_path_task_and_policy_are_both_needed(argv):
    with pytest.raises(ValueError, match="Either path to run directory or task/policy must be provided"):
        _resolve(argv)


def test_video_is_refused(tmp_path):
    run = _run_dir(tmp_path, [0])
    with pytest.raises(ValueError, match="--video is not supported"):
        _resolve(["-p", str(run), "--video"])


def test_the_script_reports_refusals_as_an_error_exit(capsys):
    assert _play_policy().main(["--video"]) == 2
    assert "--video is not supported" in capsys.readouterr().err


def test_checkpoint_resolution_picks_the_highest_iteration_or_the_one_asked_for(tmp_path):
    run = _run_dir(tmp_path, [0, 50, 100, 250, 9])
    r = _resolve(["-p", str(run)])
    assert Path(r["policy_path"]) == run / "models" / "model_250.pt"      # numeric, not lexical: 250 > 100 > 9
    assert Path(r["playback_dir"]) == run / "playback"
    r = _resolve(["-p", str(run), "--checkpoint", "50"])
    assert Path(r["policy_path"]) == run / "models" / "model_50.pt"


def test_a_missing_checkpoint_is_a_clear_error(tmp_path):
    run = _run_dir(tmp_path, [0, 50])
    with pytest.raises(FileNotFoundError, match="model_7.pt does not exist"):
        _resolve(["-p", str(run), "--checkpoint", "7"])
    empty = _run_dir(tmp_path / "e", [])
    with pytest.raises(FileNotFoundError, match="no checkpoint"):
        _resolve(["-p", str(empty)])
    with pytest.raises(FileNotFoundError, match="does not exist"):
        _resolve(["--task", "Isaac-MushrDriftRL-v0", "--policy-path", str(tmp_path / "nope.pt")])


def test_run_json_round_trip_gives_task_activation_size_and_seed(tmp_path):
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    from wheeledlab_b200.runs import load_run_config
    run = _run_dir(tmp_path, [3])
    cfg = load_run_config(str(run))
    assert cfg["task"] == "Isaac-MushrElevationRL-v0" and cfg["num_envs"] == 1024 and cfg["seed"] == 7
    assert json.loads((run / "run.json").read_text()) == cfg
    r = _resolve(["-p", str(run)])
    assert (r["task"], r["num_envs"], r["seed"]) == ("Isaac-MushrElevationRL-v0", 1024, 7)
    s = FusedOnPolicyRunner.settings(r["agent_cfg"])
    assert s.activation == "relu" and s.num_steps_per_env == 24 and s.save_interval == 10
    r = _resolve(["-p", str(run), "--num-envs", "64", "--seed", "1", "--task", "Isaac-MushrDriftRL-v0"])
    assert (r["task"], r["num_envs"], r["seed"]) == ("Isaac-MushrDriftRL-v0", 64, 1)


def test_without_run_json_the_activation_follows_the_task(tmp_path):
    from wheeledlab_b200.learner import FusedOnPolicyRunner
    from wheeledlab_b200.runs import task_activation
    run = _run_dir(tmp_path, [0], run_json=False)
    with pytest.raises(ValueError, match="no run.json"):
        _resolve(["-p", str(run)])
    for task, act in (("Isaac-MushrDriftRL-v0", "elu"), ("Isaac-F1TenthDriftRL-v0", "elu"), ("hound_4wd", "elu"),
                      ("Isaac-MushrElevationRL-v0", "relu"), ("Isaac-MushrVisualRL-v0", "relu")):
        assert task_activation(task) == act
        r = _resolve(["-p", str(run), "--task", task])
        assert FusedOnPolicyRunner.settings(r["agent_cfg"]).activation == act
        assert r["num_envs"] is None and r["seed"] is None


def test_a_malformed_run_json_is_refused(tmp_path):
    from wheeledlab_b200.runs import load_run_config
    (tmp_path / "run.json").write_text(json.dumps({"num_envs": 4}))
    with pytest.raises(ValueError, match="not a run config"):
        load_run_config(str(tmp_path))


# wl_actor_mean checks its arguments before any device call, so these run without a GPU.  The pointers are never
# dereferenced: aligned fake addresses.
@pytest.mark.parametrize("n,obs_dim,act,blob_off,mean_off,obs_off,code,msg", [
    (0, 14, 0, 0, 0, 0, -1, b"n must be"),
    (4, 0, 1, 0, 0, 0, -3, b"obs_dim"),
    (4, 4097, 1, 0, 0, 0, -3, b"obs_dim"),
    (4, 17, 0, 0, 0, 0, -3, b"ELU"),
    (4, 14, 2, 0, 0, 0, -1, b"activation"),
    (4, 14, -1, 0, 0, 0, -1, b"activation"),
    (4, 14, 0, 8, 0, 0, -1, b"16-byte"),
    (4, 689, 1, 0, 4, 0, -1, b"8-byte"),
    (4, 689, 1, 0, 0, 2, -1, b"aligned"),
])
def test_actor_mean_refuses_bad_arguments_before_any_device_call(n, obs_dim, act, blob_off, mean_off, obs_off, code, msg):
    from wheeledlab_b200._lib import lib
    base = 1 << 20
    rc = lib.wl_actor_mean(C.c_void_p(base + obs_off), n, obs_dim, C.c_void_p(base + blob_off), act, C.c_void_p(base + mean_off), None)
    assert rc == code
    assert msg in lib.wl_last_error()


def test_actor_mean_refuses_null_pointers():
    from wheeledlab_b200._lib import lib
    p = C.c_void_p(1 << 20)
    assert lib.wl_actor_mean(None, 4, 14, p, 0, p, None) == -1
    assert lib.wl_actor_mean(p, 4, 14, None, 0, p, None) == -1
    assert lib.wl_actor_mean(p, 4, 14, p, 0, None, None) == -1
    assert b"null" in lib.wl_last_error()


def test_infer_step_refuses_a_null_handle():
    from wheeledlab_b200._lib import lib
    p = C.c_void_p(1 << 20)
    assert lib.wl_act_infer_step(None, p, p, p, p, p, p, p, None, 0, None) == -1
    assert b"wl_act_infer_step" in lib.wl_last_error()
