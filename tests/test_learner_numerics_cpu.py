"""The learner entry points refuse malformed arguments before anything is launched: compute_returns (every tensor,
time_outs included) with the library replaced by a stub that fails the test if a launch is reached, and wl_dp_adam_step's
own checks through the C-ABI with pointers that are never dereferenced."""
import ctypes as C

import pytest
import torch

T, N = 20, 33


class _NoLaunch:
    """Stands in for the library: any call fails the test (an argument check is missing if one is reached)."""

    def __getattr__(self, name):
        def launch(*args, **kwargs):
            pytest.fail(f"{name} was reached: the call should have been refused before any launch")
        return launch


def _inputs():
    return dict(rewards=torch.zeros(T, N), values=torch.zeros(T, N), last_values=torch.zeros(N),
                dones=torch.zeros(T, N, dtype=torch.bool), time_outs=torch.zeros(T, N, dtype=torch.uint8))


# each case breaks one input; the checks run in the order dtype, shape, device, CUDA / contiguity, so host tensors reach
# the specific refusal here (on a GPU the host-tensor and non-contiguous cases are covered with CUDA inputs)
CASES = [
    ("rewards", lambda x: x.double(), "rewards must be float32"),
    ("rewards", lambda x: x.half(), "rewards must be float32"),
    ("rewards", lambda x: x[0], r"rewards must be \[T, N\]"),
    ("values", lambda x: x.double(), "values must be float32"),
    ("values", lambda x: x.to(torch.bfloat16), "values must be float32"),
    ("values", lambda x: torch.zeros(T, N + 1), "values must have shape"),
    ("values", lambda x: torch.zeros(N, T), "values must have shape"),
    ("values", lambda x: x.to("meta"), "values is on meta"),
    ("last_values", lambda x: x.double(), "last_values must be float32"),
    ("last_values", lambda x: x[:-1], "last_values must have shape"),
    ("last_values", lambda x: x[None], "last_values must have shape"),
    ("last_values", lambda x: x.to("meta"), "last_values is on meta"),
    ("dones", lambda x: x.int(), "dones must be uint8 or bool"),
    ("dones", lambda x: x.float(), "dones must be uint8 or bool"),
    ("dones", lambda x: x[:, :-1], "dones must have shape"),
    ("dones", lambda x: x.to("meta"), "dones is on meta"),
    ("time_outs", lambda x: x.long(), "time_outs must be uint8 or bool"),
    ("time_outs", lambda x: x.float(), "time_outs must be uint8 or bool"),
    ("time_outs", lambda x: x[:-1], "time_outs must have shape"),
    ("time_outs", lambda x: x.reshape(-1), "time_outs must have shape"),
    ("time_outs", lambda x: x.to("meta"), "time_outs is on meta"),
    ("rewards", lambda x: x, "rewards must be a contiguous CUDA tensor"),
]


@pytest.mark.parametrize("name,bad,match", CASES)
def test_compute_returns_refuses_before_any_launch(monkeypatch, name, bad, match):
    from wheeledlab_b200 import learner
    kw = _inputs()
    kw[name] = bad(kw[name])
    monkeypatch.setattr(learner, "lib", _NoLaunch())
    with pytest.raises(ValueError, match=match):
        learner.compute_returns(kw["rewards"], kw["values"], kw["last_values"], kw["dones"], 0.99, 0.95, time_outs=kw["time_outs"])


def test_dp_adam_step_rejects_bad_arguments_before_any_launch():
    import wheeledlab_b200 as wl
    lib = wl.lib
    fake = C.c_void_p(1 << 20)
    grads = (C.c_void_p * 9)(*([1 << 21] * 9))
    call = lambda n_ranks=2, g=grads, step=1, n=256: lib.wl_dp_adam_step(fake, fake, fake, n_ranks, g, 1e-3, 0.9, 0.999, 1e-8, 0.0,
                                                                        step, n, None)
    for kw in (dict(n_ranks=0), dict(n_ranks=9), dict(step=0), dict(step=-1), dict(n=0), dict(n=-5)):
        assert call(**kw) == -1 and b"bad argument" in lib.wl_last_error(), kw
    with_null = (C.c_void_p * 3)(1 << 21, None, 1 << 21)
    assert call(n_ranks=3, g=with_null) == -1 and b"null gradient pointer" in lib.wl_last_error()
    assert call(g=None) == -1 and b"bad argument" in lib.wl_last_error()
    assert lib.wl_dp_adam_step(None, fake, fake, 1, grads, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1, 256, None) == -1
