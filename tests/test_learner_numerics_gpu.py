"""The learner kernels against fp64 references, at the shapes and edges where they can go wrong.

* ``wl_gae`` (``learner.compute_returns``): both scans (segment-parallel and streaming) on both sides of every dispatch
  edge, against rsl_rl's ``compute_returns`` + time-out bootstrap restated in fp64, with a running rounding-error bound per
  element; done / time-out patterns on segment boundaries; NaN isolation; bitwise properties (flag forms, embedding,
  repeat runs, graph replay).
* ``wl_dp_adam_step`` with 1..8 emulated ranks on one GPU (every gradient buffer on the one device) against torch.optim.Adam's
  arithmetic in fp64, checked at every step and element for 2000 steps; ``DataParallelAdam`` the same way, and with
  ``Module.zero_grad()`` (gradients set to None) between steps.
* The argument checks of ``compute_returns`` / ``EpisodeStatistics.update`` on CUDA tensors, with the library replaced by a
  stub that fails the test if a launch is reached.

Each numeric test prints the largest |error| / bound it saw (``pytest -s``)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24                       # unit roundoff of fp32 (round to nearest)
f32 = lambda x: float(np.float32(x))


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _ratio(got, want, bound):
    """(all |got - want| <= bound, largest |got - want| / bound, flat index of it); a zero bound admits only a zero error."""
    err = (got.double() - want).abs()
    ratio = torch.where(bound > 0, err / bound.clamp(min=1e-300), torch.where(err > 0, math.inf, 0.0))
    k = int(ratio.argmax())
    return bool((err <= bound).all()), float(ratio.reshape(-1)[k]), k


class _NoLaunch:
    """Stands in for the library: any call fails the test (an argument check is missing if one is reached)."""

    def __getattr__(self, name):
        def launch(*args, **kwargs):
            pytest.fail(f"{name} was reached: the call should have been refused before any launch")
        return launch


# ---------------------------------------------------------------------------------------------------------------- GAE

def gae_kernel(T, N):
    """wl_gae's dispatch rule (wl_api.cu, wl_gae): the segment-parallel scan when N <= 65536 and the T steps make 2..16
    segments of 16 (T in 17..256), the streaming scan otherwise."""
    S = -(-T // 16)
    return "seg" if N <= 65536 and 2 <= S <= 16 else "stream"


# every T on both kernels where the rule allows it (N = 65537 forces the streaming scan); N crosses the 32-env tail of the
# segment kernel's CTA (31 / 32 / 33) and the 65536 threshold
SHAPES = [(1, 33, "stream"), (2, 31, "stream"), (15, 4096, "stream"), (16, 32, "stream"), (16, 65537, "stream"),
          (17, 1, "seg"), (17, 65537, "stream"), (31, 33, "seg"), (31, 65537, "stream"), (32, 31, "seg"),
          (32, 65537, "stream"), (33, 65536, "seg"), (33, 65537, "stream"), (128, 4096, "seg"), (128, 65537, "stream"),
          (255, 32, "seg"), (255, 65537, "stream"), (256, 65536, "seg"), (256, 65537, "stream"), (257, 33, "stream"),
          (257, 65536, "stream"), (1000, 31, "stream"), (1000, 4096, "stream")]

C_STREAM, C_SEG = 8, 86


def gae_reference(rew, val, last, done, tout, gamma, lam):
    """rsl_rl's compute_returns with the time-out bootstrap (r += gamma * V * time_out), in fp64 on the fp32 inputs and the
    fp32 coefficients the kernel receives, and B_t, the running magnitude the error bound scales with:
        A_t = delta_t + k_t A_{t+1},  delta_t = r'_t + (1 - d_t) gamma V_{t+1} - V_t,  k_t = (1 - d_t) gamma lam,  V_T = last
        B_t = |r'_t| + (1 - d_t) gamma |V_{t+1}| + |V_t| + |A_t| + k_t B_{t+1},  |r'_t| = |r_t| + gamma |V_t| time_out_t.

    Bound |A32 - A64| <= C u B_t (u = 2^-24), |ret32 - ret64| <= C u B_t + u |ret|; every rounding below is at most u times
    the magnitude it acts on (first order; the second-order terms and the fp64 reference's own error are below one unit of C
    for T <= 1000, as T u < 1e-4):
    * streaming scan, per step: r' (2 roundings) and delta (3) <= 5u D_t, D_t = |r'| + (1-d) gamma |V_{t+1}| + |V_t|; k in
      fp32 (1) and k A_{t+1} (1) <= 2u k|A_{t+1}| <= 2u (|A_t| + D_t); the sum (1) <= u |A_t|.  So
      e_t <= 7u (D_t + |A_t|) + k_t e_{t+1} <= 7u B_t: C_STREAM = 7 + 1.
    * segment scan: an env's steps are cut into segments of 16, each reduced to A_t = c_t + p_t a_in (c with a_in = 0, p the
      product of the k to the segment's end), the segments chained from the last.  c_t carries the streaming scan's 5u D and
      3u |c| per step, and |c_s| <= |A_s| + p_s |a_in|, so over up to 16 steps e(c_t) <= 5u B + 3 * 16 u p_t |a_in|; p_t
      multiplies up to 16 fp32 k (31 roundings) and p_t a_in (1), the sum (1) <= u |A_t|: the term at a segment's end is
      p_t |A_end| <= p_t B_end with coefficient 48 + 31 + 1 = 80, the rest 5.  a_in is the same form one segment on, and
      each term of B_t meets one segment end, so e_t <= (80 + 5) u B_t: C_SEG = 85 + 1."""
    g, l = f32(gamma), f32(lam)
    r, v = rew.double(), val.double()
    to = tout.double() if tout is not None else torch.zeros_like(r)
    nt = 1.0 - done.double()
    rp = r + g * v * to
    rp_abs = r.abs() + g * v.abs() * to
    T, N = r.shape
    A, B = torch.empty_like(r), torch.empty_like(r)
    a, b, nv = torch.zeros_like(r[0]), torch.zeros_like(r[0]), last.double()
    for t in range(T - 1, -1, -1):
        k = nt[t] * (g * l)
        a = rp[t] + nt[t] * g * nv - v[t] + k * a
        b = rp_abs[t] + nt[t] * g * nv.abs() + v[t].abs() + a.abs() + k * b
        A[t], B[t], nv = a, b, v[t]
    return A, A + v, B


def gae_inputs(T, N, seed, dones="random", touts="mixed"):
    """fp32 rewards over four decades, values with an offset (delta = r + gamma V' - V cancels), flags of a pattern."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    rand = lambda *s: torch.rand(*s, generator=g, device=DEV)
    rew = (torch.randn(T, N, generator=g, device=DEV) * 10.0 ** torch.randint(-2, 2, (T, N), generator=g, device=DEV).float()).contiguous()
    val = (2.0 + torch.randn(T, N, generator=g, device=DEV)).contiguous()
    last = (2.0 + torch.randn(N, generator=g, device=DEV)).contiguous()
    t = torch.arange(T, device=DEV)[:, None]
    if dones == "none":
        d = torch.zeros(T, N, dtype=torch.bool, device=DEV)
    elif dones == "all":
        d = torch.ones(T, N, dtype=torch.bool, device=DEV)
    elif dones == "random":
        d = rand(T, N) < 0.05
    elif dones == "seg_edges":                     # the last step of a segment and the first of the next
        d = ((t % 16 == 15) | (t % 16 == 0)) & (rand(T, N) < 0.5)
    elif dones == "t0":
        d = (t == 0) & (rand(T, N) < 0.5) | (rand(T, N) < 0.01)
    elif dones == "tlast":
        d = (t == T - 1) & (rand(T, N) < 0.5) | (rand(T, N) < 0.01)
    else:
        raise ValueError(dones)
    if touts == "none":
        to = None
    elif touts == "with_done":
        to = d & (rand(T, N) < 0.5)
    elif touts == "without_done":
        to = ~d & (rand(T, N) < 0.05)
    elif touts == "mixed":
        to = (d & (rand(T, N) < 0.5)) | (rand(T, N) < 0.02)
    else:
        raise ValueError(touts)
    return rew, val, last, d.contiguous(), None if to is None else to.contiguous()


def _check_gae(T, N, rew, val, last, d, to, gamma, lam, what):
    from wheeledlab_b200.learner import compute_returns
    ret, adv = compute_returns(rew, val, last, d, gamma, lam, time_outs=to)
    A, R, B = gae_reference(rew, val, last, d, to, gamma, lam)
    c = C_SEG if gae_kernel(T, N) == "seg" else C_STREAM
    ok_a, ra, ka = _ratio(adv, A, c * U * B)
    ok_r, rr, kr = _ratio(ret, R, c * U * B + U * R.abs())
    assert ok_a, f"{what}: advantage outside the bound at (t, env) = {divmod(ka, N)}, |err| / bound = {ra:.3g}"
    assert ok_r, f"{what}: return outside the bound at (t, env) = {divmod(kr, N)}, |err| / bound = {rr:.3g}"
    return max(ra, rr)


def _launched(fn):
    """Names of the wl_gae kernels fn launches (torch.profiler).  A profiling session now and then records no kernel
    activity at all; such a session is repeated (up to three times), a session that records the wrong kernel is not."""
    from torch.profiler import ProfilerActivity, profile
    names = []
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
        names = sorted({e.key.split("(")[0] for e in prof.key_averages() if e.key.startswith("wl_gae")})
        if names:
            break
    return names


@pytest.mark.parametrize("T,N,kernel", SHAPES)
def test_gae_matches_fp64_at_the_dispatch_edges(T, N, kernel):
    _need_gpu()
    from wheeledlab_b200.learner import compute_returns
    assert gae_kernel(T, N) == kernel, "case list disagrees with the dispatch rule"
    rew, val, last, d, to = gae_inputs(T, N, seed=T * 100003 + N)
    want = {"seg": "wl_gae_seg_kernel", "stream": "wl_gae_kernel"}[kernel]
    assert _launched(lambda: compute_returns(rew, val, last, d, 0.99, 0.95, time_outs=to)) == [want]
    ratio = _check_gae(T, N, rew, val, last, d, to, 0.99, 0.95, f"T={T} N={N}")
    print(f"gae {kernel} T={T} N={N}: max |err| / bound = {ratio:.3g}")


COEFS = [(0.99, 0.95), (1.0, 1.0), (0.99, 0.0), (0.0, 0.95), (0.999, 1.0)]


@pytest.mark.parametrize("gamma,lam", COEFS)
@pytest.mark.parametrize("T,N", [(256, 33), (17, 4096), (1000, 65), (257, 31)])
def test_gae_coefficients(T, N, gamma, lam):
    """(1, 1) is undiscounted: with no dones the error accumulates over all T steps."""
    _need_gpu()
    rew, val, last, d, to = gae_inputs(T, N, seed=7 + T + N, dones="none", touts="without_done")
    ratio = _check_gae(T, N, rew, val, last, d, to, gamma, lam, f"gamma={gamma} lam={lam} T={T} N={N}")
    print(f"gae {gae_kernel(T, N)} gamma={gamma} lam={lam} T={T} N={N}: max |err| / bound = {ratio:.3g}")


PATTERNS = [("none", "none"), ("all", "mixed"), ("random", "mixed"), ("seg_edges", "with_done"), ("seg_edges", "without_done"),
            ("t0", "mixed"), ("tlast", "mixed"), ("random", "with_done"), ("random", "without_done")]


@pytest.mark.parametrize("dones,touts", PATTERNS)
@pytest.mark.parametrize("T,N", [(256, 33), (100, 1000), (257, 33), (40, 65537)])
def test_gae_done_and_time_out_patterns(T, N, dones, touts):
    _need_gpu()
    rew, val, last, d, to = gae_inputs(T, N, seed=11 * T + N, dones=dones, touts=touts)
    ratio = _check_gae(T, N, rew, val, last, d, to, 0.99, 0.95, f"{dones}/{touts} T={T} N={N}")
    print(f"gae {gae_kernel(T, N)} {dones}/{touts} T={T} N={N}: max |err| / bound = {ratio:.3g}")


def _bits(x):
    return x.view(torch.int32)


@pytest.mark.parametrize("T,N", [(17, 33), (256, 4096), (300, 33), (16, 65537)])
def test_gae_flag_forms_give_identical_bits(T, N):
    """time_outs=None == all-zero time_outs; bool == uint8 flags; two runs are equal."""
    _need_gpu()
    from wheeledlab_b200.learner import compute_returns
    rew, val, last, d, to = gae_inputs(T, N, seed=3 * T + N)
    none = compute_returns(rew, val, last, d, 0.99, 0.95)
    zeros = compute_returns(rew, val, last, d, 0.99, 0.95, time_outs=torch.zeros(T, N, dtype=torch.uint8, device=DEV))
    zeros_b = compute_returns(rew, val, last, d.to(torch.uint8), 0.99, 0.95, time_outs=torch.zeros(T, N, dtype=torch.bool, device=DEV))
    for x, y in zip(none, zeros):
        assert torch.equal(_bits(x), _bits(y))
    for x, y in zip(none, zeros_b):
        assert torch.equal(_bits(x), _bits(y))
    b = compute_returns(rew, val, last, d, 0.99, 0.95, time_outs=to)
    u8 = compute_returns(rew, val, last, d.to(torch.uint8), 0.99, 0.95, time_outs=to.to(torch.uint8))
    again = compute_returns(rew, val, last, d, 0.99, 0.95, time_outs=to)
    for x, y, z in zip(b, u8, again):
        assert torch.equal(_bits(x), _bits(y)) and torch.equal(_bits(x), _bits(z))
    assert not torch.equal(_bits(b[0]), _bits(none[0])), "the time-outs changed nothing: the bootstrap was dropped"


@pytest.mark.parametrize("T,N", [(33, 33), (256, 65), (17, 1), (300, 33), (16, 40)])
def test_gae_nan_reaches_only_its_env_and_earlier_steps(T, N):
    """A NaN at (t, i) in the rewards or the values may change env i at steps <= t only: every other env, including the dead
    lanes of the segment kernel's tail CTA (which load env N - 1), and env i after t keep their bits."""
    _need_gpu()
    from wheeledlab_b200.learner import compute_returns
    rew, val, last, d, to = gae_inputs(T, N, seed=5 * T + N)
    ret0, adv0 = compute_returns(rew, val, last, d, 0.99, 0.95, time_outs=to)
    spots = {(0, 0), (T - 1, N - 1), (min(15, T - 1), N - 1), (min(16, T - 1), N // 2), (T // 2, 0)}
    for which in ("rewards", "values"):
        for t, i in sorted(spots):
            r, v = rew.clone(), val.clone()
            (r if which == "rewards" else v)[t, i] = float("nan")
            ret, adv = compute_returns(r, v, last, d, 0.99, 0.95, time_outs=to)
            keep = torch.ones(T, N, dtype=torch.bool, device=DEV)
            keep[: t + 1, i] = False
            for got, want in ((ret, ret0), (adv, adv0)):
                assert torch.equal(_bits(got)[keep], _bits(want)[keep]), f"NaN in {which} at {(t, i)} leaked"
            assert torch.isnan(adv[t, i]), f"NaN in {which} at {(t, i)} was lost"


@pytest.mark.parametrize("T,narrow,wide", [(100, 33, 4096), (256, 1, 65536), (300, 33, 1000), (1000, 31, 65537)])
def test_gae_env_outputs_do_not_depend_on_the_slab_width(T, narrow, wide):
    """An env's outputs keep their bits when it sits in a wider slab that selects the same kernel."""
    _need_gpu()
    from wheeledlab_b200.learner import compute_returns
    assert gae_kernel(T, narrow) == gae_kernel(T, wide)
    rew, val, last, d, to = gae_inputs(T, wide, seed=T + wide)
    sl = lambda x: x[..., :narrow].contiguous()
    small = compute_returns(sl(rew), sl(val), sl(last), sl(d), 0.99, 0.95, time_outs=sl(to))
    big = compute_returns(rew, val, last, d, 0.99, 0.95, time_outs=to)
    for x, y in zip(small, big):
        assert torch.equal(_bits(x), _bits(sl(y)))


@pytest.mark.parametrize("T,N", [(128, 4096), (300, 1000)])
def test_gae_graph_replay_equals_the_eager_call(T, N):
    _need_gpu()
    from wheeledlab_b200.learner import compute_returns
    rew, val, last, d, to = gae_inputs(T, N, seed=T * N)
    eager = compute_returns(rew, val, last, d, 0.99, 0.95, time_outs=to)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        compute_returns(rew, val, last, d, 0.99, 0.95, time_outs=to)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = compute_returns(rew, val, last, d, 0.99, 0.95, time_outs=to)
    for k in range(2):
        for x in out:
            x.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        for x, y in zip(out, eager):
            assert torch.equal(_bits(x), _bits(y)), f"replay {k}"


# ------------------------------------------------------------------------------------------------------- fused Adam

def _dp_adam(p, m, v, ptrs, lr, betas, eps, wd, step):
    from wheeledlab_b200._lib import check, lib
    arr = (C.c_void_p * len(ptrs))(*ptrs)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    check(lib.wl_dp_adam_step(C.c_void_p(p.data_ptr()), C.c_void_p(m.data_ptr()), C.c_void_p(v.data_ptr()), len(ptrs), arr,
                              lr, betas[0], betas[1], eps, wd, step, p.numel(), stream), "wl_dp_adam_step")


class GradStream:
    """A fixed gradient stream for R ranks (no backprop, so kernel and reference cannot drift apart chaotically): per element
    a rank-specific value over three decades times cos(w t + phi) (smooth sign changes), times a stream scale that walks
    over six decades (1e-3 .. 1e3, a decade every 150 steps); every 5th element flips sign every step, every 11th is
    exactly zero always, and every 17th step rank 0 contributes exact zeros."""

    def __init__(self, R, n, seed):
        g = torch.Generator(device=DEV).manual_seed(seed)
        self.base = torch.randn(R, n, generator=g, device=DEV, dtype=torch.float64) * \
            10.0 ** torch.randint(-3, 1, (R, n), generator=g, device=DEV).double()
        self.w = 0.01 + 0.3 * torch.rand(n, generator=g, device=DEV, dtype=torch.float64)
        self.phi = 2 * math.pi * torch.rand(n, generator=g, device=DEV, dtype=torch.float64)
        idx = torch.arange(n, device=DEV)
        self.flip, self.zero = idx % 5 == 1, idx % 11 == 3
        self.bufs = torch.zeros(R, n, dtype=torch.float32, device=DEV)

    def fill(self, t):
        scale = 10.0 ** (abs((t // 150) % 12 - 6) - 3)
        x = self.base * torch.cos(self.w * t + self.phi) * scale
        x = torch.where(self.flip, self.base.abs() * scale * (1.0 if t % 2 else -1.0), x)
        x = torch.where(self.zero, 0.0, x)
        self.bufs.copy_(x)
        if t % 17 == 0:
            self.bufs[0].zero_()
        return self.bufs


class AdamReference:
    """torch.optim.Adam's arithmetic (torch/optim/adam.py, amsgrad off, L2 weight decay) in fp64, one step from the kernel's
    own fp32 state, on the fp64 mean of the R rank gradients:
        g = mean_r g_r + wd p;  m' = m + w1 (g - m)  (exp_avg.lerp_(grad, 1 - beta1));  v' = beta2 v + cb2 g^2
        update = -(lr / bc1) m' / (sqrt(v') / sqrt(bc2) + eps),  bc = 1 - beta ** step in Python doubles,
    with w1 = fp32(1 - beta1), beta2 and cb2 = fp32(1 - beta2) as torch hands them to its fp32 kernels.

    Bounds (each rounding <= u = 2^-24 of the magnitude it acts on; G = mean_r |g_r| + wd |p|):
    * gradient: R - 1 sums, the division, the weight-decay FMA, wd in fp32: e_g = (R + 2) u G.
    * m: the fp32 coefficient (beta1 vs 1 - w1), the product cb1 g, the FMA: e_m = 3u M + w1 e_g, M = (1 - w1)|m| + w1 G.
    * v: g g, cb2 (g g), the FMA: e_v = 3u V + 2 cb2 G e_g, V = beta2 v + cb2 G^2.
    * update, lr (m / bc1) / (sqrt(v / bc2) + eps): bc1 and bc2 in fp32 (2), the division by bc1, the product by lr and lr
      in fp32 (3), v / bc2 and the square root (2: the square root halves the first), eps in fp32 and the sum (2), the
      division (1): 9u |update|; m' and v' reach it with e_m and e_s = min(sqrt(e_v / bc2), e_v / (2 bc2 s)) on
      s = sqrt(v' / bc2): (lr / bc1) e_m / D + |update| e_s / D, D = max(s + eps - e_s, eps) (exact for the perturbed
      quotient, and the eps floor where v' ~ 0); p - x rounds once: u |p_new|.  The check is on p_new - p_old (exact in
      fp64), so a systematic 1e-6 relative bias (~17 u) is visible wherever |p| is not far above |update|."""

    def __init__(self, lr, betas, eps, wd):
        self.lr, self.beta1, self.beta2, self.eps, self.wd = lr, betas[0], betas[1], eps, wd
        self.w1, self.b2, self.cb2 = f32(1 - betas[0]), f32(betas[1]), f32(1 - betas[1])

    def ratios(self, step, p0, m0, v0, grads, p1, m1, v1):
        """Largest |err| / bound of (update, m, v) as a device tensor; raises nothing (no host sync)."""
        R = grads.shape[0]
        p, m, v, G = p0.double(), m0.double(), v0.double(), grads.double()
        g = G.sum(0) / R + self.wd * p
        gabs = G.abs().sum(0) / R + self.wd * p.abs()
        e_g = (R + 2) * U * gabs
        mn = m + self.w1 * (g - m)
        e_m = 3 * U * ((1 - self.w1) * m.abs() + self.w1 * gabs) + self.w1 * e_g
        vn = self.b2 * v + self.cb2 * g * g
        e_v = 3 * U * (self.b2 * v + self.cb2 * gabs * gabs) + 2 * self.cb2 * gabs * e_g
        bc1, bc2 = 1 - self.beta1 ** step, 1 - self.beta2 ** step
        s = vn.sqrt() / math.sqrt(bc2)
        upd = -(self.lr / bc1) * mn / (s + self.eps)
        e_s = torch.minimum((e_v / bc2).sqrt(), e_v / bc2 / (2 * s).clamp(min=1e-300))
        d_lo = (s + self.eps - e_s).clamp(min=f32(self.eps))
        e_u = 9 * U * upd.abs() + (self.lr / bc1) * e_m / d_lo + upd.abs() * e_s / d_lo + U * p1.double().abs()

        def r(got, want, bound):
            err = (got - want).abs()
            return torch.where(bound > 0, err / bound.clamp(min=1e-300), torch.where(err > 0, math.inf, 0.0)).max()
        return torch.stack([r(p1.double() - p, upd, e_u), r(m1.double(), mn, e_m), r(v1.double(), vn, e_v)])


DRIFT_AC_PARAMS = (14 * 64 + 64 + 64 * 64 + 64 + 64 * 2 + 2) + (14 * 64 + 64 + 64 * 64 + 64 + 64 + 1) + 2   # 64x64 actor + critic + std
ADAM_NS = [1, 255, 256, 257, DRIFT_AC_PARAMS, 2 ** 20 + 3]
ADAM_CASES = [(n, R, 1e-2 if (k + j) % 2 else 0.0) for k, n in enumerate(ADAM_NS) for j, R in enumerate((1, 2, 3, 8))]
ADAM_STEPS = 2000


def _p0(n, lr, seed):
    """Parameters of the order of a few updates (and up to 100x more), so that the final rounding of p - x does not hide
    errors in the update; the test restores them before every step."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (lr * torch.randn(n, generator=g, device=DEV) * 10.0 ** torch.randint(0, 3, (n,), generator=g, device=DEV).float()).contiguous()


@pytest.mark.parametrize("n,R,wd", ADAM_CASES)
def test_dp_adam_matches_fp64_torch_adam_every_step(n, R, wd):
    """R emulated ranks (R gradient buffers on this device) for 2000 steps; every step and element of the update, m and v
    within the bounds of AdamReference."""
    _need_gpu()
    lr, betas, eps = 3e-3, (0.9, 0.999), 1e-8
    ref, stream = AdamReference(lr, betas, eps, wd), GradStream(R, n, seed=n * 10 + R)
    p0 = _p0(n, lr, seed=n)
    p, m, v = p0.clone(), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    ptrs = [stream.bufs[r].data_ptr() for r in range(R)]
    worst = torch.zeros(3, dtype=torch.float64, device=DEV)
    for step in range(1, ADAM_STEPS + 1):
        grads = stream.fill(step)
        p.copy_(p0)
        m0, v0 = m.clone(), v.clone()
        _dp_adam(p, m, v, ptrs, lr, betas, eps, wd, step)
        worst = torch.maximum(worst, ref.ratios(step, p0, m0, v0, grads, p, m, v))
    worst = worst.tolist()
    print(f"dp_adam n={n} R={R} wd={wd}: max |err| / bound update {worst[0]:.3g}, m {worst[1]:.3g}, v {worst[2]:.3g}")
    assert max(worst) <= 1.0, f"n={n} R={R} wd={wd}: |err| / bound (update, m, v) = {worst}"
    assert v.abs().max() > 0 and m.abs().max() > 0


@pytest.mark.parametrize("n", [257, DRIFT_AC_PARAMS, 2 ** 20 + 3])
def test_dp_adam_replicas_on_one_pointer_list_stay_identical(n):
    """k replicas (own param / m / v) stepping on the same 8 gradient buffers keep identical bits: every rank forms the
    same mean in the same order."""
    _need_gpu()
    stream = GradStream(8, n, seed=n + 1)
    ptrs = [stream.bufs[r].data_ptr() for r in range(8)]
    p0 = _p0(n, 1e-3, seed=2 * n)
    reps = [(p0.clone(), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)) for _ in range(3)]
    for step in range(1, 301):
        stream.fill(step)
        for p, m, v in reps:
            _dp_adam(p, m, v, ptrs, 1e-3, (0.9, 0.999), 1e-8, 1e-2, step)
    for p, m, v in reps[1:]:
        for x, y in zip((p, m, v), reps[0]):
            assert torch.equal(_bits(x), _bits(y))
    assert not torch.equal(reps[0][0], p0)


def _actor_critic_params(seed):
    torch.manual_seed(seed)
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(14, 64), torch.nn.ELU(), torch.nn.Linear(64, 64), torch.nn.ELU(),
                                         torch.nn.Linear(64, out)).to(DEV)
    actor, critic = mk(2), mk(1)
    std = torch.nn.Parameter(torch.ones(2, device=DEV))
    return torch.nn.ModuleList([actor, critic]), [*actor.parameters(), *critic.parameters(), std]


def test_data_parallel_adam_world_size_one_matches_fp64_every_step():
    """DataParallelAdam (world size 1) on the 64x64 Drift actor-critic's parameters, gradients written into p.grad from
    the fixed stream, 2000 steps, every step and element within AdamReference's bounds."""
    _need_gpu()
    from wheeledlab_b200.learner import DataParallelAdam
    _, params = _actor_critic_params(0)
    n = sum(p.numel() for p in params)
    assert n == DRIFT_AC_PARAMS
    lr, betas, eps, wd = 1e-3, (0.9, 0.999), 1e-8, 0.0
    opt = DataParallelAdam(params, lr=lr, betas=betas, eps=eps, weight_decay=wd)
    ref, stream = AdamReference(lr, betas, eps, wd), GradStream(1, n, seed=4)
    p0 = _p0(n, lr, seed=9)
    worst = torch.zeros(3, dtype=torch.float64, device=DEV)
    for step in range(1, ADAM_STEPS + 1):
        grads = stream.fill(step)
        off = 0
        with torch.no_grad():
            for p in params:
                k = p.numel()
                p.copy_(p0[off:off + k].view_as(p))
                p.grad.copy_(grads[0, off:off + k].view_as(p))
                off += k
        m0, v0 = opt.m.clone(), opt.v.clone()
        opt.step()
        p1 = torch.cat([p.detach().reshape(-1) for p in params])
        worst = torch.maximum(worst, ref.ratios(step, p0, m0, v0, grads, p1, opt.m, opt.v))
    worst = worst.tolist()
    print(f"DataParallelAdam world 1: max |err| / bound update {worst[0]:.3g}, m {worst[1]:.3g}, v {worst[2]:.3g}")
    assert max(worst) <= 1.0, worst


def test_data_parallel_adam_after_module_zero_grad():
    """Module.zero_grad() sets p.grad to None; backward then writes fresh gradients.  step() must train on them, exactly as
    after DataParallelAdam.zero_grad(), and a parameter left without a gradient is refused."""
    _need_gpu()
    from wheeledlab_b200.learner import DataParallelAdam
    net_a, pa = _actor_critic_params(0)
    net_b, pb = _actor_critic_params(0)
    net_r, pr = _actor_critic_params(0)
    opt_a, opt_b = DataParallelAdam(pa, lr=3e-3), DataParallelAdam(pb, lr=3e-3)
    opt_r = torch.optim.Adam(pr, lr=3e-3)
    g = torch.Generator(device=DEV).manual_seed(1)
    loss = lambda net, params, x, y: ((net[0](x) * params[-1] - y) ** 2).mean() + (net[1](x) ** 2).mean()
    for it in range(30):
        x, y = torch.randn(512, 14, generator=g, device=DEV), torch.randn(512, 2, generator=g, device=DEV)
        opt_a.zero_grad(); loss(net_a, pa, x, y).backward(); opt_a.step()
        net_b.zero_grad(); pb[-1].grad = None; loss(net_b, pb, x, y).backward(); opt_b.step()
        opt_r.zero_grad(); loss(net_r, pr, x, y).backward(); opt_r.step()
    for p, q in zip(pa, pb):
        assert torch.equal(p, q)
    err = max(float((p - q).detach().abs().max()) for p, q in zip(pb, pr))
    assert err < 5e-6, err
    net_b.zero_grad()
    pb[-1].grad = None
    with pytest.raises(ValueError, match="no gradient"):
        opt_b.step()


# ----------------------------------------------------------------------------------------- refusals on CUDA tensors

def _good(T=20, N=33):
    rew, val, last, d, to = gae_inputs(T, N, seed=1)
    return dict(rewards=rew, values=val, last_values=last, dones=d, time_outs=to)


def _call(**kw):
    from wheeledlab_b200.learner import compute_returns
    return compute_returns(kw["rewards"], kw["values"], kw["last_values"], kw["dones"], 0.99, 0.95, time_outs=kw["time_outs"])


@pytest.mark.parametrize("name,bad,match", [
    ("time_outs", lambda x: x.cpu(), "time_outs is on cpu"),
    ("time_outs", lambda x: x.t().contiguous().t(), "time_outs must be a contiguous"),
    ("time_outs", lambda x: x.long(), "time_outs must be uint8 or bool"),
    ("time_outs", lambda x: x[:-1].contiguous(), "time_outs must have shape"),
    ("dones", lambda x: x.cpu(), "dones is on cpu"),
    ("dones", lambda x: x.t().contiguous().t(), "dones must be a contiguous"),
    ("values", lambda x: x.double(), "values must be float32"),
    ("values", lambda x: x.t().contiguous().t(), "values must be a contiguous"),
    ("last_values", lambda x: x[:-1].contiguous(), "last_values must have shape"),
    ("last_values", lambda x: x.cpu(), "last_values is on cpu"),
    ("rewards", lambda x: x.t().contiguous().t(), "rewards must be a contiguous"),
])
def test_compute_returns_refuses_bad_cuda_tensors_before_any_launch(monkeypatch, name, bad, match):
    _need_gpu()
    from wheeledlab_b200 import learner
    kw = _good()
    kw[name] = bad(kw[name])
    monkeypatch.setattr(learner, "lib", _NoLaunch())
    with pytest.raises(ValueError, match=match):
        _call(**kw)


def test_episode_statistics_refuses_bad_dtypes_before_any_launch(monkeypatch):
    _need_gpu()
    from wheeledlab_b200 import learner
    T, N = 8, 33
    ep = learner.EpisodeStatistics(N, T, DEV)
    rew = torch.zeros(T, N, device=DEV)
    flag = torch.zeros(T, N, dtype=torch.uint8, device=DEV)
    monkeypatch.setattr(learner, "lib", _NoLaunch())
    with pytest.raises(ValueError, match="rewards must be float32"):
        ep.update(rew.double(), flag, flag)
    with pytest.raises(ValueError, match="uint8 or bool"):
        ep.update(rew, flag.long(), flag)
    with pytest.raises(ValueError, match="uint8 or bool"):
        ep.update(rew, flag, flag.long())
