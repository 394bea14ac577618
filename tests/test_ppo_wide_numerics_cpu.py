"""fp64 references with a per-element rounding-error bound for the PPO update's kernels, and the margin batches the GPU
tests (tests/test_ppo_wide_numerics_gpu.py) run them on.  The tests in this file check the machinery without a GPU, against
an fp32 emulation of the kernels' summation orders.

``TV`` holds an fp64 value v and a bound e on |fp32 result - v|, where the fp32 result is what the kernel's sequence of
fp32 operations gives on the same fp32 inputs (u = 2^-24, gamma(L) = L u / (1 - L u)):

* an elementwise fp32 operation adds u (|v| + e) to the propagated input bounds (``add``, ``mul``, ``div``); a
  cancellation such as ``act - m0`` or ``lp - lp_old`` therefore keeps its inputs' bounds, not a bound relative to its
  result; ``expf`` is within 2 ulp and ``logf`` within 1 ulp (CUDA C Programming Guide, single-precision mathematical
  functions; the library is built without fast math), and 1 ulp <= 2u |result|;
* every rounding also adds 2^-149 (fp32's smallest subnormal) for results near underflow;
* a sum of products accumulated through at most L roundings is within gamma(L) sum |terms| (first order: the inputs'
  bounds times the coefficients' magnitudes, plus their own rounding) -- ``dot`` and ``outer_sum``;
* relu is 1-Lipschitz, so |relu(z_fp32) - relu(z)| <= e(z).  Its derivative is a mask that the bound decides where
  |z| > e(z); an undecided mask entry m * g is given the hull of {g, 0}: bound |g| + e(g).

The chain lengths L, read from csrc/wl_wide.cuh and csrc/wl_ppo.cuh (the library is built with -fmad=false, so every fmaf
is explicit and nothing else fuses):

* wide layer 1 (``wide_layer1``): each 32-input chunk is an fmaf chain on 0 (<= 32 roundings), added to a running sum that
  starts at the bias (one rounding per later chunk): L = 32 + ceil(ceil4(D) / 32) + 1.
* layer 2 and the backward dz1 = dz2 W2 (``mlp_tile_layer``, bias or zero first, then 64 fmaf): L = 64 (+1 kept).
* the heads: 8 fmaf per thread on 0, the 3-step butterfly, then the bias: L = 12.  dz2 = d0 w0 + d1 w1: L = 2.
* the narrow network's layer 1 (``wl_ppo_grad_kernel``): bias, then ceil4(D) <= 16 fmaf: L = ceil4(D) + 1.
* the gradient sums: CTA (split) s accumulates tiles s, s + ctas, ... in sample order, at most ceil(tiles / ctas) * 32
  samples (the zero tail rows add exact zeros); ``wl_ppo_reduce_kernel`` then adds the ctas rows to 0 in CTA order:
  a CTA row has L = ceil(tiles / ctas) * 32, the reduced row L = ceil(tiles / ctas) * 32 + ctas.

Every check reports the largest |err| / bound it saw."""
from __future__ import annotations

import copy
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

U = 2.0 ** -24                      # fp32 unit roundoff
ETA = 2.0 ** -149                   # fp32's smallest subnormal: the absolute error of a rounding near underflow
ROWS = 32                           # WL_PPO_TILE = WL_WIDE_ROWS: samples per tile
KC = 32                             # WL_WIDE_KC: inputs per layer-1 chunk
HID = 64
LOG_SQRT_2PI = 0.5 * math.log(2.0 * math.pi)


def gam(n: int) -> float:
    return n * U / (1.0 - n * U)


def f32(x: float) -> float:
    return float(np.float32(x))


class TV:
    """fp64 value v and a bound e on |fp32 result - v|."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=None):
        self.v = v
        self.e = torch.zeros_like(v) if e is None else e

    def __getitem__(self, k):
        return TV(self.v[k], self.e[k])


def const(x: float, like: torch.Tensor) -> TV:
    """The fp64 constant x where the kernel uses fp32(x): bound |fp32(x) - x|."""
    return TV(torch.full_like(like, x), torch.full_like(like, abs(f32(x) - x)))


def _rnd(v, e):
    return TV(v, e + U * (v.abs() + e) + ETA)


def add(a: TV, b: TV) -> TV:
    return _rnd(a.v + b.v, a.e + b.e)


def sub(a: TV, b: TV) -> TV:
    return _rnd(a.v - b.v, a.e + b.e)


def mul(a: TV, b: TV) -> TV:
    return _rnd(a.v * b.v, a.v.abs() * b.e + b.v.abs() * a.e + a.e * b.e)


def div(a: TV, b: TV) -> TV:
    v = a.v / b.v
    return _rnd(v, (a.e + v.abs() * b.e) / (b.v.abs() - b.e))


def neg(a: TV) -> TV:
    return TV(-a.v, a.e)


def scale(a: TV, s) -> TV:
    """Multiplication by an exact power of two, or by a 0 / 1 / 0.5 flag: no rounding."""
    return TV(a.v * s, a.e * (s.abs() if torch.is_tensor(s) else abs(s)))


def expf(a: TV) -> TV:
    v = torch.exp(a.v)
    e = v * torch.expm1(a.e)
    return TV(v, e + 4 * U * (v + e) + 2 * ETA)


def logf(a: TV) -> TV:
    v = torch.log(a.v)
    e = -torch.log1p(-a.e / a.v)
    return TV(v, e + 2 * U * (v.abs() + e))


def expm1f(a: TV) -> TV:
    v = torch.expm1(a.v)
    e = torch.exp(a.v + a.e) * a.e
    return TV(v, e + 2 * U * (v.abs() + e))


def dot(x: TV, W: torch.Tensor, b: torch.Tensor | None, L: int) -> TV:
    """x [n, K] . W [K, m] (+ b [m]), W and b exact, summed through at most L roundings."""
    aw = W.abs()
    v = x.v @ W
    mag = (x.v.abs() + x.e) @ aw
    if b is not None:
        v = v + b
        mag = mag + b.abs()
    return TV(v, gam(L) * mag + x.e @ aw + L * ETA)


def outer_sum(a: TV, b: TV, L: int, groups: int = 1) -> TV:
    """sum over samples of a[s, p] b[s, q] -> [groups, p, q] for a, b [groups * n, .] (group g: rows g n .. g n + n - 1),
    each through at most L roundings."""
    A, Ae, B, Be = (t.reshape(groups, -1, t.shape[-1]) for t in (a.v, a.e, b.v, b.e))
    At = A.transpose(1, 2)
    v = At @ B
    aa, ab = A.abs(), B.abs()
    prop = aa.transpose(1, 2) @ Be + Ae.transpose(1, 2) @ ab + Ae.transpose(1, 2) @ Be
    return TV(v, gam(L) * ((aa + Ae).transpose(1, 2) @ (ab + Be)) + prop + L * ETA)


def relu(z: TV) -> TV:
    return TV(z.v.clamp(min=0.0), z.e)


def masked(g: TV, z: TV | None = None, mask: torch.Tensor | None = None) -> TV:
    """relu'(z) * g.  With `mask` (the kernel's own h > 0) the mask is exact; otherwise z > 0 in fp64, and where the bound
    does not decide it the entry gets the hull of {g, 0}."""
    if mask is not None:
        m = mask.to(g.v.dtype)
        return TV(g.v * m, g.e * m)
    m = (z.v > 0).to(g.v.dtype)
    dec = z.v.abs() > z.e
    return TV(g.v * m, torch.where(dec, g.e * m, g.v.abs() + g.e))


# ---- the network -------------------------------------------------------------------------------------------------------

def params(blob: torch.Tensor, D: int) -> dict:
    """The blob's tensors in fp64 on its device, input-major weights (Wt [in, out]) and std."""
    from wheeledlab_b200.policy import actor_critic_state_dict
    sd = {k: v.double() for k, v in actor_critic_state_dict(blob, D).items()}
    p = {"std": sd["std"]}
    for net in ("actor", "critic"):
        for k in (0, 2, 4):
            p[f"{net}.{k}.Wt"] = sd[f"{net}.{k}.weight"].t().contiguous()
            p[f"{net}.{k}.b"] = sd[f"{net}.{k}.bias"]
    return p


def l1_chain(D: int, activation: str) -> int:
    nin1 = (D + 3) & ~3
    return nin1 + 1 if activation == "elu" else KC + (nin1 + KC - 1) // KC + 1


def layer1(p: dict, X: torch.Tensor, activation: str = "relu") -> TV:
    """Pre-activation of layer 1 of both nets [n, 128] (actor | critic) from exact fp32 rows X [n, D] (fp64)."""
    L = l1_chain(X.shape[1], activation)
    x = TV(X)
    return TV(*(torch.cat(t, 1) for t in zip(*((z.v, z.e) for z in (dot(x, p[f"{n}.0.Wt"], p[f"{n}.0.b"], L) for n in ("actor", "critic"))))))


def act(z: TV, activation: str) -> TV:
    if activation == "relu":
        return relu(z)
    ex = expm1f(TV(z.v.clamp(max=0.0), z.e))                 # ELU: z > 0 ? z : expm1f(z), 1-Lipschitz across 0
    pos = z.v > 0
    return TV(torch.where(pos, z.v, ex.v), torch.where(pos, z.e, torch.maximum(ex.e, z.e)))


def act_grad(h: TV, z: TV | None, activation: str, mask=None):
    """The derivative factor the kernel forms from h, as a function on g: g -> relu'/elu' * g."""
    if activation == "relu":
        return lambda g: masked(g, z, mask)
    # ELU: elu'(h) = h > 0 ? 1 : fp32(h + 1), continuous at 0: where undecided, the hull of both forms (they differ by |h|)
    one = torch.ones_like(h.v)
    hp1 = add(h, TV(one))
    pos = h.v > 0
    dec = h.v.abs() > h.e
    f = TV(torch.where(pos, one, hp1.v), torch.where(pos & dec, 0.0 * one, torch.where(dec, hp1.e, hp1.e + h.v.abs() + h.e)))
    return lambda g: mul(g, f)


def layer2(p: dict, h1: TV) -> TV:
    zs = [dot(h1[:, k * HID:(k + 1) * HID], p[f"{n}.2.Wt"], p[f"{n}.2.b"], 65) for k, n in enumerate(("actor", "critic"))]
    return TV(torch.cat([z.v for z in zs], 1), torch.cat([z.e for z in zs], 1))


def heads(p: dict, h2: TV):
    m = dot(h2[:, :HID], p["actor.4.Wt"], p["actor.4.b"], 12)
    v = dot(h2[:, HID:], p["critic.4.Wt"], p["critic.4.b"], 12)
    return m[:, 0], m[:, 1], v[:, 0]


# ---- the loss derivatives (ppo_sample_derivs, in its order) --------------------------------------------------------------

def _share(x: TV, y: TV):
    """torch.max(x, y) backward share of x (1, 0.5 at ties, 0) and whether the bounds decide the comparison."""
    w = torch.where(x.v > y.v, 1.0, torch.where(x.v == y.v, 0.5, 0.0)).to(x.v.dtype)
    return w, (x.v - y.v).abs() > x.e + y.e


def sample_derivs(m0: TV, m1: TV, vv: TV, b: SimpleNamespace, cfg, B: int):
    """d[0..7] of every sample as TVs, the branches the fp64 evaluation took, and a per-sample flag of branches the bounds do
    not decide.  b: the mini-batch's stored rows in fp64 (act [n, 2], mu_old [n, 2], lp_old, v_old, R, A as a TV, sigma
    [2] and its snapshot so [2], exact fp32 values)."""
    z = m0.v
    C = const(LOG_SQRT_2PI, z)
    clip = cfg.clip_param
    inv_B = const(1.0 / B, z)
    sg = [TV(torch.full_like(z, float(b.sigma[a]))) for a in range(2)]
    so = [TV(torch.full_like(z, float(b.so[a]))) for a in range(2)]
    mus = (m0, m1)
    dd = [sub(TV(b.act[:, a]), mus[a]) for a in range(2)]
    var = [mul(sg[a], sg[a]) for a in range(2)]
    lps = [sub(sub(neg(div(mul(dd[a], dd[a]), scale(var[a], 2.0))), logf(sg[a])), C) for a in range(2)]
    lp = add(lps[0], lps[1])
    ratio = expf(sub(lp, TV(b.lp_old)))
    A = b.A
    # the ratio's region (below, inside, above the clip range) against both the kernel's fp32 and torch's fp64 bounds
    lo, hi = 1.0 - clip, 1.0 + clip
    lo32, hi32 = f32(1.0 - f32(clip)), f32(1.0 + f32(clip))
    margin = lambda t, t32: (ratio.v - t).abs() - abs(t32 - t)
    inside_r = (ratio.v >= lo) & (ratio.v <= hi)
    # inside the clip range both losses are -A ratio bit for bit (a tie: half each) whatever A's sign; outside, A's sign
    # orders them
    undecided = (margin(lo, lo32) <= ratio.e) | (margin(hi, hi32) <= ratio.e) | ((A.v.abs() <= A.e) & ~inside_r)
    clamped = TV(ratio.v.clamp(lo, hi), torch.where(inside_r, ratio.e, torch.full_like(z, abs(lo32 - lo))
                                                    .where(ratio.v < lo, torch.full_like(z, abs(hi32 - hi)))))
    su1 = mul(neg(A), ratio)
    su2 = mul(neg(A), clamped)
    w = torch.where(inside_r, 0.5, torch.where(su1.v > su2.v, 1.0, 0.0)).to(z.dtype)
    in_r = inside_r.to(z.dtype)
    dratio = add(mul(scale(inv_B, w), neg(A)), scale(mul(scale(inv_B, 1.0 - w), neg(A)), in_r))
    dlp = mul(dratio, ratio)
    d = [None] * 8
    for a in range(2):
        d[a] = mul(dlp, div(dd[a], var[a]))
        d[3 + a] = mul(dlp, sub(div(mul(mul(dd[a], dd[a]), sg[a]), mul(var[a], var[a])), div(TV(torch.ones_like(z)), sg[a])))
    vo, R = TV(b.v_old), TV(b.R)
    vcoef = const(cfg.value_loss_coef, z)
    if cfg.use_clipped_value_loss:
        dvo = sub(vv, vo)
        inside = dvo.v.abs() <= clip
        undecided |= (dvo.v.abs() - clip).abs() - abs(f32(clip) - clip) <= dvo.e
        vc_in = add(vo, dvo)
        vc_out = add(vo, TV(torch.where(dvo.v > 0, 1.0, -1.0).to(z.dtype) * clip, const(clip, z).e))
        vc = TV(torch.where(inside, vc_in.v, vc_out.v), torch.where(inside, vc_in.e, vc_out.e))
        r1, r2 = sub(vv, R), sub(vc, R)
        l1, l2 = mul(r1, r1), mul(r2, r2)
        wv, dec = _share(l1, l2)
        undecided |= ~inside & ~dec
        in_v = inside.to(z.dtype)

        def dv_of(wv_):
            return add(mul(scale(inv_B, wv_), scale(r1, 2.0)), scale(mul(scale(inv_B, 1.0 - wv_), scale(r2, 2.0)), in_v))
        dv = dv_of(wv)
        # inside the value clip vc = vv up to rounding, so l1 and l2 tie up to rounding and the share can be anything:
        # every share gives the same derivative up to |r2 - r1|, the hull of the three is the bound
        for alt in (0.0, 0.5, 1.0):
            da = dv_of(torch.full_like(z, alt))
            dv = TV(dv.v, torch.where(inside, torch.maximum(dv.e, (da.v - dv.v).abs() + da.e), dv.e))
        vl = TV(torch.maximum(l1.v, l2.v), torch.maximum(l1.e, l2.e))
    else:
        r = sub(vv, R)
        dv = mul(inv_B, scale(r, 2.0))
        rr = sub(R, vv)
        vl = mul(rr, rr)
    d[2] = mul(vcoef, dv)
    d[5] = TV(torch.maximum(su1.v, su2.v), torch.maximum(su1.e, su2.e))
    d[6] = vl
    e1e5 = const(1e-5, z)
    kls = []
    for a in range(2):
        ea = sub(TV(b.mu_old[:, a]), mus[a])
        kls.append(sub(add(logf(add(div(sg[a], so[a]), e1e5)), div(add(mul(so[a], so[a]), mul(ea, ea)), scale(var[a], 2.0))), TV(torch.full_like(z, 0.5))))
    d[7] = add(kls[0], kls[1])
    info = SimpleNamespace(ratio=ratio, A=A, w=w, in_r=in_r, lp=lp)
    if cfg.use_clipped_value_loss:
        info.dvo, info.l1, info.l2 = dvo, l1, l2
    return d, undecided, info


# ---- forward, backward and the gradient rows ------------------------------------------------------------------------------

def backward(p: dict, d, h1: TV, z1: TV | None, h2: TV, z2: TV, activation: str, h1_mask=None):
    """dz2 and dz1 [n, 128] from the sample derivatives (the grad kernels' order)."""
    w3a, w3c = p["actor.4.Wt"], p["critic.4.Wt"]
    dha = add(mul(d[0][:, None], TV(w3a[:, 0].expand_as(h2.v[:, :HID]))), mul(d[1][:, None], TV(w3a[:, 1].expand_as(h2.v[:, :HID]))))
    dhc = mul(d[2][:, None], TV(w3c[:, 0].expand_as(h2.v[:, HID:])))
    dh2 = TV(torch.cat([dha.v, dhc.v], 1), torch.cat([dha.e, dhc.e], 1))
    dz2 = act_grad(h2, z2, activation)(dh2)
    dh1s = [dot(dz2[:, k * HID:(k + 1) * HID], p[f"{n}.2.Wt"].t(), None, 65) for k, n in enumerate(("actor", "critic"))]
    dh1 = TV(torch.cat([t.v for t in dh1s], 1), torch.cat([t.e for t in dh1s], 1))
    dz1 = act_grad(h1, z1, activation, h1_mask)(dh1)
    return dz2, dz1


class Split:
    """Which samples each gradient row sums: tiles = ceil(B / 32), ctas = min(tiles, sms), CTA s takes tiles s, s + ctas, ..."""

    def __init__(self, B: int, sms: int):
        self.B, self.tiles = B, (B + ROWS - 1) // ROWS
        self.ctas = min(self.tiles, sms)
        self.kt = (self.tiles + self.ctas - 1) // self.ctas
        self.n_row = self.kt * ROWS                  # samples a CTA row sums through (zero rows included)
        self.n_red = self.n_row + self.ctas

    def grouped(self, t: torch.Tensor) -> torch.Tensor:
        """[B, ...] -> [ctas * kt * 32, ...], zero-padded, CTA s's samples contiguous (in sample order)."""
        pad = torch.zeros((self.kt * self.ctas * ROWS - t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
        x = torch.cat([t, pad]).reshape((self.kt, self.ctas, ROWS) + tuple(t.shape[1:]))
        return x.transpose(0, 1).reshape((-1,) + tuple(t.shape[1:]))


def _g(t: TV, split: Split) -> TV:
    return TV(split.grouped(t.v), split.grouped(t.e))


def _col(t: TV) -> TV:
    return TV(t.v[:, None], t.e[:, None])


def grad_sums(p, X, d, h1: TV, h2: TV, dz2: TV, dz1: TV, split: Split, per_row: bool, with_w1: bool = True) -> dict:
    """Every gradient tensor (state-dict names, out-major weights) and the three loss sums: per CTA row ([ctas, ...]) or
    reduced (+ the entropy term on std).  Values fp64, bounds for the kernel's order."""
    G, L = (split.ctas, split.n_row) if per_row else (1, split.n_red)
    g = lambda t: _g(t, split) if per_row else t
    B = h1.v.shape[0]
    one = TV(torch.ones(B, 1, dtype=h1.v.dtype, device=h1.v.device))
    out = {}
    s = lambda a, b: outer_sum(g(a), g(b), L, G)
    for k, n in enumerate(("actor", "critic")):
        cs = slice(k * HID, (k + 1) * HID)
        if with_w1:
            w = s(TV(X), dz1[:, cs])                                  # [G, D, 64]
            out[f"{n}.0.weight"] = TV(w.v.transpose(1, 2), w.e.transpose(1, 2))
        b1 = s(one, dz1[:, cs])
        out[f"{n}.0.bias"] = TV(b1.v[:, 0], b1.e[:, 0])
        w2 = s(h1[:, cs], dz2[:, cs])
        out[f"{n}.2.weight"] = TV(w2.v.transpose(1, 2), w2.e.transpose(1, 2))
        b2 = s(one, dz2[:, cs])
        out[f"{n}.2.bias"] = TV(b2.v[:, 0], b2.e[:, 0])
    dy = TV(torch.stack([d[0].v, d[1].v], 1), torch.stack([d[0].e, d[1].e], 1))
    w3 = s(h2[:, :HID], dy)
    out["actor.4.weight"] = TV(w3.v.transpose(1, 2), w3.e.transpose(1, 2))
    w3c = s(h2[:, HID:], _col(d[2]))
    out["critic.4.weight"] = TV(w3c.v.transpose(1, 2), w3c.e.transpose(1, 2))
    b3 = s(one, dy)
    out["actor.4.bias"] = TV(b3.v[:, 0], b3.e[:, 0])
    b3c = s(one, _col(d[2]))
    out["critic.4.bias"] = TV(b3c.v[:, 0], b3c.e[:, 0])
    st = s(one, TV(torch.stack([d[k].v for k in (3, 4, 5, 6, 7)], 1), torch.stack([d[k].e for k in (3, 4, 5, 6, 7)], 1)))
    out["std"] = TV(st.v[:, 0, :2], st.e[:, 0, :2])
    out["sums"] = TV(st.v[:, 0, 2:], st.e[:, 0, 2:])            # surrogate, value loss, KL
    if not per_row:
        out = {k: TV(t.v[0], t.e[0]) for k, t in out.items()}
    return out


def add_entropy(red: dict, p: dict, entropy_coef: float) -> dict:
    """wl_ppo_reduce_kernel's std column: g -= entropy_coef / sigma (two more roundings)."""
    sg = TV(p["std"])
    t = div(const(entropy_coef, p["std"]), sg)
    red = dict(red)
    red["std"] = sub(red["std"], t)
    return red


def reference(p: dict, X: torch.Tensor, b: SimpleNamespace, cfg, activation: str, h1_kernel: torch.Tensor | None = None,
              h1_mask: torch.Tensor | None = None):
    """The mini-batch through the network in fp64 with bounds.  X [B, D] fp64 (exact fp32 rows).  With h1_kernel (the
    kernel's own H1 rows [B, 128]), layer 1 is taken from it: its values exact, its mask the kernel's.  With h1_mask
    alone, layer 1 is evaluated but its derivative mask is h1_mask."""
    B = X.shape[0]
    if h1_kernel is None:
        z1 = layer1(p, X, activation)
        h1, mask = act(z1, activation), h1_mask
    else:
        z1, h1, mask = None, TV(h1_kernel), h1_kernel > 0
    z2 = layer2(p, h1)
    h2 = act(z2, activation)
    m0, m1, vv = heads(p, h2)
    d, undecided, info = sample_derivs(m0, m1, vv, b, cfg, B)
    dz2, dz1 = backward(p, d, h1, z1, h2, z2, activation, mask)
    return SimpleNamespace(z1=z1, h1=h1, z2=z2, h2=h2, m0=m0, m1=m1, vv=vv, d=d, undecided=undecided, info=info, dz2=dz2, dz1=dz1)


def undecided_units(z: TV) -> torch.Tensor:
    return z.v.abs() <= z.e


# ---- the mini-batch's stored rows and the margin batches -----------------------------------------------------------------

def minibatch(slab, ret, adv, perm, row0: int, B: int, blob: torch.Tensor, D: int, mean32=None, std32=None):
    """The stored rows of mini-batch perm[row0 : row0 + B] in fp64, A = (adv - mean) / (std + 1e-8) as the kernel forms it.
    mean32 / std32: the kernel's fp32 advantage statistics (d_state[4], [5]); default: the fp64 ones rounded to fp32, with
    the rounding in the bound."""
    from wheeledlab_b200.policy import blob_layout
    idx = perm[row0:row0 + B]
    a64 = adv.reshape(-1).double()
    m64, s64 = a64.mean(), a64.std()
    em, es = (0.0, 0.0) if mean32 is not None else (U * abs(float(m64)) * 2, U * float(s64) * 2)
    m = float(mean32) if mean32 is not None else float(m64)
    s = float(std32) if std32 is not None else float(s64)
    a = TV(a64[idx])
    A = div(sub(a, TV(torch.full_like(a.v, m), torch.full_like(a.v, em))),
            add(TV(torch.full_like(a.v, s), torch.full_like(a.v, es)), const(1e-8, a.v)))
    off, _ = blob_layout(D)
    sigma = blob[off[12]:off[12] + 2].double().cpu()
    X = slab.obs_in.reshape(-1, D)[idx].double()
    return X, SimpleNamespace(act=slab.actions.reshape(-1, 2)[idx].double(), mu_old=slab.mean.reshape(-1, 2)[idx].double(),
                              lp_old=slab.log_prob.reshape(-1)[idx].double(), v_old=slab.values.reshape(-1)[idx].double(),
                              R=ret.reshape(-1)[idx].double(), A=A, sigma=sigma, so=sigma)


def synthetic(D: int, n: int, seed: int, device, obs: torch.Tensor | None = None, activation: str = "relu"):
    """tests/test_ppo_wide_gpu.py's synthetic batch (rows collected by a perturbed copy of the network) on any device;
    obs [n, D] replaces its N(0, 1) rows when given."""
    from wheeledlab_b200.policy import pack_actor_critic
    torch.manual_seed(seed)
    A = torch.nn.ReLU if activation == "relu" else torch.nn.ELU
    mk = lambda out: torch.nn.Sequential(torch.nn.Linear(D, 64), A(), torch.nn.Linear(64, 64), A(), torch.nn.Linear(64, out)).to(device)
    actor, critic, std = mk(2), mk(1), torch.tensor((0.8, 1.2), device=device)
    g = torch.Generator(device=device).manual_seed(seed + 1)
    ap, cp = copy.deepcopy(actor), copy.deepcopy(critic)
    with torch.no_grad():
        for net in (ap, cp):
            for q in net.parameters():
                q.add_(0.15 * q.abs().mean() * torch.randn(q.shape, device=device, generator=g))
        sp = std * torch.tensor([1.15, 0.9], device=device)
        x = torch.randn(n, D, device=device, generator=g)
        if obs is not None:
            x = obs.reshape(n, D).to(device=device, dtype=torch.float32)
        mu = ap(x)
        val = cp(x).squeeze(-1) + 0.25 * torch.randn(n, device=device, generator=g)
        a = mu + sp * torch.randn(n, 2, device=device, generator=g)
        lp = torch.distributions.Normal(mu, sp).log_prob(a).sum(-1)
        ret = val + 0.5 * torch.randn(n, device=device, generator=g)
        adv = 0.3 + torch.randn(n, device=device, generator=g)
    blob = pack_actor_critic(actor, critic, std, D, device)
    slab = SimpleNamespace(obs_in=x.contiguous(), actions=a.contiguous(), values=val.contiguous(), log_prob=lp.contiguous(),
                           mean=mu.contiguous())
    return blob, slab, ret.contiguous(), adv.contiguous(), torch.randperm(n, device=device, generator=g)


def _free_point(lo: np.ndarray, hi: np.ndarray, b: float) -> float:
    """The point nearest b outside every open interval (lo_i, hi_i), at least a quarter of its gap's width (or, in an
    unbounded gap, one interval width) inside the gap."""
    o = np.argsort(lo)
    lo, hi = lo[o], hi[o]
    a = np.concatenate([[-np.inf], np.maximum.accumulate(hi)])
    c = np.concatenate([lo, [np.inf]])
    ok = c > a
    a, c = a[ok], c[ok]
    fa, fc = np.isfinite(a), np.isfinite(c)
    pad = float(np.max(hi - lo))
    q = np.where(fa & fc, 0.25 * (c - a), pad)
    x = np.clip(b, np.where(fa, a + q, -np.inf), np.where(fc, c - q, np.inf))
    return float(x[np.argmin(np.abs(x - b))])


def _shift_biases(z: TV, bias: torch.Tensor, k: float) -> torch.Tensor:
    """New fp32 biases [m] that put every sample's pre-activation at least k times its bound from 0."""
    zb = (z.v - bias).cpu().numpy()
    e = (z.e + 2 * gam(1) * bias.abs()).cpu().numpy()     # (slack for the bias's own change)
    out = bias.clone().cpu()
    for j in range(zb.shape[1]):
        lo, hi = -zb[:, j] - k * e[:, j], -zb[:, j] + k * e[:, j]
        out[j] = f32(_free_point(lo, hi, float(bias[j])))
    return out.to(bias.device)


def margin_batch(D: int, n: int, seed: int, device, row0: int = 0, B: int | None = None, obs=None, k: float = 4.0, cfg=None,
                 activation: str = "relu"):
    """The synthetic batch with every (sample, unit) of the checked mini-batch perm[row0 : row0 + B] at least k bounds from
    the ReLU edge in both layers (biases shifted), and its loss branches k bounds from their edges (the stored log_prob /
    values of the few that are not moved away).  Asserts its margins; returns (blob, slab, ret, adv, perm)."""
    from wheeledlab_b200.learner import PPOConfig
    cfg = cfg or PPOConfig()
    blob, slab, ret, adv, perm = synthetic(D, n, seed, device, obs, activation)
    apply_margins(blob, D, [(slab, ret, adv, perm)], row0, n if B is None else B, cfg, k, activation)
    return blob, slab, ret, adv, perm


def apply_margins(blob, D, batches, row0, B, cfg, k=4.0, activation="relu"):
    """margin_batch's edits in place for one blob and several ranks' batches [(slab, ret, adv, perm)]: the biases from every
    rank's mini-batch rows together, the loss edits per rank.  Asserts the margins."""
    from wheeledlab_b200.policy import blob_layout
    off, _ = blob_layout(D)
    if activation == "relu":
        X = torch.cat([minibatch(*bt, row0, B, blob, D)[0] for bt in batches])
        p = params(blob, D)
        z1 = layer1(p, X)
        for k_, o in enumerate((off[1], off[7])):
            blob[o:o + HID] = _shift_biases(z1[:, k_ * HID:(k_ + 1) * HID], p[("actor", "critic")[k_] + ".0.b"], 2 * k).float()
        p = params(blob, D)
        z2 = layer2(p, relu(layer1(p, X)))
        for k_, o in enumerate((off[3], off[9])):
            blob[o:o + HID] = _shift_biases(z2[:, k_ * HID:(k_ + 1) * HID], p[("actor", "critic")[k_] + ".2.b"], 2 * k).float()
    p = params(blob, D)
    for slab, ret, adv, perm in batches:
        for _ in range(8):
            X, b = minibatch(slab, ret, adv, perm, row0, B, blob, D)
            r = _loss_reference(p, X, b, cfg, activation)
            bad_r, bad_a, bad_v = _loss_margin(r, cfg, k, split=True)
            if not bool((bad_r | bad_a | bad_v).any()):
                break
            lp_old, vals, rows = slab.log_prob.reshape(-1), slab.values.reshape(-1), perm[row0:row0 + B]
            # the ratio up by 1 % (or 3 k bounds), away from 1 +- clip
            i = r.info
            lp_old[rows[bad_r]] -= torch.clamp(3 * k * i.ratio.e[bad_r] / i.ratio.v[bad_r], min=0.01).to(lp_old.dtype)
            lp_old[rows[bad_a]] = i.lp.v[bad_a].to(lp_old.dtype)     # A ~ 0: the ratio to ~1, where A's sign is moot
            vv, vo = r.vv.v[bad_v].to(vals.dtype), vals[rows[bad_v]]
            step = torch.clamp(3 * k * i.dvo.e[bad_v], min=0.02).to(vo.dtype)
            vals[rows[bad_v]] = vo - step * torch.where(vv > vo, 1.0, -1.0).to(vo.dtype)    # |v - v_old| up by step
        check_margins(blob, slab, ret, adv, perm, D, row0, B, cfg, k, activation)


def _loss_margin(r, cfg, k: float, split: bool = False):
    """Samples whose loss branches are not k bounds from their edges (the fp32 / fp64 gap of the clip constants included):
    the ratio near 1 +- clip, A near 0 outside the clip range, |v - v_old| near clip, or the two value losses outside it."""
    c = cfg.clip_param
    i = r.info
    rb = i.ratio.e + 1e-7 * i.ratio.v
    bad_r = ((i.ratio.v - (1 - c)).abs() <= k * rb) | ((i.ratio.v - (1 + c)).abs() <= k * rb)
    bad_a = (i.A.v.abs() <= k * i.A.e) & (i.in_r == 0) & ~bad_r
    bad_v = torch.zeros_like(bad_r)
    if cfg.use_clipped_value_loss:
        db = i.dvo.e + 1e-8
        bad_v = ((i.dvo.v.abs() - c).abs() <= k * db) | ((i.dvo.v.abs() > c) & ((i.l1.v - i.l2.v).abs() <= k * (i.l1.e + i.l2.e)))
    return (bad_r, bad_a, bad_v) if split else bad_r | bad_a | bad_v


def _loss_reference(p, X, b, cfg, activation):
    """The reference whose bounds the loss margins are measured in: for ReLU, from layer 1 rounded to fp32 and taken as
    exact, as the gradient kernel's check evaluates it from the kernel's own H1 (the bounds carried from X through three
    layers grow by sum |W| per layer and, on wide or large rows, leave no margin a loss branch could keep)."""
    if activation != "relu":
        return reference(p, X, b, cfg, activation)
    return reference(p, X, b, cfg, activation, h1_kernel=relu(layer1(p, X)).v.float().double())


def check_margins(blob, slab, ret, adv, perm, D, row0, B, cfg, k, activation="relu"):
    """Every (sample, unit) of both layers at least k bounds (carried from X) from the ReLU edge, and every loss branch of
    the mini-batch at least k bounds (``_loss_reference``'s) from its edge.  Returns the reference from X."""
    X, b = minibatch(slab, ret, adv, perm, row0, B, blob, D)
    p = params(blob, D)
    r = reference(p, X, b, cfg, activation)
    if activation == "relu":
        for name, z in (("layer 1", r.z1), ("layer 2", r.z2)):
            ratio = (z.e / z.v.abs()).max().item()
            assert ratio * k <= 1, f"{name}: a pre-activation is within {1 / ratio:.3g} bounds of 0"
    bad = _loss_margin(_loss_reference(p, X, b, cfg, activation), cfg, k)
    assert not bool(bad.any()), f"{int(bad.sum())} samples with a loss branch within {k} bounds of its edge"
    return r


def branch_counts(r, cfg) -> dict:
    i = r.info
    lo, hi = 1 - cfg.clip_param, 1 + cfg.clip_param
    ratio, A = i.ratio.v, i.A.v
    out = {"ratio > 1+clip, A > 0": (ratio > hi) & (A > 0), "ratio > 1+clip, A < 0": (ratio > hi) & (A < 0),
           "ratio < 1-clip, A > 0": (ratio < lo) & (A > 0), "ratio < 1-clip, A < 0": (ratio < lo) & (A < 0),
           "ratio inside the clip range": (ratio >= lo) & (ratio <= hi)}
    if cfg.use_clipped_value_loss:
        out.update({"value clipped": i.dvo.v.abs() > cfg.clip_param, "value unclipped": i.dvo.v.abs() <= cfg.clip_param,
                    "clipped value loss larger": i.l2.v > i.l1.v, "plain value loss larger": i.l1.v > i.l2.v})
    return {k: int(v.sum()) for k, v in out.items()}


def worst(got: torch.Tensor, want: TV, slack: float = 2.0 ** -20):
    """(every |got - want| <= bound, largest |got - want| / bound, flat index of it); a zero bound admits only a zero error.
    The bound is widened by 2^-20 of itself for the fp64 evaluation's own rounding."""
    err = (got.double() - want.v).abs()
    bnd = want.e * (1 + slack)
    ratio = torch.where(bnd > 0, err / bnd.clamp(min=1e-300), torch.where(err > 0, math.inf, 0.0))
    k = int(ratio.reshape(-1).argmax())
    return bool((err <= bnd).all()), float(ratio.reshape(-1)[k]), k


# ---- the fp32 emulation of the kernels' orders (CPU tests only) -------------------------------------------------------------

def _fma(a, b, c):
    return (a.double() * b.double() + c.double()).float()


def emulate(blob, D, X32, b32, cfg, split: Split, activation: str):
    """The kernels' fp32 operations in their order on the CPU: layer 1 (wide: chunked two-level sum; narrow: one chain),
    layer 2, the heads' butterfly, ppo_sample_derivs, back-propagation, the CTA rows and the reduced row."""
    from wheeledlab_b200.policy import actor_critic_state_dict
    sd = {k: v.float() for k, v in actor_critic_state_dict(blob, D).items()}
    n = X32.shape[0]
    f = lambda t: t.float()

    def lin_chain(x, Wt, bias, chunks):
        acc = bias.expand(x.shape[0], -1).clone()
        for c0, c1 in chunks:
            part = torch.zeros_like(acc)
            for j in range(c0, c1):
                part = _fma(x[:, j:j + 1], Wt[j:j + 1], part)
            acc = acc + part
        return acc

    def chain(x, Wt, bias):
        acc = bias.expand(x.shape[0], -1).clone()
        for j in range(x.shape[1]):
            acc = _fma(x[:, j:j + 1], Wt[j:j + 1], acc)
        return acc
    actf = (lambda z: torch.relu(z)) if activation == "relu" else (lambda z: torch.where(z > 0, z, torch.expm1(z)))
    gradf = (lambda h: (h > 0).float()) if activation == "relu" else (lambda h: torch.where(h > 0, torch.ones_like(h), h + 1.0))
    z1 = []
    for net in ("actor", "critic"):
        Wt, bias = sd[f"{net}.0.weight"].t(), sd[f"{net}.0.bias"]
        if activation == "relu":
            z1.append(lin_chain(X32, Wt, bias, [(c, min(c + KC, D)) for c in range(0, D, KC)]))
        else:
            z1.append(chain(X32, Wt, bias))
    z1 = torch.cat(z1, 1)
    h1 = actf(z1)
    h2 = actf(torch.cat([chain(h1[:, k * HID:(k + 1) * HID], sd[f"{nm}.2.weight"].t(), sd[f"{nm}.2.bias"])
                         for k, nm in enumerate(("actor", "critic"))], 1))

    def head(h, Wt, bias):
        parts = []
        for q in range(8):
            acc = torch.zeros(n, Wt.shape[1])
            for kk in range(8):
                j = 8 * q + kk
                acc = _fma(h[:, j:j + 1], Wt[j:j + 1], acc)
            parts.append(acc)
        for x in (1, 2, 4):
            parts = [parts[q] + parts[q ^ x] for q in range(8)]
        return parts[0] + bias
    m = head(h2[:, :HID], sd["actor.4.weight"].t(), sd["actor.4.bias"])
    vv = head(h2[:, HID:], sd["critic.4.weight"].t(), sd["critic.4.bias"])[:, 0]
    m0, m1 = m[:, 0], m[:, 1]
    # ppo_sample_derivs in fp32
    sg, so = f(b32.sigma), f(b32.sigma)
    clip = torch.tensor(cfg.clip_param, dtype=torch.float32)
    inv_B = torch.tensor(1.0 / split.B, dtype=torch.float32)
    C = torch.tensor(LOG_SQRT_2PI, dtype=torch.float32)
    act_, mo = f(b32.act), f(b32.mu_old)
    A = f(b32.A32)
    d0, d1 = act_[:, 0] - m0, act_[:, 1] - m1
    var0, var1 = sg[0] * sg[0], sg[1] * sg[1]
    lp = ((-(d0 * d0) / (2.0 * var0) - torch.log(sg[0])) - C) + ((-(d1 * d1) / (2.0 * var1) - torch.log(sg[1])) - C)
    ratio = torch.exp(lp - f(b32.lp_old))
    lo, hi = 1.0 - clip, 1.0 + clip
    su1, su2 = -A * ratio, -A * torch.minimum(torch.maximum(ratio, lo), hi)
    w = torch.where(su1 > su2, 1.0, torch.where(su1 == su2, 0.5, 0.0))
    in_r = ((ratio >= lo) & (ratio <= hi)).float()
    dratio = (w * inv_B) * -A + ((1.0 - w) * inv_B) * -A * in_r
    dlp = dratio * ratio
    d = [None] * 8
    d[0], d[1] = dlp * (d0 / var0), dlp * (d1 / var1)
    d[3] = dlp * ((d0 * d0) * sg[0] / (var0 * var0) - 1.0 / sg[0])
    d[4] = dlp * ((d1 * d1) * sg[1] / (var1 * var1) - 1.0 / sg[1])
    vo, R = f(b32.v_old), f(b32.R)
    dvo = vv - vo
    vc = vo + torch.minimum(torch.maximum(dvo, -clip), clip)
    l1, l2 = (vv - R) * (vv - R), (vc - R) * (vc - R)
    wv = torch.where(l1 > l2, 1.0, torch.where(l1 == l2, 0.5, 0.0))
    in_v = ((dvo >= -clip) & (dvo <= clip)).float()
    dv = (wv * inv_B) * (2.0 * (vv - R)) + ((1.0 - wv) * inv_B) * (2.0 * (vc - R)) * in_v
    d[2] = torch.tensor(cfg.value_loss_coef, dtype=torch.float32) * dv
    d[5], d[6] = torch.maximum(su1, su2), torch.maximum(l1, l2)
    e0, e1 = mo[:, 0] - m0, mo[:, 1] - m1
    e5 = torch.tensor(1e-5, dtype=torch.float32)
    d[7] = ((torch.log(sg[0] / so[0] + e5) + (so[0] * so[0] + e0 * e0) / (2.0 * var0)) - 0.5) \
        + ((torch.log(sg[1] / so[1] + e5) + (so[1] * so[1] + e1 * e1) / (2.0 * var1)) - 0.5)
    w3a, w3c = sd["actor.4.weight"].t(), sd["critic.4.weight"].t()
    dh = torch.cat([d[0][:, None] * w3a[:, 0] + d[1][:, None] * w3a[:, 1], d[2][:, None] * w3c[:, 0]], 1)
    dz2 = dh * gradf(h2)
    zero = torch.zeros(HID)
    dh1 = torch.cat([chain(dz2[:, k * HID:(k + 1) * HID], sd[f"{nm}.2.weight"], zero) for k, nm in enumerate(("actor", "critic"))], 1)
    dz1 = dh1 * gradf(h1)

    # the CTA rows: per split, fmaf / add chains in sample order; then the reduce in CTA order
    def rows_of(a, bb, L_fma=True):
        ga, gb = split.grouped(a).reshape(split.ctas, split.n_row, -1), split.grouped(bb).reshape(split.ctas, split.n_row, -1)
        acc = torch.zeros(split.ctas, ga.shape[2], gb.shape[2])
        for s in range(split.n_row):
            if L_fma:
                acc = _fma(ga[:, s, :, None], gb[:, s, None, :], acc)
            else:
                acc = acc + gb[:, s, None, :]
        return acc
    one = torch.ones(n, 1)
    out = {}
    for k, nm in enumerate(("actor", "critic")):
        cs = slice(k * HID, (k + 1) * HID)
        out[f"{nm}.0.weight"] = rows_of(X32, dz1[:, cs]).transpose(1, 2)
        out[f"{nm}.0.bias"] = rows_of(one, dz1[:, cs], False)[:, 0]
        out[f"{nm}.2.weight"] = rows_of(h1[:, cs], dz2[:, cs]).transpose(1, 2)
        out[f"{nm}.2.bias"] = rows_of(one, dz2[:, cs], False)[:, 0]
    dy = torch.stack([d[0], d[1]], 1)
    out["actor.4.weight"] = rows_of(h2[:, :HID], dy).transpose(1, 2)
    out["critic.4.weight"] = rows_of(h2[:, HID:], d[2][:, None]).transpose(1, 2)
    out["actor.4.bias"] = rows_of(one, dy, False)[:, 0]
    out["critic.4.bias"] = rows_of(one, d[2][:, None], False)[:, 0]
    st = rows_of(one, torch.stack([d[k] for k in (3, 4, 5, 6, 7)], 1), False)[:, 0]
    out["std"], out["sums"] = st[:, :2], st[:, 2:]
    red = {}
    for key, t in out.items():
        acc = torch.zeros_like(t[0])
        for r_ in range(split.ctas):
            acc = acc + t[r_]
        red[key] = acc
    red["std"] = red["std"] - torch.tensor(cfg.entropy_coef, dtype=torch.float32) / sg
    return SimpleNamespace(z1=z1, h1=h1, h2=h2, dz2=dz2, dz1=dz1, d=d, rows=out, red=red, ratio=ratio)


# ---- tests --------------------------------------------------------------------------------------------------------------

def _emulation_case(D, n, sms, seed, activation, margins):
    from wheeledlab_b200.learner import PPOConfig
    cfg = PPOConfig()
    if margins:
        blob, slab, ret, adv, perm = margin_batch(D, n, seed, "cpu", cfg=cfg, activation=activation)
    else:
        blob, slab, ret, adv, perm = synthetic(D, n, seed, "cpu", activation=activation)
    X, b = minibatch(slab, ret, adv, perm, 0, n, blob, D)
    a64 = adv.reshape(-1).double()
    m32, s32 = f32(float(a64.mean())), f32(float(a64.std()))
    b.A32 = ((adv.reshape(-1)[perm].float() - m32) / (torch.tensor(s32) + torch.tensor(1e-8, dtype=torch.float32)))
    em = emulate(blob, D, X.float(), b, cfg, Split(n, sms), activation)
    p = params(blob, D)
    r = reference(p, X, b, cfg, activation)
    return cfg, p, X, r, em


@pytest.mark.parametrize("D,n,sms,seed,activation", [(1, 100, 3, 0, "relu"), (33, 77, 2, 1, "relu"), (100, 257, 4, 2, "relu"),
                                                     (14, 100, 3, 3, "elu"), (5, 31, 2, 4, "elu")])
def test_bounds_hold_and_are_not_vacuous_against_the_fp32_emulation(D, n, sms, seed, activation):
    """On margin batches every emulated fp32 value lies within its bound of the fp64 value, the largest ratio is well
    above 0, and the emulation's masks and branches equal the fp64 ones."""
    cfg, p, X, r, em = _emulation_case(D, n, sms, seed, activation, margins=True)
    split = Split(n, sms)
    ratios = {}
    checks = [("z1", em.z1, r.z1), ("h2", em.h2, r.h2), ("dz2", em.dz2, r.dz2), ("dz1", em.dz1, r.dz1)]
    checks += [(f"d[{k}]", em.d[k], r.d[k]) for k in range(8)]
    rows = grad_sums(p, X, r.d, r.h1, r.h2, r.dz2, r.dz1, split, per_row=True)
    red = add_entropy(grad_sums(p, X, r.d, r.h1, r.h2, r.dz2, r.dz1, split, per_row=False), p, cfg.entropy_coef)
    checks += [(f"row {k}", em.rows[k], rows[k]) for k in rows] + [(f"reduced {k}", em.red[k], red[k]) for k in red]
    for name, got, want in checks:
        ok, q, _ = worst(got, want)
        assert ok, f"{name}: |err| / bound {q:.3g}"
        ratios[name] = q
    print(f"\nD={D} n={n} {activation}: largest |err| / bound " + ", ".join(f"{k} {v:.2g}" for k, v in ratios.items()))
    assert max(ratios.values()) > 1e-2, f"the bounds are vacuous: largest ratio {max(ratios.values()):.3g}"
    if activation == "relu":
        assert torch.equal(em.h1 > 0, r.z1.v > 0) and torch.equal(em.h2 > 0, r.z2.v > 0)
    assert not bool(r.undecided.any())


def test_margin_batch_keeps_every_branch_and_asserts_its_margins():
    """A 689-wide margin batch of 4096 rows: margins of 4 bounds hold in both layers and the loss, every PPO branch is
    still taken by more than 100 samples, and a batch without the margins fails the margin check."""
    from wheeledlab_b200.learner import PPOConfig
    cfg = PPOConfig()
    D, n = 689, 4096
    blob, slab, ret, adv, perm = margin_batch(D, n, 5, "cpu", cfg=cfg)
    r = check_margins(blob, slab, ret, adv, perm, D, 0, n, cfg, 4.0)
    counts = branch_counts(r, cfg)
    for name, c in counts.items():
        assert c > 100, f"the margin batch misses the branch {name} ({c})"
    raw = synthetic(D, n, 5, "cpu")
    with pytest.raises(AssertionError, match="bounds of 0|loss branch"):
        check_margins(*raw, D, 0, n, cfg, 4.0)


def test_split_groups_tiles_by_cta():
    s = Split(32 * 7 + 5, 3)                              # 8 tiles over 3 CTAs: 0 3 6 | 1 4 7 | 2 5
    assert (s.tiles, s.ctas, s.kt, s.n_row, s.n_red) == (8, 3, 3, 96, 99)
    g = s.grouped(torch.arange(s.B)).reshape(3, 3, 32)
    assert g[0, :, 0].tolist() == [0, 96, 192] and g[1, :, 0].tolist() == [32, 128, 224] and g[2, :, 0].tolist() == [64, 160, 0]
    assert g[1, 2, :5].tolist() == [224, 225, 226, 227, 228] and g[1, 2, 5:].abs().sum() == 0
