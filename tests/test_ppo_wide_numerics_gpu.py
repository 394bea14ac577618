"""Each kernel of the PPO update against fp64 per element, with the rounding-error bounds of
tests/test_ppo_wide_numerics_cpu.py (its docstring derives every chain length).

The wide (ReLU) update, ``wl_ppo_update_wide``, leaves its last mini-batch's intermediates in the workspace: the reduced
row, one gradient row per CTA, H1 and dZ1.  Each is checked on its own, on margin batches (every ReLU pre-activation and
every loss branch at least 4 bounds from its edge, so fp32 and fp64 take the same masks and branches):

* ``wl_ppo_wide_fwd_kernel``: H1 against relu(z) in fp64; rows past B are relu(b1) bit for bit;
* ``wl_ppo_wide_grad_kernel``: dZ1 and the CTA rows (dW2, dW3, biases, dsigma, loss sums) from the kernel's own H1;
  rows past B of dZ1 are zero;
* ``wl_ppo_wide_dw1_kernel``: each CTA row's dW1 against the sum over its tiles s, s + ctas, ... of X[perm]^T dZ1 (the
  kernel's dZ1), then the reduced dW1;
* the whole reduced row against fp64 autograd (tests/ppo_reference_relu.py) with the bound carried from X.

Updates run with learning rate 0, so every mini-batch sees the packed weights and the last one (row0 > 0) is checked
against them.  The narrow (ELU) update, ``wl_ppo_update``, gets the CTA-row and reduced-row checks.  The obs_dim 689 case
of DESIGN 6j (N(0, 1) rows, B = 8192, no margins) is rebuilt to settle which sum its 1.5e-3 gradient gap comes from.
Every check prints the largest |err| / bound it saw (``pytest -s``)."""
import pytest
import torch

from test_ppo_wide_numerics_cpu import (HID, ROWS, Split, TV, add_entropy, apply_margins, branch_counts, check_margins,
                                        grad_sums, layer1, margin_batch, minibatch, outer_sum, params, reference, relu,
                                        synthetic, undecided_units, worst)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SEEDS = [0, 1, 2]
K = 4.0                                              # margin, in bounds


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _a256(x):
    return (x + 255) & ~255


def _layout(D, batch, mb, wide):
    """wl_api.cu's ppo_rows_layout / ppo_wide_workspace restated; the total must be what the library reports."""
    from wheeledlab_b200._lib import lib
    from wheeledlab_b200.policy import blob_layout
    _, blob_floats = blob_layout(D)
    rowlen = (blob_floats + 3 + 3) & ~3
    tiles = (batch // mb + ROWS - 1) // ROWS
    ctas = min(tiles, _sms())
    norm_parts = (rowlen + 255) // 256
    norm_off = _a256(4 * rowlen)
    rows_off = _a256(norm_off + 8 * norm_parts)
    total = rows_off + 4 * rowlen * ctas
    lay = dict(blob_floats=blob_floats, rowlen=rowlen, tiles=tiles, ctas=ctas, rows_off=rows_off)
    if wide:
        hb = 4 * 2 * HID * ROWS * tiles
        lay["h1_off"] = _a256(total)
        lay["dz_off"] = _a256(lay["h1_off"] + hb)
        total = lay["dz_off"] + hb
        assert total == lib.wl_ppo_wide_workspace_bytes(D, batch, mb), "the wide workspace layout changed"
    else:
        assert total == lib.wl_ppo_workspace_bytes(D, batch, mb), "the workspace layout changed"
    return lay


def _f32(ws, off, n):
    return ws[off:off + 4 * n].view(torch.float32)


def _row_tensors(rows, D, blob_floats):
    """Gradient rows [r, rowlen] in blob layout -> the state-dict tensors [r, ...] (weights out-major) and the loss sums."""
    from wheeledlab_b200.policy import blob_layout
    off, _ = blob_layout(D)
    r = rows.shape[0]
    seg = lambda o, n: rows[:, o:o + n]
    out = {}
    for k, net in enumerate(("actor", "critic")):
        o, nout = off[6 * k:6 * k + 6], (2, 1)[k]
        out[f"{net}.0.weight"] = seg(o[0], D * HID).reshape(r, D, HID).transpose(1, 2)
        out[f"{net}.0.bias"] = seg(o[1], HID)
        out[f"{net}.2.weight"] = seg(o[2], HID * HID).reshape(r, HID, HID).transpose(1, 2)
        out[f"{net}.2.bias"] = seg(o[3], HID)
        out[f"{net}.4.weight"] = seg(o[4], HID * nout).reshape(r, HID, nout).transpose(1, 2)
        out[f"{net}.4.bias"] = seg(o[5], nout)
    out["std"] = seg(off[12], 2)
    out["sums"] = seg(blob_floats, 3)
    return out


def _run(blob, D, slab, ret, adv, perm, cfg, activation):
    from wheeledlab_b200.learner import FusedPPO
    ppo = FusedPPO(blob, D, cfg, activation=activation)
    ppo.update(slab, ret, adv, perm)
    torch.cuda.synchronize()
    return ppo


def _zero_lr(mb):
    from wheeledlab_b200.learner import PPOConfig
    return PPOConfig(num_learning_epochs=1, num_mini_batches=mb, learning_rate=0.0, schedule="fixed")


def _report(tag, ratios):
    print(f"\n{tag}: largest |err| / bound " + ", ".join(f"{k} {v:.3g}" for k, v in ratios.items()))
    for k, v in ratios.items():
        assert v <= 1.0, f"{tag}: {k} {v}"


def _check(name, got, want, ratios):
    ok, q, i = worst(got, want)
    ratios[name] = max(ratios.get(name, 0.0), q)
    assert ok, f"{name}: |err| / bound {q:.3g} at flat index {i} (got {got.reshape(-1)[i].item()!r}, fp64 {want.v.reshape(-1)[i].item()!r})"


def _rows_of(kind, D, n, seed):
    """[n, D] observation rows: N(0, 1) (None: the synthetic recipe's own), N(0, 1) * 100 + 50, or rows of an Elevation
    (256 envs) or camera Visual (64 envs) rollout of a ReLU policy."""
    if kind == "normal":
        return None
    if kind == "shifted":
        g = torch.Generator(device=DEV).manual_seed(seed + 11)
        return torch.randn(n, D, device=DEV, generator=g) * 100 + 50
    import wheeledlab_b200 as wl
    from wheeledlab_b200.policy import FusedPolicyRollout
    envs = 256 if kind == "elevation" else 64
    spec = wl.elevation_task(num_envs=envs, seed=seed) if kind == "elevation" else wl.visual_task(num_envs=envs, seed=seed, camera="aug")
    assert spec.obs_dim == D
    blob = synthetic(D, 2, seed + 5, DEV)[0]
    sim = wl.WheeledSim(spec, DEV); sim.startup(); sim.reset(None, 0)
    slab = FusedPolicyRollout(sim, blob, -(-n // envs), activation="relu").capture(0).run()
    return slab.obs_in.reshape(-1, D)[:n].clone()


# ---- the wide update, kernel by kernel --------------------------------------------------------------------------------

# (obs_dim, mini-batch size, mini-batches, rows).  Sizes in SMs are taken from the device: 32 SMs rows fill every CTA with
# one tile, one more row starts a second tile on CTA 0, and 3 SMs + 5 tiles (the last one partial) give CTAs 0-4 four
# tiles and the rest three.  obs_dim 32 and 64 fill their last layer-1 chunk and dW1 block exactly; 4096 is the limit.
WIDE = [(1, 4231, 1, "normal"), (4, 31, 2, "normal"), (31, 33, 1, "normal"), (32, "32sms", 1, "normal"),
        (33, "32sms+1", 2, "normal"), (64, 1, 2, "normal"), (65, 16384, 1, "normal"), (689, 16384, 1, "normal"),
        (689, 4231, 2, "elevation"), (3208, "3sms+5", 1, "visual"), (4093, 4231, 1, "shifted"), (4096, "3sms+5", 2, "normal")]


def _B(spec):
    s = _sms()
    return {"32sms": 32 * s, "32sms+1": 32 * s + 1, "3sms+5": 32 * (3 * s + 5) - 9}.get(spec, spec)


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("D,Bspec,mb,rows", WIDE, ids=[f"D{c[0]}-B{c[1]}-mb{c[2]}-{c[3]}" for c in WIDE])
def test_wide_update_kernels_against_fp64(D, Bspec, mb, rows, seed):
    _need_gpu()
    B = _B(Bspec)
    n, row0 = mb * B, (mb - 1) * B
    cfg = _zero_lr(mb)
    blob, slab, ret, adv, perm = margin_batch(D, n, seed, DEV, row0=row0, B=B, obs=_rows_of(rows, D, n, seed), k=K, cfg=cfg)
    blob0 = blob.clone()
    ppo = _run(blob, D, slab, ret, adv, perm, cfg, "relu")
    assert torch.equal(blob, blob0), "a zero learning rate moved the blob"
    lay = _layout(D, n, mb, wide=True)
    split = Split(B, _sms())
    assert (split.tiles, split.ctas) == (lay["tiles"], lay["ctas"])
    ws = ppo.workspace
    rowlen, T32 = lay["rowlen"], lay["tiles"] * ROWS
    rows_k = _f32(ws, lay["rows_off"], rowlen * lay["ctas"]).view(lay["ctas"], rowlen)
    H1 = _f32(ws, lay["h1_off"], T32 * 2 * HID).view(T32, 2 * HID)
    dZ1 = _f32(ws, lay["dz_off"], T32 * 2 * HID).view(T32, 2 * HID)
    red_k = _f32(ws, 0, rowlen)                       # the reduced row, loss sums included
    p = params(blob, D)
    ratios = {}

    # forward: H1 against relu(z1), masks equal (the margins), the tail rows relu(b1) bit for bit
    st = ppo.state
    X, b = minibatch(slab, ret, adv, perm, row0, B, blob, D, mean32=st[4].item(), std32=st[5].item())
    z1 = layer1(p, X)
    _check("fwd H1", H1[:B], relu(z1), ratios)
    flips = (H1[:B] > 0) != (z1.v > 0)
    assert not bool(flips.any()), f"{int(flips.sum())} layer-1 mask disagreements on a margin batch"
    b1 = torch.cat([p["actor.0.b"], p["critic.0.b"]]).float()
    tail = torch.where(b1 > 0, b1, torch.zeros_like(b1)).expand(T32 - B, -1)
    assert torch.equal(H1[B:].view(torch.int32), tail.contiguous().view(torch.int32)), "H1 rows past B are not relu(b1)"

    # the gradient kernel from the kernel's own H1
    r = reference(p, X, b, cfg, "relu", h1_kernel=H1[:B].double())
    excl = r.undecided | undecided_units(r.z2).any(1)
    assert int(excl.sum()) == 0, f"{int(excl.sum())} samples the bounds cannot decide on a margin batch"
    _check("grad dZ1", dZ1[:B], r.dz1, ratios)
    assert not bool(dZ1[B:].any()), "dZ1 rows past B are not zero"
    got = _row_tensors(rows_k, D, lay["blob_floats"])
    want = grad_sums(p, X, r.d, r.h1, r.h2, r.dz2, r.dz1, split, per_row=True, with_w1=False)
    for k, t in want.items():
        _check(f"grad row {k}", got[k], t, ratios)

    # dW1 from X[perm] and the kernel's dZ1: a pure sum per CTA row (its tiles s, s + ctas, ...), then the reduced row
    Z = TV(dZ1[:B].double())
    for k, net in enumerate(("actor", "critic")):
        cs = slice(k * HID, (k + 1) * HID)
        w = outer_sum(_grouped(TV(X), split), _grouped(Z[:, cs], split), split.n_row, split.ctas)
        _check("dw1 row", got[f"{net}.0.weight"], TV(w.v.transpose(1, 2), w.e.transpose(1, 2)), ratios)
        w = outer_sum(TV(X), Z[:, cs], split.n_red)
        _check("dw1 reduced", _row_tensors(red_k[None], D, lay["blob_floats"])[f"{net}.0.weight"][0], TV(w.v[0].t(), w.e[0].t()), ratios)
    red_ref = add_entropy(grad_sums(p, X, r.d, r.h1, r.h2, r.dz2, r.dz1, split, per_row=False, with_w1=False), p, cfg.entropy_coef)
    red_got = {k: v[0] for k, v in _row_tensors(red_k[None], D, lay["blob_floats"]).items()}
    for k, t in red_ref.items():
        _check(f"reduce {k}", red_got[k], t, ratios)

    # the whole reduced row against fp64 autograd, the bound carried from X: where that bound decides every loss branch
    # (on N(0, 1) rows; through three layers of rollout or shifted rows it grows too wide to decide some of them)
    ran = _whole_gradient(blob0, D, slab, ret, adv, perm, cfg, "relu", red_got, split, row0, B, ratios)
    print(f"\nwhole reduced row against fp64 autograd: {'checked' if ran else 'not decided by the bounds carried from X'}")
    _report(f"wide D={D} B={B} mb={mb} {rows} seed={seed}", ratios)


def _grouped(t, split):
    return TV(split.grouped(t.v), split.grouped(t.e))


def _whole_gradient(blob0, D, slab, ret, adv, perm, cfg, activation, red_got, split, row0, B, ratios):
    """Every tensor of the reduced row and the three loss sums against fp64 autograd, per element, within the bound the
    tracker carries from the observation rows (fp64 advantage statistics; their fp32 rounding is in the bound)."""
    from ppo_reference_relu import torch_ppo
    X, b = minibatch(slab, ret, adv, perm, row0, B, blob0, D)
    p = params(blob0, D)
    r = reference(p, X, b, cfg, activation)
    if bool(r.undecided.any()):
        return False
    bound = add_entropy(grad_sums(p, X, r.d, r.h1, r.h2, r.dz2, r.dz1, split, per_row=False), p, cfg.entropy_coef)
    t64 = torch_ppo(blob0.clone(), D, cfg, torch.float64, activation)
    t64.update(slab.obs_in, slab.actions, slab.values, slab.log_prob, slab.mean, ret, adv, perm, keep_grads=True)
    tr = t64.trace[-1]
    g64 = dict(tr["grads"])
    g64["sums"] = torch.tensor([tr["surrogate"], tr["value_function"], tr["kl"]], dtype=torch.float64, device=DEV) * B
    for k, t in bound.items():
        _check(f"whole {k}", red_got[k], TV(g64[k].reshape(t.v.shape), t.e), ratios)
    return True


# ---- the narrow (ELU) update ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("D,B", [(1, 17), (14, 17), (16, 17), (1, 16384), (14, 16384), (16, 16384)])
def test_narrow_update_rows_against_fp64(D, B, seed):
    """wl_ppo_update: ELU's derivative is continuous, so only the loss branches need margins.  Every CTA row (dW1
    included: the narrow kernel sums it in registers) and the reduced row per element, and the reduced row against fp64
    autograd."""
    _need_gpu()
    cfg = _zero_lr(1)
    blob, slab, ret, adv, perm = margin_batch(D, B, seed, DEV, k=K, cfg=cfg, activation="elu")
    blob0 = blob.clone()
    ppo = _run(blob, D, slab, ret, adv, perm, cfg, "elu")
    lay = _layout(D, B, 1, wide=False)
    split = Split(B, _sms())
    rows_k = _f32(ppo.workspace, lay["rows_off"], lay["rowlen"] * lay["ctas"]).view(lay["ctas"], lay["rowlen"])
    st = ppo.state
    X, b = minibatch(slab, ret, adv, perm, 0, B, blob, D, mean32=st[4].item(), std32=st[5].item())
    p = params(blob, D)
    r = reference(p, X, b, cfg, "elu")
    assert not bool(r.undecided.any())
    ratios = {}
    got = _row_tensors(rows_k, D, lay["blob_floats"])
    for k, t in grad_sums(p, X, r.d, r.h1, r.h2, r.dz2, r.dz1, split, per_row=True).items():
        _check(f"row {k}", got[k], t, ratios)
    red_got = {k: v[0] for k, v in _row_tensors(_f32(ppo.workspace, 0, lay["rowlen"])[None], D, lay["blob_floats"]).items()}
    for k, t in add_entropy(grad_sums(p, X, r.d, r.h1, r.h2, r.dz2, r.dz1, split, per_row=False), p, cfg.entropy_coef).items():
        _check(f"reduce {k}", red_got[k], t, ratios)
    assert _whole_gradient(blob0, D, slab, ret, adv, perm, cfg, "elu", red_got, split, 0, B, ratios)
    _report(f"narrow D={D} B={B} seed={seed}", ratios)


# ---- DESIGN 6j / 10.8: the 1.5e-3 gap at obs_dim 689 ------------------------------------------------------------------

@pytest.mark.parametrize("seed", [703, 704, 705])
def test_obs689_gradient_gap_is_the_relu_edge(seed):
    """The DESIGN 6j case without margins: obs_dim 689, N(0, 1) rows, one rank, one mini-batch of 8192 (the data-parallel
    test's recipe; seed 703 is its R = 2 seed).  Counts the layer-1 mask disagreements of the fused H1 and of torch fp32
    with fp64, then recomputes the fp64 gradient under the kernel's masks (layer 1 from H1 > 0; layer 2 where the bound
    decides it, the hull of both where it does not) and requires the fused reduced row within the per-element bound of it."""
    _need_gpu()
    from ppo_reference_relu import torch_ppo
    from wheeledlab_b200.learner import PPOConfig
    D, B = 689, 8192
    cfg = PPOConfig(num_learning_epochs=1, num_mini_batches=1)
    blob, slab, ret, adv, perm = synthetic(D, B, seed, DEV)
    blob0 = blob.clone()
    ppo = _run(blob, D, slab, ret, adv, perm, cfg, "relu")
    lay = _layout(D, B, 1, wide=True)
    split = Split(B, _sms())
    H1 = _f32(ppo.workspace, lay["h1_off"], B * 2 * HID).view(B, 2 * HID)
    red_got = {k: v[0] for k, v in _row_tensors(_f32(ppo.workspace, 0, lay["rowlen"])[None], D, lay["blob_floats"]).items()}
    X, b = minibatch(slab, ret, adv, perm, 0, B, blob0, D)
    p = params(blob0, D)
    z1 = layer1(p, X)
    fused_flips = int(((H1 > 0) != (z1.v > 0)).sum())
    t32 = torch_ppo(blob0.clone(), D, cfg, torch.float32, "relu")
    z32 = torch.cat([t32.actor[0](X.float()), t32.critic[0](X.float())], 1)
    torch_flips = int(((z32 > 0) != (z1.v > 0)).sum())
    near = int(undecided_units(z1).sum())
    # the fp64 gradient under the kernel's layer-1 masks: values fp64 (no bound: the bounds carried from X leave some loss
    # branches undecided), and the same evaluated from the kernel's H1 with its bound (layer-2 units the bound cannot
    # decide get the hull of both masks)
    masked64 = reference(p, X, b, cfg, "relu", h1_mask=H1 > 0)
    g_masked = add_entropy(grad_sums(p, X, masked64.d, masked64.h1, masked64.h2, masked64.dz2, masked64.dz1, split, per_row=False),
                           p, cfg.entropy_coef)
    r = reference(p, X, b, cfg, "relu", h1_kernel=H1.double())
    near2, loss_undecided = int(undecided_units(r.z2).sum()), int(r.undecided.sum())
    t64 = torch_ppo(blob0.clone(), D, cfg, torch.float64, "relu")
    t64.update(slab.obs_in, slab.actions, slab.values, slab.log_prob, slab.mean, ret, adv, perm, keep_grads=True)
    t32.update(slab.obs_in, slab.actions, slab.values, slab.log_prob, slab.mean, ret, adv, perm, keep_grads=True)
    g64, g32 = t64.trace[-1]["grads"]["actor.0.weight"], t32.trace[-1]["grads"]["actor.0.weight"]
    e = lambda g, ref: ((g.double() - ref).norm() / ref.norm()).item()
    print(f"\nobs689 seed={seed}: layer-1 units within the bound of 0: {near}; mask flips vs fp64: fused {fused_flips}, "
          f"torch fp32 {torch_flips}; layer-2 units undecided: {near2}; actor.0.weight err vs fp64: fused "
          f"{e(red_got['actor.0.weight'], g64):.3g}, torch fp32 {e(g32, g64):.3g}, fused vs fp64 under its masks "
          f"{e(red_got['actor.0.weight'], g_masked['actor.0.weight'].v):.3g}; loss branches undecided: {loss_undecided}")
    for k in g_masked:
        if k != "sums":
            assert e(red_got[k], g_masked[k].v) <= max(4 * e(t32.trace[-1]["grads"][k], t64.trace[-1]["grads"][k]), 1e-6), k
    if loss_undecided == 0:        # then the whole row is within the per-element bound too
        bound = add_entropy(grad_sums(p, X, r.d, r.h1, r.h2, r.dz2, r.dz1, split, per_row=False), p, cfg.entropy_coef)
        ratios = {}
        for k, t in bound.items():
            _check(f"under the kernel's masks {k}", red_got[k], t, ratios)
        _report(f"obs689 seed={seed}", ratios)


# ---- the margin batches on the device ---------------------------------------------------------------------------------

def test_margin_batch_on_the_device_keeps_every_branch():
    """The 689-wide margin batch of 16384 rows the one-mini-batch test uses: margins asserted, every branch > 100 samples."""
    _need_gpu()
    from wheeledlab_b200.learner import PPOConfig
    cfg = PPOConfig(num_learning_epochs=1, num_mini_batches=1)
    blob, slab, ret, adv, perm = margin_batch(689, 16384, 0, DEV, cfg=cfg)
    r = check_margins(blob, slab, ret, adv, perm, 689, 0, 16384, cfg, K)
    for name, c in branch_counts(r, cfg).items():
        assert c > 100, f"the margin batch misses the branch {name} ({c})"
    blob2, batches = blob.clone(), [synthetic(689, 2048, s, DEV)[1:] for s in (1, 2)]
    apply_margins(blob2, 689, batches, 0, 2048, cfg, K)
