"""Reset-mode domain randomisation (DESIGN 6n) without a GPU: the compat lowering of the reference's own cfg objects with their
DR events' mode edited, and the oracle's twin of wl_reset_dr_kernel -- which envs it redraws, what it leaves at the start-up
values, the distributions it draws from, and its invariance under sharding."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(Path(__file__).resolve().parent))

MATERIAL, GAINS, BASE, WHEEL = 1, 2, 4, 8
G_POS, G_PMASS, G_PMU_D, G_PMU_C, G_PKD, G_PIW = 0, 9, 10, 11, 12, 15
DR_GROUPS = [G_PMASS, G_PMU_D, G_PMU_C, G_PKD, G_PIW]


@pytest.fixture(scope="module")
def ref_registry():
    if str(ROOT / "shims") not in sys.path:
        sys.path.insert(0, str(ROOT / "shims"))
    import recorded_cfgs
    return recorded_cfgs.load()


def _cfg(reg, gid, entry="env_cfg_entry_point", n=8, **modes):
    c = reg[gid]["cfgs"][entry]()
    c.scene.num_envs = n
    for name, mode in modes.items():
        setattr(getattr(c.events, name), "mode", mode)
    return c


def test_registered_cfgs_lower_to_start_up_dr_only(ref_registry):
    from wheeledlab_b200.compat import spec_from_reference_cfg
    for gid, rec in ref_registry.items():
        for entry in rec["cfgs"]:
            assert spec_from_reference_cfg(_cfg(ref_registry, gid, entry)).reset_events == [], (gid, entry)


@pytest.mark.parametrize("gid,entry,modes,want", [
    ("Isaac-MushrDriftRL-v0", "env_cfg_entry_point", {"change_wheel_friction": "reset"}, ["material"]),
    ("Isaac-MushrDriftRL-v0", "env_cfg_entry_point", {"randomize_gains": "reset"}, ["actuator_gains"]),
    ("Isaac-MushrDriftRL-v0", "env_cfg_entry_point", {"add_base_mass": "reset"}, ["base_mass"]),
    ("Isaac-MushrDriftRL-v0", "env_cfg_entry_point", {"change_wheel_friction": "reset", "randomize_gains": "reset", "add_base_mass": "reset"},
     ["material", "actuator_gains", "base_mass"]),
    ("Isaac-F1TenthDriftRL-v0", "env_cfg_entry_point", {"randomize_gains": "reset", "add_base_mass": "reset"}, ["actuator_gains", "base_mass"]),
    ("Isaac-MushrElevationRL-v0", "env_cfg_entry_point", {"change_wheel_friction": "reset", "add_base_mass": "reset"}, ["material", "base_mass"]),
    ("Isaac-MushrVisualRL-v0", "play_env_cfg_entry_point", {"add_base_mass": "reset"}, ["base_mass"]),
    ("Isaac-MushrVisualRL-v0", "play_env_cfg_entry_point", {"add_wheel_mass": "reset"}, ["wheel_mass"]),
])
def test_reset_mode_lowers_to_its_event(ref_registry, gid, entry, modes, want):
    from wheeledlab_b200.compat import spec_from_reference_cfg
    start = spec_from_reference_cfg(_cfg(ref_registry, gid, entry))
    spec = spec_from_reference_cfg(_cfg(ref_registry, gid, entry, **modes))
    assert spec.reset_events == want
    assert bytes(spec.cfg) == bytes(start.cfg), "the mode changes nothing in the config"


def test_other_modes_and_a_minimum_step_count_are_refused_by_name(ref_registry):
    from wheeledlab_b200.compat import spec_from_reference_cfg
    with pytest.raises(NotImplementedError, match="randomize_gains.*'interval'"):
        spec_from_reference_cfg(_cfg(ref_registry, "Isaac-MushrDriftRL-v0", randomize_gains="interval"))
    with pytest.raises(NotImplementedError, match="add_wheel_mass.*'prestartup'"):
        spec_from_reference_cfg(_cfg(ref_registry, "Isaac-MushrVisualRL-v0", "play_env_cfg_entry_point", add_wheel_mass="prestartup"))
    c = _cfg(ref_registry, "Isaac-MushrDriftRL-v0", add_base_mass="reset")
    c.events.add_base_mass.min_step_count_between_reset = 5
    with pytest.raises(NotImplementedError, match="add_base_mass: min_step_count_between_reset 5"):
        spec_from_reference_cfg(c)


# ---- the oracle twin ----------------------------------------------------------------------------------------------------------

def _oracle(task, n, mask, seed=3, offset=0):
    import reset_dr_oracle
    import wheeledlab_b200 as wl
    spec = wl.make_task(task, num_envs=n, seed=seed, env_id_offset=offset)
    o = reset_dr_oracle.Oracle(spec.cfg, heightfield=spec.heightfield, mask=mask)
    o.startup()
    o.reset(None, 0)
    return o


def test_oracle_refusals_leave_the_mask_as_it_was():
    import reset_dr_oracle
    import wheeledlab_b200 as wl
    for task, bad in (("drift", 16), ("drift", WHEEL), ("elevation", GAINS), ("visual", MATERIAL), ("visual_random", GAINS)):
        spec = wl.make_task(task, num_envs=4, seed=1)
        o = reset_dr_oracle.Oracle(spec.cfg, heightfield=spec.heightfield)
        assert o.set_reset_events(bad) != 0, (task, bad)
    ref, o = _oracle("drift", 64, MATERIAL), _oracle("drift", 64, MATERIAL)
    assert o.set_reset_events(MATERIAL | 32) != 0 and o.set_reset_events(WHEEL) != 0
    for t in range(1, 260):
        a = ref.synth_actions(t)
        ref.step(a, t)
        o.step(a, t)
    assert np.array_equal(ref.export_state().view(np.uint32), o.export_state().view(np.uint32))


def test_only_envs_that_reset_are_redrawn_and_start_up_components_keep_their_bits():
    """Visual random cfg, base mass in reset mode, wheel masses in start-up mode (as its own cfg splits them)."""
    n = 256
    o, start = _oracle("visual_random", n, BASE), _oracle("visual_random", n, 0)
    s0 = start.export_state()
    prev = o.export_state()
    redrawn = 0
    for t in range(1, 400):
        o.step(o.synth_actions(t), t)
        s = o.export_state()
        reset = s[G_POS, :, 3].view(np.int32) == 0
        keep = ~reset
        for g in DR_GROUPS:
            assert np.array_equal(s[g][keep].view(np.uint32), prev[g][keep].view(np.uint32)), (t, g)
        for g in (G_PMU_D, G_PMU_C, G_PKD, G_PIW):
            assert np.array_equal(s[g].view(np.uint32), s0[g].view(np.uint32)), (t, g)
        assert (s[G_PMASS][reset, 0] != prev[G_PMASS][reset, 0]).all()
        redrawn += int(reset.sum())
        prev = s
    assert redrawn > n


def test_explicit_reset_redraws_exactly_its_ids():
    o = _oracle("drift", 128, MATERIAL | GAINS | BASE)
    before = o.export_state()
    ids = np.array([3, 77, 100], np.int64)
    o.reset(ids, 42)
    after = o.export_state()
    other = np.setdiff1d(np.arange(128), ids)
    for g in (G_PMASS, G_PKD):
        assert np.array_equal(after[g][other].view(np.uint32), before[g][other].view(np.uint32))
        assert (after[g][ids, 0] != before[g][ids, 0]).all()


def test_redraw_distributions():
    """10^5 and more redraws of Drift's events: bucket frequencies (chi-square), damping and added mass (KS against the
    uniform range), and consecutive draws of one env differ."""
    from scipy import stats
    import wheeledlab_b200 as wl
    n, rounds = 4096, 25
    spec = wl.make_task("drift", num_envs=n, seed=11)
    c = spec.cfg
    o = _oracle("drift", n, MATERIAL | GAINS | BASE, seed=11)
    D = np.array(c.dr_bucket_D[:c.dr_num_buckets], np.float32)
    Cb = np.array(c.dr_bucket_C[:c.dr_num_buckets], np.float32)
    key = {(d.tobytes(), cc.tobytes()): k for k, (d, cc) in enumerate(zip(D, Cb))}
    assert len(key) == c.dr_num_buckets, "buckets are told apart by their (D, C) pair"
    counts = np.zeros(c.dr_num_buckets)
    kd, dm, masses = [], [], []
    for r in range(rounds):
        o.reset(None, 1000 + r)
        s = o.export_state()
        for d, cc in zip(s[G_PMU_D].reshape(-1), s[G_PMU_C].reshape(-1)):
            counts[key[(np.float32(d).tobytes(), np.float32(cc).tobytes())]] += 1
        kd.append(s[G_PKD][:, :2].reshape(-1))                           # the 2WD Drift randomises the rear wheels
        assert np.array_equal(s[G_PKD][:, 2:].view(np.uint32), np.broadcast_to(np.array(c.dc_damping[2:4], np.float32), (n, 2)).view(np.uint32))
        dm.append(s[G_PMASS][:, 0].astype(np.float64) - np.float32(c.mass_nominal))
        masses.append(s[G_PMASS][:, 0].copy())
    assert counts.sum() >= 4e5
    assert stats.chisquare(counts).pvalue > 1e-3
    kd, dm = np.concatenate(kd), np.concatenate(dm)
    assert kd.size >= 1e5 and dm.size >= 1e5
    assert stats.kstest(kd, stats.uniform(c.dr_kd_range[0], c.dr_kd_range[1] - c.dr_kd_range[0]).cdf).pvalue > 1e-3
    assert stats.kstest(dm, stats.uniform(c.dr_mass_add[0], c.dr_mass_add[1] - c.dr_mass_add[0]).cdf).pvalue > 1e-3
    m = np.stack(masses)
    assert (m[1:] != m[:-1]).all(), "consecutive draws of one env differ"


def test_two_shards_equal_one_handle():
    n = 192
    whole = _oracle("hound_4wd", 2 * n, MATERIAL | GAINS | BASE)
    shards = [_oracle("hound_4wd", n, MATERIAL | GAINS | BASE, offset=k * n) for k in range(2)]
    for t in range(1, 300):
        a = whole.synth_actions(t)
        whole.step(a, t)
        for k, s in enumerate(shards):
            s.step(a[k * n:(k + 1) * n], t)
    got = np.concatenate([s.export_state() for s in shards], axis=1)
    assert np.array_equal(got.view(np.uint32), whole.export_state().view(np.uint32))
