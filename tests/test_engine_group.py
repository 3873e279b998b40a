"""Engine groups: one MC iteration on several engines from one call (tb200_group_*, EngineGroup, get_engine([...])).

CPU tests cover the Python plumbing with fakes.  GPU tests compare groups whose members share device 0 ([0], [0, 0],
[0, 0, 0], with peer access on and off) against one Engine(0) over the same packets: per-packet outputs, last-interaction
columns, counters, J_blue, Edotlu, the event log and the virtual-packet log bit for bit; J, nu_bar, vhist, the fused
spectra, the luminosity sums and the continuum estimators to rtol 1e-13, and bit-identical on every member."""
from types import SimpleNamespace

import numpy as np
import pytest

from golden_util import CASES, load_case, make_golden

EXACT = ("output_nus", "output_energies", "j_blue", "edotlu", "last_interaction_type", "last_event_id", "last_shell_id",
         "last_line_absorb_id", "last_line_emit_id", "last_radius", "last_before_nu", "last_before_mu", "last_before_energy",
         "last_after_nu", "last_after_mu", "last_after_energy", "event_counts")
CLOSE = ("j", "nu_bar", "vhist", "spectrum_emitted", "spectrum_reabsorbed", "luminosity_sums", "photo_ion_estimator",
         "stim_recomb_estimator", "bf_heating_estimator", "stim_recomb_cooling_estimator", "ff_heating_estimator")
SUMMED = ("j", "nu_bar", "vhist", "spectrum_emitted", "spectrum_reabsorbed", "luminosity_sums", "j_blue", "edotlu",
          "photo_ion_estimator", "stim_recomb_estimator", "bf_heating_estimator", "stim_recomb_cooling_estimator",
          "ff_heating_estimator", "photo_ion_estimator_statistics")
CONTINUUM_FIELDS = ("bf_threshold_list_nu", "photo_ion_nu_threshold_mins", "photo_ion_nu_threshold_maxs", "chi_bf", "x_sect",
                    "phot_nus", "ff_opacity_factor", "emissivities", "absorbing_markov_probabilities",
                    "photo_ion_block_references", "photo_ion_activation_idx", "k_packet_idx")


# ---------------------------------------------------------------------------------------------------------------------
# CPU: plumbing
# ---------------------------------------------------------------------------------------------------------------------
def test_get_engine_caches_one_group_per_device_list(monkeypatch):
    from tardis_b200 import montecarlo as mc

    made = []

    class FakeGroup:
        def __init__(self, devices):
            made.append(devices)

    class FakeEngine:
        def __init__(self, device):
            made.append(device)

    monkeypatch.setattr(mc, "_engines", {})
    monkeypatch.setattr(mc, "EngineGroup", FakeGroup)
    monkeypatch.setattr(mc, "Engine", FakeEngine)
    g = mc.get_engine([0, 0])
    assert isinstance(g, FakeGroup) and mc.get_engine((0, 0)) is g and mc.get_engine(np.array([0, 0])) is g
    assert mc.get_engine([0, 1]) is not g
    e = mc.get_engine(0)
    assert isinstance(e, FakeEngine) and mc.get_engine(np.int64(0)) is e and mc.get_engine() is e
    assert made == [(0, 0), (0, 1), 0]


def test_solvers_pass_the_device_list_through(monkeypatch):
    from tardis_b200 import montecarlo as mc
    from test_host_logic import FakeEngine, _fake_config, _setup

    model, geo, opa, pc = _setup()
    eng = FakeEngine()
    asked = []
    monkeypatch.setattr(mc, "get_engine", lambda device=0: asked.append(device) or eng)
    source = SimpleNamespace(base_seed=1, create_packets=lambda n, seed_offset=0: pc)
    solver = mc.MCTransportSolverB200.from_config(_fake_config(), source, device=[0, 1, 2, 3])
    assert solver.device == [0, 1, 2, 3]
    if isinstance(solver.radfield_prop_solver, mc.MCRadiationFieldPropertiesSolverB200):
        assert solver.radfield_prop_solver.device == [0, 1, 2, 3]
    sim_state = SimpleNamespace(geometry=SimpleNamespace(to_numba=lambda: geo, v_inner_boundary_idx=0, v_outer_boundary_idx=6),
                                time_explosion=model.time_explosion)
    opacity_host = SimpleNamespace(to_numba=lambda macro_atom_state, lit: opa)
    plasma = SimpleNamespace(continuum_interaction_species=SimpleNamespace(empty=True))
    state = solver.initialize_transport_state(sim_state, opacity_host, None, plasma, 50)
    solver.run(state, show_progress_bars=False)
    assert asked == [[0, 1, 2, 3]]


def test_group_shards_follow_parallel_shard_bounds():
    from tardis_b200 import parallel
    from tardis_b200.engine import EngineGroup

    for g in (1, 2, 3, 8):
        fake = SimpleNamespace(members=[None] * g)
        for n in (0, 1, g - 1, 1009, 10**8 + 7):
            assert EngineGroup.shard_bounds(fake, n) == [parallel.shard_bounds(n, r, g) for r in range(g)]


# ---------------------------------------------------------------------------------------------------------------------
# GPU: against one engine
# ---------------------------------------------------------------------------------------------------------------------
def _config(rk, sig):
    cfg = dict(enable_full_relativity=rk.get("enable_full_relativity", False),
               disable_line_scattering=rk.get("disable_line_scattering", False),
               number_of_vpackets=rk.get("number_of_vpackets", 0),
               vpacket_spawn_start_frequency=rk.get("spawn_start", 0.0), vpacket_spawn_end_frequency=rk.get("spawn_end", 1e200),
               survival_probability=rk.get("survival_probability", 0.0))
    if sig is not None:
        cfg["sigma_thomson"] = sig
    return cfg


def same(a, b):
    """Equal element for element (NaN, where an entry is unset, equals NaN); structured arrays field by field."""
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype.names:
        return a.shape == b.shape and all(same(a[f], b[f]) for f in a.dtype.names)
    return np.array_equal(a, b, equal_nan=a.dtype.kind == "f")


def _vlog_rows(res):
    m = min(res["vlog_count"], len(res["vlog_nus"]))
    cols = [res[k][:m] for k in ("vlog_packet_index", "vlog_nus", "vlog_energies", "vlog_initial_mus", "vlog_initial_rs")]
    order = np.lexsort(cols[::-1])
    return [c[order] for c in cols]


def assert_group_matches(res, ref):
    """`res` (group) against `ref` (one engine over the same packets).  The f64 sums are compared to rounding even for a
    one-member group: one engine's J / nu_bar / spectra come from atomic adds and vary in the last bits from run to run."""
    assert res["counters"] == ref["counters"]
    for k in EXACT:
        if k in ref:
            assert same(res[k], ref[k]), k
    for k in CLOSE:
        if k in ref:
            a, b = np.asarray(res[k]), np.asarray(ref[k])
            np.testing.assert_allclose(a, b, rtol=1e-13, atol=1e-13 * (np.abs(b).max() if b.size else 0.0), err_msg=k)
    if "photo_ion_estimator_statistics" in ref:
        assert np.array_equal(res["photo_ion_estimator_statistics"], ref["photo_ion_estimator_statistics"])
    if "events" in ref:
        assert len(res["events"]) == len(ref["events"])
        for a, b in zip(res["events"], ref["events"]):
            assert same(a, b)
    if "vlog_count" in ref:
        assert res["vlog_count"] == ref["vlog_count"]
        for a, b in zip(_vlog_rows(res), _vlog_rows(ref)):
            assert same(a, b)


def assert_members_agree(group):
    first = group.members[0].download(per_packet=False)
    for m in group.members[1:]:
        other = m.download(per_packet=False)
        for k in SUMMED:
            if k in first:
                assert same(other[k], first[k]), k


@pytest.fixture(scope="module")
def single():
    from tardis_b200.engine import Engine

    eng = Engine(0)
    yield eng
    eng.close()


@pytest.fixture(scope="module", params=[(1, 1), (2, 1), (2, 0), (3, 1), (3, 0)], ids=lambda p: f"G{p[0]}-peer{p[1]}")
def group(request):
    from tardis_b200.engine import EngineGroup

    g = EngineGroup([0] * request.param[0])
    g.set_option("peer_access", request.param[1])
    yield g
    g.close()


def _run(eng, model, packets, rk, sig):
    eng.set_model_from(model, **_config(rk, sig))
    vlog = 2_000_000 if rk.get("number_of_vpackets", 0) else 0
    return eng.run_packets(packets, track_last_interaction=True, n_tracked_packets=make_golden.N_TRACKED,
                           max_events_per_packet=4096, vlog_capacity=vlog)


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_group_matches_one_engine(group, single, name):
    model, packets, rk, sig, _ = load_case(name)
    ref = _run(single, model, packets, rk, sig)
    res = _run(group, model, packets, rk, sig)
    assert_group_matches(res, ref)
    assert_members_agree(group)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [0, 1, 2, 1009])
def test_group_edge_packet_counts(single, n):
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import EngineGroup

    model = syn.make_model(6, 800, "macroatom", mu_tau=-3.0, seed=31)
    packets = syn.make_packets(max(n, 1), model.r_inner[0], base_seed=5)
    arrays = [a[:n] for a in (packets.initial_radii, packets.initial_nus, packets.initial_mus, packets.initial_energies,
                              packets.packet_seeds)]
    single.set_model_from(model, number_of_vpackets=2)
    ref = single.run(*arrays, track_last_interaction=True, n_tracked_packets=5, max_events_per_packet=512, vlog_capacity=100000)
    g = EngineGroup([0, 0, 0])
    try:
        g.set_model_from(model, number_of_vpackets=2)
        res = g.run(*arrays, track_last_interaction=True, n_tracked_packets=5, max_events_per_packet=512, vlog_capacity=100000)
        assert_group_matches(res, ref)
        res = g.run(*arrays)  # and again, without tracking
        assert np.array_equal(res["j_blue"], ref["j_blue"]) and res["counters"] == ref["counters"]
    finally:
        g.close()


@pytest.mark.gpu
def test_vlog_capacity_overflow_matches_one_engine(single):
    """Fewer log rows than virtual packets: the total count comes back, rows beyond the capacity are dropped."""
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import EngineGroup

    model = syn.make_model(6, 800, "macroatom", mu_tau=-3.0, seed=31)
    packets = syn.make_packets(3000, model.r_inner[0], base_seed=5)
    single.set_model_from(model, number_of_vpackets=3)
    ref = single.run_packets(packets, vlog_capacity=500)
    g = EngineGroup([0, 0])
    try:
        g.set_model_from(model, number_of_vpackets=3)
        res = g.run_packets(packets, vlog_capacity=500)
        assert res["vlog_count"] == ref["vlog_count"] > 500
        assert np.array_equal(res["j_blue"], ref["j_blue"])
    finally:
        g.close()


@pytest.mark.gpu
def test_common_scale_keeps_shards_of_different_energies_exact(single):
    """Members holding packets of very different energies still sum the fixed-point accumulators (one scale for all)."""
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import EngineGroup

    model = syn.make_model(8, 2000, "macroatom", mu_tau=-3.0, seed=7)
    packets = syn.make_packets(20000, model.r_inner[0], base_seed=9)
    energies = packets.initial_energies.copy()
    energies[:10000] *= 1.0 / 64
    energies[10000:] *= 64.0
    arrays = (packets.initial_radii, packets.initial_nus, packets.initial_mus, energies, packets.packet_seeds)
    single.set_model_from(model)
    ref = single.run(*arrays)
    g = EngineGroup([0, 0])
    try:
        g.set_model_from(model)
        assert_group_matches(g.run(*arrays), ref)
        g.upload_packets(*arrays)
        g.transport()
        assert g.allreduce() is True
        res = g.download()
        assert np.array_equal(res["j_blue"], ref["j_blue"]) and np.array_equal(res["edotlu"], ref["edotlu"])
        assert np.array_equal(res["output_nus"], ref["output_nus"]) and res["counters"] == ref["counters"]
        assert_members_agree(g)
    finally:
        g.close()


@pytest.mark.gpu
def test_scan_algorithm_takes_the_f64_collective(single):
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import EngineGroup

    model = syn.make_model(8, 2000, "downbranch", mu_tau=-3.0, seed=8)
    packets = syn.make_packets(20000, model.r_inner[0], base_seed=10)
    single.set_option("algorithm", 0)
    try:
        single.set_model_from(model)
        ref = single.run_packets(packets)
    finally:
        single.set_option("algorithm", 1)
    g = EngineGroup([0, 0])
    try:
        g.set_option("algorithm", 0)
        g.set_model_from(model)
        res = g.run_packets(packets)
        for k in ("output_nus", "output_energies"):
            assert np.array_equal(res[k], ref[k]), k
        assert res["counters"] == ref["counters"]
        for k in (k for k in SUMMED if k in ref):
            np.testing.assert_allclose(res[k], ref[k], rtol=1e-13, atol=1e-13 * np.abs(ref[k]).max(), err_msg=k)
        g.upload_packets(packets.initial_radii, packets.initial_nus, packets.initial_mus, packets.initial_energies,
                         packets.packet_seeds)
        g.transport()
        assert g.allreduce() is False
        assert_members_agree(g)
    finally:
        g.close()


@pytest.mark.gpu
def test_group_errors_name_the_member_and_the_group_runs_again(single):
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import EngineGroup, MacroAtomError

    model = syn.make_model(4, 300, "macroatom", mu_tau=-2.0, seed=14)
    bad = syn.make_model(4, 300, "macroatom", mu_tau=-2.0, seed=14)
    bad.macro.transition_probabilities[:] = 0.0  # every activated block runs out -> MacroAtomError
    packets = syn.make_packets(500, model.r_inner[0])
    g = EngineGroup([0, 0])
    try:
        g.set_model_from(bad)
        with pytest.raises(MacroAtomError, match=r"group member 0 \(device 0, global packets \[0, 250\)\)"):
            g.run_packets(packets)
        g.set_model_from(model)
        single.set_model_from(model)
        assert_group_matches(g.run_packets(packets), single.run_packets(packets))
    finally:
        g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("beta", [None, 0.01])
def test_group_device_packet_source(single, beta):
    """Member g generates exactly its range of what one engine generates; run_resident then equals run."""
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import EngineGroup

    model = syn.make_model(8, 2000, "macroatom", mu_tau=-3.0, seed=12)
    n, seed, radius, temp = 100_003, 77, float(model.r_inner[0]), 9500.0
    single.create_packets(n, seed, radius, temp, beta=beta)
    ref_packets = single.download_packets()
    g = EngineGroup([0, 0, 0])
    try:
        g.create_packets(n, seed, radius, temp, beta=beta)
        got = g.download_packets()
        for k in ref_packets:
            assert np.array_equal(got[k], ref_packets[k]), k
        g.set_model_from(model)
        res = g.run_resident()
        single.set_model_from(model)
        ref = single.run(*(ref_packets[k] for k in ("initial_radii", "initial_nus", "initial_mus", "initial_energies",
                                                    "packet_seeds")))
        assert_group_matches(res, ref)
    finally:
        g.close()


@pytest.mark.gpu
def test_solver_with_a_device_list_matches_device_0(monkeypatch):
    """MCTransportSolverB200.from_config(..., device=[0, 0]) through the reference-shaped objects."""
    from tardis_b200 import montecarlo as mc
    from tardis_b200 import synthetic as syn
    from test_host_logic import _fake_config

    monkeypatch.setattr(mc, "_engines", {})
    full = syn.make_model(10, 2500, "macroatom", mu_tau=-3.5, seed=41)
    sl = slice(1, 9)
    packets = syn.make_packets(1500, full.r_inner[sl][0], base_seed=3)
    geo = mc.HomologousGeometry(full.r_inner[sl], full.r_outer[sl], full.v_inner[sl], full.v_outer[sl], full.time_explosion)
    cfg = _fake_config(**{"spectrum.virtual.virtual_packet_logging": True, "spectrum.start": full.spectrum_frequency_grid[-1],
                          "spectrum.stop": full.spectrum_frequency_grid[0], "spectrum.num": len(full.spectrum_frequency_grid) - 1})
    sim_state = SimpleNamespace(geometry=SimpleNamespace(to_numba=lambda: geo, v_inner_boundary_idx=1, v_outer_boundary_idx=9),
                                time_explosion=full.time_explosion)
    opacity_host = SimpleNamespace(to_numba=lambda macro_atom_state, lit: mc.OpacityState.from_model(full))
    plasma = SimpleNamespace(continuum_interaction_species=SimpleNamespace(empty=True))

    def state_for(device):
        pc = mc.PacketCollection(packets.initial_radii, packets.initial_nus, packets.initial_mus, packets.initial_energies,
                                 packets.packet_seeds, packets.radiation_field_luminosity)
        source = SimpleNamespace(base_seed=1, create_packets=lambda n, seed_offset=0: pc)
        solver = mc.MCTransportSolverB200.from_config(cfg, source, device=device)
        state = solver.initialize_transport_state(sim_state, opacity_host, None, plasma, len(pc.initial_nus), no_of_virtual_packets=3)
        return solver.run(state, show_progress_bars=False), state, pc

    vh0, s0, pc0 = state_for(0)
    vh1, s1, pc1 = state_for([0, 0])
    assert isinstance(mc.get_engine([0, 0]), mc.EngineGroup)
    assert np.array_equal(pc1.output_nus, pc0.output_nus) and np.array_equal(pc1.output_energies, pc0.output_energies)
    assert np.array_equal(s1.j_blue_estimator, s0.j_blue_estimator)
    np.testing.assert_allclose(s1.j_estimator, s0.j_estimator, rtol=1e-13)
    np.testing.assert_allclose(vh1, vh0, rtol=1e-13, atol=1e-13 * np.abs(vh0).max())
    assert s1.tracker_last_interaction_df.equals(s0.tracker_last_interaction_df)
    v0, v1 = (np.asarray(getattr(s.virt_packet_nus, "value", s.virt_packet_nus)) for s in (s0, s1))
    assert np.array_equal(np.sort(v1), np.sort(v0))
    for eng in list(mc._engines.values()):
        eng.close()


@pytest.mark.gpu
def test_two_device_group_matches_one_engine(single):
    """[0, 1] on a box with two GPUs, peer access on and off."""
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from tardis_b200.engine import EngineGroup

    model, packets, rk, sig, _ = load_case("macroatom_vpackets")
    ref = _run(single, model, packets, rk, sig)
    g = EngineGroup([0, 1])
    try:
        for peer in (1, 0):
            g.set_option("peer_access", peer)
            assert_group_matches(_run(g, model, packets, rk, sig), ref)
            assert_members_agree(g)
    finally:
        g.close()


@pytest.mark.gpu
def test_collective_runs_once_per_transport():
    """A second collective without a transport in between would add the sums again: it is refused."""
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import EngineError, EngineGroup

    model = syn.make_model(4, 300, "scatter", seed=3)
    packets = syn.make_packets(1000, model.r_inner[0])
    g = EngineGroup([0, 0])
    try:
        g.set_model_from(model)
        g.upload_packets(packets.initial_radii, packets.initial_nus, packets.initial_mus, packets.initial_energies,
                         packets.packet_seeds)
        g.transport()
        first = (g.allreduce(), g.download(per_packet=False)["j_blue"])
        with pytest.raises(EngineError, match="no transport since the last collective"):
            g.allreduce()
        assert same(g.download(per_packet=False)["j_blue"], first[1])
        g.run_packets(packets)  # a run is a transport: the group goes on
    finally:
        g.close()


# ---- the steps around the transport: device-built tables, radiation field, source function, formal integral ----------
def _macro_setup():
    from tardis_b200 import synthetic as syn

    S, L, n_levels = 8, 4000, 300
    model = syn.make_model(S, L, "macroatom", mu_tau=-4.0, seed=71)
    atomic = syn.make_atomic_data(model.line_list_nu, n_levels, "macroatom", seed=72, nlte_fraction=0.0)
    plasma = syn.make_plasma_state(atomic, S, model.time_explosion, seed=73, zero_fraction=0.0, inversion_fraction=0.0, noise=0.0)
    plasma.level_number_density *= 1e-9
    return model, atomic, plasma, n_levels


def _device_tables(eng, model, atomic, plasma):
    eng.set_option("keep_opacity_tables", 1)
    eng.set_model(r_inner=model.r_inner, r_outer=model.r_outer, time_explosion=model.time_explosion,
                  electron_density=model.electron_density, line_list_nu=model.line_list_nu, tau_sobolev=None,
                  line_interaction_type="macroatom", transition_probabilities=None,
                  line2macro_level_upper=atomic.line2macro_level_upper, macro_block_edge_index=atomic.macro_block_edge_index,
                  transition_type=atomic.transition_type, destination_level_id=atomic.destination_level_id,
                  transition_line_id=atomic.transition_line_idx, spectrum_frequency_grid=model.spectrum_frequency_grid)
    eng.set_atomic_data(lines_lower_level_index=atomic.lower_level, lines_upper_level_index=atomic.upper_level, g=atomic.g,
                        metastability=atomic.metastable, wavelength_cm=atomic.wavelength_cm, f_lu=atomic.f_lu, f_ul=atomic.f_ul,
                        energy_lower=atomic.energy[atomic.lower_level], energy_upper=atomic.energy[atomic.upper_level],
                        nlte_line=atomic.nlte_line)
    eng.build_opacity(plasma.level_number_density, plasma.time_explosion, plasma.j_blues)


@pytest.mark.gpu
@pytest.mark.parametrize("members", [2, 3])
def test_group_tables_radiation_field_source_function_and_formal_integral(single, members):
    """One iteration's surroundings on a group against Engine(0): device-built opacity tables, transport, radiation field,
    source function and the frequency-sharded formal integral (with fewer frequencies than members too)."""
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import Engine, EngineGroup

    model, atomic, plasma, n_levels = _macro_setup()
    volume = 4.0 / 3.0 * np.pi * (model.r_outer**3 - model.r_inner**3)
    t_exp, t_sim, t_inner, points = float(model.time_explosion), 2.0e5, 1.1e4, 120
    packets = syn.make_packets(50000, model.r_inner[0], base_seed=13)
    z_max = model.r_outer[-1] / t_exp / 2.99792458e10
    nu = model.line_list_nu
    freq = np.linspace(nu[-1] / (1 - z_max) * 1.001, nu[0] * 1.02, 200)
    rf = dict(time_explosion=t_exp, time_of_simulation=t_sim, volume=volume)
    sf = dict(time_explosion=t_exp, time_of_simulation=t_sim, volume=volume, wavelength_cm=atomic.wavelength_cm,
              lines_lower_level_idx=atomic.lower_level, lines_upper_level_idx=atomic.upper_level, n_levels=n_levels)

    def iteration(eng):
        _device_tables(eng, model, atomic, plasma)
        out = {"opacity": eng.download_opacity(transition_probabilities=True)}
        out["run"] = eng.run_packets(packets)
        out["radfield"] = eng.solve_radiation_field(**rf)
        out["source"] = eng.solve_source_function(**sf)
        out["integral"] = eng.formal_integral(inner_temperature=t_inner, frequencies=freq, points=points, interpolate_shells=0,
                                              want_intensities=True)
        out["few"] = eng.formal_integral(inner_temperature=t_inner, frequencies=freq[:members - 1], points=points,
                                         interpolate_shells=0, want_intensities=True)
        return out

    ref = iteration(single)
    g = EngineGroup([0] * members)
    try:
        got = iteration(g)
        for m in g.members:  # the device-built tables: bit-identical on every member and to one engine
            tables = m.download_opacity(transition_probabilities=True)
            for k, v in ref["opacity"].items():
                assert same(tables[k], v), k
        assert same(got["run"]["j_blue"], ref["run"]["j_blue"]) and same(got["run"]["edotlu"], ref["run"]["edotlu"])
        # radiation field: J / nu_bar differ from one engine's by rounding; every member computes the same bits
        for a, b in zip(got["radfield"], ref["radfield"]):
            np.testing.assert_allclose(a, b, rtol=1e-12)
        per_member = [Engine.solve_radiation_field(m, **rf) for m in g.members]
        for res in per_member[1:]:
            for a, b in zip(res, per_member[0]):
                assert same(a, b)
        # source function: reads tau / the kept probabilities / the exact line estimators -> bit-identical
        for k in ("att_S_ul", "Jred_lu", "Jblue_lu", "e_dot_u"):
            assert same(got["source"][k], ref["source"][k]), k
        per_member = [Engine.solve_source_function(m, **sf) for m in g.members]
        for res in per_member[1:]:
            for k in ("att_S_ul", "Jred_lu", "Jblue_lu", "e_dot_u"):
                assert same(res[k], per_member[0][k]), k
        for key in ("integral", "few"):
            assert same(got[key]["luminosity_densities"], ref[key]["luminosity_densities"]), key
            assert same(got[key]["intensities_nu_p"], ref[key]["intensities_nu_p"]), key
        assert got["integral"]["integral_ms"] > 0.0
    finally:
        g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(make_golden.FORMAL_INTEGRAL_CASES))
def test_group_formal_integral_matches_one_engine_on_the_goldens(single, name):
    """Host-given tables of the formal-integral goldens: luminosity densities and I(nu, p) equal one engine's bit for bit."""
    from tardis_b200.engine import EngineGroup

    i = make_golden.formal_integral_inputs(name)
    s = make_golden.source_function_inputs(i["source_function_case"])
    a, m = s["atomic"], i["model"]

    def integral(eng, frequencies):
        eng.set_option("keep_opacity_tables", 1)
        eng.set_model(r_inner=m.r_inner, r_outer=m.r_outer, time_explosion=m.time_explosion, electron_density=m.electron_density,
                      line_list_nu=m.line_list_nu, tau_sobolev=i["tau_sobolev"], line_interaction_type=s["mode"],
                      transition_probabilities=s["transition_probabilities"], line2macro_level_upper=a.line2macro_level_upper,
                      macro_block_edge_index=a.macro_block_edge_index, transition_type=a.transition_type,
                      destination_level_id=a.destination_level_id, transition_line_id=a.transition_line_idx,
                      spectrum_frequency_grid=m.spectrum_frequency_grid)
        return eng.formal_integral(inner_temperature=i["inner_temperature"], frequencies=frequencies, points=i["points"],
                                   interpolate_shells=i["interpolate_shells"], tables=(i["att_S_ul"], i["Jred_lu"], i["Jblue_lu"]),
                                   want_intensities=True)

    g = EngineGroup([0, 0, 0])
    try:
        for frequencies in (i["frequencies"], i["frequencies"][:2]):
            ref, got = integral(single, frequencies), integral(g, frequencies)
            assert same(got["luminosity_densities"], ref["luminosity_densities"])
            assert same(got["intensities_nu_p"], ref["intensities_nu_p"])
    finally:
        g.close()


@pytest.mark.gpu
def test_iip_solver_and_radiation_field_solver_with_a_device_list(monkeypatch):
    """MCTransportSolverB200IIP.from_config(..., device=[0, 0]) and MCRadiationFieldPropertiesSolverB200(device=[0, 0])
    against device=0."""
    from tardis_b200 import montecarlo as mc
    from test_host_logic import _fake_config

    monkeypatch.setattr(mc, "_engines", {})
    model, packets, _, _ = make_golden.build_inputs("iip_basic")
    geo = mc.HomologousGeometry(model.r_inner, model.r_outer, model.v_inner, model.v_outer, model.time_explosion)
    base = vars(mc.OpacityState.from_model(model))
    opa = SimpleNamespace(**base, **{k: getattr(model.continuum, k) for k in CONTINUUM_FIELDS})
    sim_state = SimpleNamespace(geometry=SimpleNamespace(to_numba=lambda: geo, v_inner_boundary_idx=0,
                                                         v_outer_boundary_idx=len(model.r_inner)),
                                time_explosion=model.time_explosion)
    plasma = SimpleNamespace(continuum_interaction_species=SimpleNamespace(empty=True))
    volume = 4.0 / 3.0 * np.pi * (model.r_outer**3 - model.r_inner**3)

    def state_for(device):
        pc = mc.PacketCollection(packets.initial_radii, packets.initial_nus, packets.initial_mus, packets.initial_energies,
                                 packets.packet_seeds, packets.radiation_field_luminosity)
        source = SimpleNamespace(base_seed=1, create_packets=lambda n, seed_offset=0: pc)
        solver = mc.MCTransportSolverB200IIP.from_config(_fake_config(), source, device=device)
        state = solver.initialize_transport_state(sim_state, SimpleNamespace(to_numba=lambda mas, lit: opa), None, plasma,
                                                  len(pc.initial_nus))
        solver.run(state, show_progress_bars=False)
        radfield = mc.MCRadiationFieldPropertiesSolverB200(1e-10, device=device).solve(
            state.estimators_bulk, state.estimators_line, model.time_explosion, pc.time_of_simulation, volume, model.line_list_nu)
        return state, pc, radfield

    s0, pc0, rf0 = state_for(0)
    s1, pc1, rf1 = state_for([0, 0])
    assert isinstance(mc.get_engine([0, 0]), mc.EngineGroup)
    assert same(pc1.output_nus, pc0.output_nus) and same(pc1.output_energies, pc0.output_energies)
    assert same(s1.j_blue_estimator, s0.j_blue_estimator)
    assert same(s1.estimators_line.energy_deposition_line_rate, s0.estimators_line.energy_deposition_line_rate)
    np.testing.assert_allclose(s1.j_estimator, s0.j_estimator, rtol=1e-13)
    for k in ("photo_ion_estimator", "stim_recomb_estimator", "bf_heating_estimator", "stim_recomb_cooling_estimator",
              "ff_heating_estimator"):
        a, b = (np.asarray(getattr(s.estimators_continuum, k)) for s in (s1, s0))
        np.testing.assert_allclose(a, b, rtol=1e-13, atol=1e-13 * np.abs(b).max(), err_msg=k)
    assert s1.tracker_last_interaction_df.equals(s0.tracker_last_interaction_df)
    t0, t1 = (np.asarray(getattr(r.dilute_blackbody_radiationfield_state.temperature, "value",
                                 r.dilute_blackbody_radiationfield_state.temperature)) for r in (rf0, rf1))
    np.testing.assert_allclose(t1, t0, rtol=1e-12)
    np.testing.assert_allclose(rf1.dilute_blackbody_radiationfield_state.dilution_factor,
                               rf0.dilute_blackbody_radiationfield_state.dilution_factor, rtol=1e-12)
    np.testing.assert_allclose(rf1.j_blues, rf0.j_blues, rtol=1e-12)
    for eng in list(mc._engines.values()):
        eng.close()
