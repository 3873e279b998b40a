"""GPU parity tests: the CUDA engine (through the C-ABI) against (a) golden vectors from the
reference Numba path and (b) the CPU oracle on seeded synthetic inputs.  Integer work
(trajectories, event counts, work counters, last-interaction ids) must be identical; floats agree
to the tolerance in golden_util (the reference's own regression tolerance is 1e-12...1e-13)."""
import numpy as np
import pytest

from golden_util import CASES, assert_close, compare_to_golden, load_case, make_golden, oracle_kwargs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", params=["scan", "jump", "jump_lane"])
def engine(request):
    """All transport kernels must produce the reference's results: `scan` streams the line list, `jump` searches
    the tau prefix table and range-updates the line estimators (DESIGN.md §3) with a packet pool per warp (classic
    mode), `jump_lane` is the same algorithm with one packet per lane (what the continuum mode runs)."""
    from tardis_b200.engine import Engine

    eng = Engine(0)
    eng.set_option("algorithm", {"scan": 0, "jump": 1, "jump_lane": 1}[request.param])
    eng.set_option("pooled", 0 if request.param == "jump_lane" else 1)
    yield eng
    eng.close()


def same_counters(engine_counters, oracle_counters):
    """The engine reports the oracle's work counters exactly (plus its own n_search_probes)."""
    return all(engine_counters[k] == v for k, v in oracle_counters.items())


def engine_config(rk, sig):
    cfg = dict(
        enable_full_relativity=rk.get("enable_full_relativity", False),
        disable_line_scattering=rk.get("disable_line_scattering", False),
        number_of_vpackets=rk.get("number_of_vpackets", 0),
        vpacket_spawn_start_frequency=rk.get("spawn_start", 0.0),
        vpacket_spawn_end_frequency=rk.get("spawn_end", 1e200),
        survival_probability=rk.get("survival_probability", 0.0),
    )
    if sig is not None:
        cfg["sigma_thomson"] = sig
    return cfg


@pytest.mark.parametrize("name", CASES)
def test_engine_matches_reference_golden(engine, name):
    model, packets, rk, sig, g = load_case(name)
    engine.set_model_from(model, **engine_config(rk, sig))
    res = engine.run_packets(packets, track_last_interaction=True, n_tracked_packets=make_golden.N_TRACKED,
                             max_events_per_packet=4096)
    compare_to_golden(res, g, make_golden.N_TRACKED)


@pytest.mark.parametrize("name", CASES)
def test_engine_matches_oracle_counters(engine, oracle, name):
    """Work counters are functions of the seeds only: the engine must report the oracle's numbers."""
    model, packets, rk, sig, g = load_case(name)
    ref = oracle.run_oracle(model, packets, **oracle_kwargs(rk, sig))
    engine.set_model_from(model, **engine_config(rk, sig))
    res = engine.run_packets(packets)
    assert same_counters(res["counters"], ref["counters"])


@pytest.mark.parametrize("mode,n_lines,mu_tau", [("scatter", 20000, -6.0), ("macroatom", 8000, -4.5), ("downbranch", 8000, -4.5)])
def test_engine_vs_oracle_larger(engine, oracle, mode, n_lines, mu_tau):
    from tardis_b200 import synthetic as syn

    model = syn.make_model(20, n_lines, mode, mu_tau=mu_tau, seed=777)
    packets = syn.make_packets(20000, model.r_inner[0], base_seed=99)
    ref = oracle.run_oracle(model, packets, nthreads=8, n_tracked_packets=500, max_events_per_packet=4096)
    engine.set_model_from(model)
    res = engine.run_packets(packets, track_last_interaction=True, n_tracked_packets=500, max_events_per_packet=4096)
    assert same_counters(res["counters"], ref["counters"])
    assert_close(res["output_nus"], ref["output_nus"], 1e-11, "output_nus")
    assert_close(res["output_energies"], ref["output_energies"], 1e-11, "output_energies")
    for k in ("j", "nu_bar", "j_blue", "edotlu"):
        assert_close(res[k], ref[k], 1e-10, k)
    for k in ("last_interaction_type", "last_event_id", "last_shell_id", "last_line_absorb_id", "last_line_emit_id"):
        assert np.array_equal(res[k], ref[k]), k
    assert np.array_equal(res["event_counts"], ref["event_counts"])
    a, b = np.concatenate(res["events"]), np.concatenate(ref["events"])
    for k in ("packet_id", "interaction_type", "status", "before_shell_id", "after_shell_id", "line_absorb_id", "line_emit_id"):
        assert np.array_equal(a[k], b[k]), k


def test_engine_rng_long_stream(engine, oracle):
    """A very optically thick single shell forces hundreds of draws per packet: exercises all three
    tiers of the lazy MT19937 (cursor-only, ring read-back, in-place recurrence)."""
    from tardis_b200 import synthetic as syn

    model = syn.make_model(3, 2000, "scatter", mu_tau=-1.0, seed=5)
    model.electron_density[:] *= 300.0
    packets = syn.make_packets(2000, model.r_inner[0], base_seed=7)
    ref = oracle.run_oracle(model, packets)
    engine.set_model_from(model)
    res = engine.run_packets(packets)
    assert ref["counters"]["n_rng_draws"] / len(packets) > 150
    draws = ref["counters"]["n_rng_draws"]
    assert same_counters(res["counters"], ref["counters"]), (res["counters"], ref["counters"], draws)
    assert_close(res["output_nus"], ref["output_nus"], 1e-10, "output_nus")
    assert_close(res["output_energies"], ref["output_energies"], 1e-10, "output_energies")


def test_empty_and_single_packet(engine, oracle):
    from tardis_b200 import synthetic as syn

    model = syn.make_model(5, 500, "scatter", mu_tau=-3.0, seed=11)
    engine.set_model_from(model)
    p0 = syn.make_packets(1, model.r_inner[0])
    res = engine.run_packets(p0.slice(0, 0))
    assert res["output_nus"].shape == (0,) and res["j"].sum() == 0.0
    res = engine.run_packets(p0)
    ref = oracle.run_oracle(model, p0)
    assert_close(res["output_nus"], ref["output_nus"], 1e-12, "nu")
    assert same_counters(res["counters"], ref["counters"])


def test_ragged_warp_fill(engine, oracle):
    """Packet counts that are not multiples of the warp / grid size."""
    from tardis_b200 import synthetic as syn

    model = syn.make_model(6, 1500, "scatter", mu_tau=-3.5, seed=12)
    engine.set_model_from(model)
    for n in (31, 33, 1000, 37889):
        pk = syn.make_packets(n, model.r_inner[0], base_seed=n)
        res = engine.run_packets(pk)
        ref = oracle.run_oracle(model, pk, nthreads=4)
        assert same_counters(res["counters"], ref["counters"])
        assert_close(res["output_energies"], ref["output_energies"], 1e-11, "energies")


def test_sliced_noncontiguous_tau(engine, oracle):
    """The reference hands tau_sobolev[:, i:j] as a non-contiguous view (modes/classic/solver.py:132-134)."""
    from tardis_b200 import synthetic as syn

    full = syn.make_model(12, 2000, "macroatom", mu_tau=-4.0, seed=13)
    sl = slice(2, 9)
    view = syn.Model(
        r_inner=full.r_inner[sl].copy(), r_outer=full.r_outer[sl].copy(), v_inner=full.v_inner[sl].copy(),
        v_outer=full.v_outer[sl].copy(), time_explosion=full.time_explosion,
        electron_density=full.electron_density[sl].copy(), t_electrons=full.t_electrons[sl].copy(),
        line_list_nu=full.line_list_nu, tau_sobolev=full.tau_sobolev[:, sl],
        macro=syn.MacroAtomTables(full.macro.transition_probabilities[:, sl], full.macro.line2macro_level_upper,
                                  full.macro.macro_block_edge_index, full.macro.transition_type,
                                  full.macro.destination_level_id, full.macro.transition_line_id),
        spectrum_frequency_grid=full.spectrum_frequency_grid, line_interaction_type="macroatom")
    assert not view.tau_sobolev.flags["C_CONTIGUOUS"]
    pk = syn.make_packets(3000, view.r_inner[0], base_seed=21)
    engine.set_model_from(view)
    res = engine.run_packets(pk)
    ref = oracle.run_oracle(view, pk, nthreads=4)
    assert same_counters(res["counters"], ref["counters"])
    assert_close(res["j_blue"], ref["j_blue"], 1e-10, "j_blue")


def test_error_conditions(engine):
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import EngineError, MacroAtomError

    model = syn.make_model(4, 300, "macroatom", mu_tau=-2.0, seed=14)
    bad = syn.make_model(4, 300, "macroatom", mu_tau=-2.0, seed=14)
    bad.macro.transition_probabilities[:] = 0.0  # every activated block runs out -> MacroAtomError in the reference
    engine.set_model_from(bad)
    with pytest.raises(MacroAtomError):
        engine.run_packets(syn.make_packets(500, bad.r_inner[0]))
    unsorted = syn.make_model(4, 300, "scatter", seed=15)
    unsorted.line_list_nu[10], unsorted.line_list_nu[200] = unsorted.line_list_nu[200], unsorted.line_list_nu[10]
    with pytest.raises(EngineError):
        engine.set_model_from(unsorted)
    engine.set_model_from(model)  # engine stays usable
    engine.run_packets(syn.make_packets(100, model.r_inner[0]))


def test_solver_surface_end_to_end(engine, oracle, monkeypatch):
    """MCTransportSolverB200.from_config / initialize_transport_state / run with duck-typed reference objects
    (shell-sliced opacity state, virtual packets + logging) against the oracle."""
    from types import SimpleNamespace

    from tardis_b200 import montecarlo as mc
    from tardis_b200 import synthetic as syn
    from test_host_logic import _fake_config

    monkeypatch.setattr(mc, "get_engine", lambda device=0: engine)
    full = syn.make_model(10, 2500, "macroatom", mu_tau=-3.5, seed=41)
    sl = slice(1, 9)
    packets = syn.make_packets(1500, full.r_inner[sl][0], base_seed=3)
    pc = mc.PacketCollection(packets.initial_radii, packets.initial_nus, packets.initial_mus, packets.initial_energies,
                             packets.packet_seeds, packets.radiation_field_luminosity)
    geo = mc.HomologousGeometry(full.r_inner[sl], full.r_outer[sl], full.v_inner[sl], full.v_outer[sl], full.time_explosion)
    cfg = _fake_config(**{"spectrum.virtual.virtual_packet_logging": True, "spectrum.start": full.spectrum_frequency_grid[-1],
                          "spectrum.stop": full.spectrum_frequency_grid[0], "spectrum.num": len(full.spectrum_frequency_grid) - 1})
    source = SimpleNamespace(base_seed=1, create_packets=lambda n, seed_offset=0: pc)
    solver = mc.MCTransportSolverB200.from_config(cfg, source)
    sim_state = SimpleNamespace(geometry=SimpleNamespace(to_numba=lambda: geo, v_inner_boundary_idx=1, v_outer_boundary_idx=9),
                                time_explosion=full.time_explosion)
    opacity_host = SimpleNamespace(to_numba=lambda macro_atom_state, lit: mc.OpacityState.from_model(full))
    plasma = SimpleNamespace(continuum_interaction_species=SimpleNamespace(empty=True))
    state = solver.initialize_transport_state(sim_state, opacity_host, None, plasma, len(pc.initial_nus), no_of_virtual_packets=3)
    vhist = solver.run(state, show_progress_bars=False)

    view = syn.Model(r_inner=geo.r_inner, r_outer=geo.r_outer, v_inner=geo.v_inner, v_outer=geo.v_outer,
                     time_explosion=full.time_explosion, electron_density=full.electron_density[sl].copy(),
                     t_electrons=full.t_electrons[sl].copy(), line_list_nu=full.line_list_nu,
                     tau_sobolev=np.ascontiguousarray(full.tau_sobolev[:, sl]),
                     macro=syn.MacroAtomTables(np.ascontiguousarray(full.macro.transition_probabilities[:, sl]),
                                               full.macro.line2macro_level_upper, full.macro.macro_block_edge_index,
                                               full.macro.transition_type, full.macro.destination_level_id,
                                               full.macro.transition_line_id),
                     spectrum_frequency_grid=np.asarray(getattr(solver.spectrum_frequency_grid, "value", solver.spectrum_frequency_grid)),
                     line_interaction_type="macroatom")
    mcfg = solver.montecarlo_configuration
    ref = oracle.run_oracle(view, packets, number_of_vpackets=3, spawn_start=mcfg.VPACKET_SPAWN_START_FREQUENCY,
                            spawn_end=mcfg.VPACKET_SPAWN_END_FREQUENCY, vlog_capacity=200000)
    assert_close(vhist, ref["vhist"], 1e-10, "vhist")
    assert_close(state.j_estimator, ref["j"], 1e-10, "j")
    assert_close(state.j_blue_estimator, ref["j_blue"], 1e-10, "j_blue")
    assert_close(pc.output_nus, ref["output_nus"], 1e-11, "output_nus")
    df = state.tracker_last_interaction_df
    assert np.array_equal(df["line_absorb_id"].to_numpy(), ref["last_line_absorb_id"])
    assert np.array_equal(df["event_id"].to_numpy(), ref["last_event_id"])
    m = ref["vlog_count"]
    vp_nus = np.asarray(getattr(state.virt_packet_nus, "value", state.virt_packet_nus))
    assert len(vp_nus) == m
    order = np.argsort(ref["vlog_packet_index"][:m], kind="stable")
    assert_close(np.sort(vp_nus), np.sort(ref["vlog_nus"][:m][order]), 1e-11, "virt_packet_nus")


def test_two_gpu_nccl_allreduce(oracle):
    """Packet sharding over 2 GPUs with the single estimator all-reduce (NCCL); skipped on a 1-GPU box."""
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import subprocess
    import sys

    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
                        "127.0.0.1", "--master-port", "29513", "tests/nccl_worker.py"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "NCCL_PARITY_OK" in r.stdout


def test_scan_and_jump_agree_at_scale(oracle):
    """Two independent formulations of the same path (streaming scan vs prefix-table jump) on the bench model
    (5e5 lines, 20 shells, macroatom) with 1e6 packets: identical integer work counters and per-packet outputs,
    estimators to 1e-10; plus size-independent invariants the domain offers."""
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import Engine

    model = syn.make_model(20, 500_000, "macroatom")
    packets = syn.make_packets(1_000_000, model.r_inner[0], base_seed=424242)
    results = {}
    for name, algo in (("scan", 0), ("jump", 1)):
        eng = Engine(0)
        eng.set_option("algorithm", algo)
        eng.set_model_from(model)
        results[name] = eng.run_packets(packets)
        eng.close()
    a, b = results["scan"], results["jump"]
    ca = {k: v for k, v in a["counters"].items() if k != "n_search_probes"}
    cb = {k: v for k, v in b["counters"].items() if k != "n_search_probes"}
    assert ca == cb
    assert np.array_equal(a["output_nus"], b["output_nus"]) or np.allclose(a["output_nus"], b["output_nus"], rtol=1e-11, atol=0)
    assert np.array_equal(np.sign(a["output_energies"]), np.sign(b["output_energies"]))
    for k in ("j", "nu_bar", "j_blue", "edotlu"):
        assert_close(a[k], b[k], 1e-10, k)
    assert np.array_equal(a["j_blue"] == 0, b["j_blue"] == 0)
    # invariants: every packet ends emitted or reabsorbed; every packet crosses at least the start and end boundary
    # events; all estimators non-negative; each packet's energy only changes by Doppler factors (bounded)
    e = b["output_energies"]
    assert np.all(e != -99.0) and np.all(np.isfinite(e)) and np.all(np.isfinite(b["output_nus"]))
    assert b["counters"]["n_boundary_events"] >= 2 * len(packets)
    assert (b["j_blue"] >= 0).all() and (b["edotlu"] >= 0).all() and (b["j"] > 0).all()
    ratio = np.abs(e) / packets.initial_energies
    assert ratio.min() > 0.5 and ratio.max() < 2.0
    # a 2 % sample against the CPU oracle
    sub = packets.slice(0, 20_000)
    ref = oracle.run_oracle(model, sub, nthreads=8)
    assert_close(b["output_nus"][:20_000], ref["output_nus"], 1e-11, "output_nus vs oracle")


def test_pipelined_run_matches_resident(engine):
    """tb200_run splits >= 4e6 packets into ranges whose H2D / kernels / D2H overlap; the result must equal the
    single-launch device-resident path (per-packet outputs bit-identical, counters equal, estimators to 1e-12)."""
    from tardis_b200 import synthetic as syn

    model = syn.make_model(12, 6000, "macroatom", mu_tau=-5.0, seed=71)
    packets = syn.make_packets(4_200_000, model.r_inner[0], base_seed=72)
    engine.set_model_from(model)
    piped = engine.run_packets(packets)
    engine.upload_packets(packets.initial_radii, packets.initial_nus, packets.initial_mus, packets.initial_energies,
                          packets.packet_seeds)
    engine.transport(True)
    engine.sync()
    resident = engine.download()
    assert np.array_equal(piped["output_nus"], resident["output_nus"])
    assert np.array_equal(piped["output_energies"], resident["output_energies"])
    assert same_counters(piped["counters"], {k: v for k, v in resident["counters"].items() if k != "n_search_probes"})
    for k in ("j", "nu_bar", "j_blue", "edotlu"):
        assert_close(piped[k], resident[k], 1e-12, k)


def test_iip_transport_surface(engine, oracle):
    """`montecarlo_transport` (IIP signature, modes/iip/montecarlo_transport.py:40) with a duck-typed
    OpacityStateNumbaIIP against the oracle: continuum estimators, adiabatic-cooling packets keep -99."""
    from types import SimpleNamespace

    from tardis_b200 import montecarlo as mc
    from tardis_b200 import synthetic as syn

    model = syn.make_model(8, 2500, "macroatom", mu_tau=-4.0, seed=131)
    syn.add_continuum(model, seed=9131, adiabatic_fraction=0.3)
    packets = syn.make_packets(2000, model.r_inner[0], base_seed=132)
    pc = mc.PacketCollection(packets.initial_radii, packets.initial_nus, packets.initial_mus, packets.initial_energies,
                             packets.packet_seeds, packets.radiation_field_luminosity)
    geo = mc.HomologousGeometry(model.r_inner, model.r_outer, model.v_inner, model.v_outer, model.time_explosion)
    c, m = model.continuum, model.macro
    opa = SimpleNamespace(electron_density=model.electron_density, t_electrons=model.t_electrons, line_list_nu=model.line_list_nu,
                          tau_sobolev=model.tau_sobolev, **{k: getattr(m, k) for k in vars(m)}, **{k: getattr(c, k) for k in vars(c)})
    cfg = mc.MonteCarloConfiguration()
    cfg.LINE_INTERACTION_TYPE = 2
    cfg.ENABLE_FULL_RELATIVITY = True
    trackers = mc.generate_tracker_last_interaction_list(len(packets))
    bulk, line, cont = mc.montecarlo_transport(pc, geo, model.time_explosion, opa, cfg,
                                               (len(c.bf_threshold_list_nu), model.n_shells), trackers, False, engine=engine)
    ref = oracle.run_oracle(model, packets)
    assert np.array_equal(pc.output_energies == -99.0, ref["output_energies"] == -99.0)
    assert_close(pc.output_nus, ref["output_nus"], 1e-11, "output_nus")
    assert_close(bulk.mean_intensity_total, ref["j"], 1e-10, "j")
    assert_close(line.mean_intensity_blueward, ref["j_blue"], 1e-10, "j_blue")
    for k in ("photo_ion_estimator", "stim_recomb_estimator", "bf_heating_estimator", "stim_recomb_cooling_estimator", "ff_heating_estimator"):
        assert_close(getattr(cont, k), ref[k], 1e-10, k)
    assert np.array_equal(cont.photo_ion_estimator_statistics, ref["photo_ion_estimator_statistics"])
    assert np.array_equal(trackers.columns["last_interaction_type"], ref["last_interaction_type"])
    assert (trackers.columns["last_interaction_type"] == 8).sum() > 0  # CONTINUUM_PROCESS
    assert same_counters(mc.montecarlo_transport.last_counters, ref["counters"])


def test_fused_spectrum_and_luminosity_sums_match_the_oracle(engine, oracle):
    """The in-kernel emitted / reabsorbed energy histograms and the four luminosity sums against what the reference's
    consumers compute from the ORACLE's per-packet outputs: numpy.histogram (SpectrumSolver.montecarlo_emitted_luminosity,
    tardis/spectrum/base.py:139-159, up to the 1/t_simulation factor) and calculate_filtered_luminosity
    (spectrum/luminosity.py:5-29, strict window)."""
    from tardis_b200 import synthetic as syn

    model = syn.make_model(10, 4000, "macroatom", mu_tau=-4.0, seed=81, n_bins=500)
    packets = syn.make_packets(60000, model.r_inner[0], base_seed=82)
    ref = oracle.run_oracle(model, packets, nthreads=8)
    nu, e = ref["output_nus"], ref["output_energies"]
    lo, hi = 4.0e14, 1.1e15
    engine.set_model_from(model, luminosity_nu_start=lo, luminosity_nu_end=hi)
    res = engine.run_packets(packets)
    grid = model.spectrum_frequency_grid
    em, _ = np.histogram(nu[e >= 0], weights=e[e >= 0], bins=grid)
    re, _ = np.histogram(nu[e < 0], weights=-e[e < 0], bins=grid)
    assert em.sum() > 0 and re.sum() > 0
    assert_close(res["spectrum_emitted"], em, 1e-11, "spectrum_emitted", atol=1e-18)
    assert_close(res["spectrum_reabsorbed"], re, 1e-11, "spectrum_reabsorbed", atol=1e-18)
    assert np.array_equal(res["spectrum_emitted"] == 0, em == 0)
    window = (nu > lo) & (nu < hi)
    want = np.array([e[e >= 0].sum(), e[(e >= 0) & window].sum(), -e[e < 0].sum(), -e[(e < 0) & window].sum()])
    assert 0 < want[1] < want[0] and 0 < want[3] < want[2]
    assert_close(res["luminosity_sums"], want, 1e-11, "luminosity_sums")
    # the per-packet arrays are optional: estimators + spectrum only
    lean = engine.run_packets(packets, per_packet=False)
    assert "output_nus" not in lean
    assert_close(lean["spectrum_emitted"], em, 1e-11, "spectrum_emitted (no per-packet D2H)", atol=1e-18)
    assert_close(lean["luminosity_sums"], want, 1e-11, "luminosity_sums (no per-packet D2H)")


def test_accumulating_across_calls_refuses_a_different_energy_scale(engine):
    """transport(zero_estimators=False) adds to what the tables hold; the jump algorithm's fixed-point difference arrays carry
    one scale, so packets of a very different typical energy must start a fresh accumulation (EngineError), while the same
    scale accumulates: twice the same packets == twice the estimators."""
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import EngineError

    model = syn.make_model(6, 2000, "scatter", mu_tau=-4.0, seed=91)
    packets = syn.make_packets(5000, model.r_inner[0], base_seed=92)
    engine.set_model_from(model)
    args = (packets.initial_radii, packets.initial_nus, packets.initial_mus, packets.initial_energies, packets.packet_seeds)
    engine.upload_packets(*args)
    engine.transport(True); engine.sync()
    once = engine.download()
    engine.transport(False); engine.sync()
    twice = engine.download()
    for k in ("j", "nu_bar", "j_blue", "edotlu"):
        assert_close(twice[k], 2 * once[k], 1e-12, k)
    engine.upload_packets(packets.initial_radii, packets.initial_nus, packets.initial_mus, packets.initial_energies * 1e6, packets.packet_seeds)
    if engine.download()["counters"]["n_search_probes"] > 0:  # jump algorithm only: the scan kernels add floating point directly
        with pytest.raises(EngineError):
            engine.transport(False)
    engine.transport(True); engine.sync()  # a fresh accumulation is fine


@pytest.mark.parametrize("n_lines,n_shells", [(1, 1), (2, 1), (3, 2), (31, 3), (32, 2), (33, 2), (65, 1)])
def test_degenerate_table_sizes(engine, oracle, n_lines, n_shells):
    """Line lists shorter than one warp step / one shell: the last line can never be interacted with
    (MISS_DISTANCE), chunk alignment and the bucket table must not assume a minimum size."""
    from tardis_b200 import synthetic as syn

    model = syn.make_model(n_shells, n_lines, "macroatom", mu_tau=-1.0, seed=900 + n_lines, duplicate_fraction=0.0,
                           n_levels=max(2, n_lines // 2))
    packets = syn.make_packets(3000, model.r_inner[0], base_seed=901)
    engine.set_model_from(model, number_of_vpackets=2)
    res = engine.run_packets(packets, track_last_interaction=True)
    ref = oracle.run_oracle(model, packets, number_of_vpackets=2, nthreads=4)
    assert same_counters(res["counters"], ref["counters"])
    assert_close(res["output_nus"], ref["output_nus"], 1e-11, "output_nus")
    assert_close(res["output_energies"], ref["output_energies"], 1e-11, "output_energies")
    for k in ("j", "nu_bar", "j_blue", "edotlu", "vhist"):
        assert_close(res[k], ref[k], 1e-10, k)
    assert np.array_equal(res["last_line_absorb_id"], ref["last_line_absorb_id"])


def test_seed_uses_low_32_bits(engine):
    """np.random.seed takes a uint32 (numba/cpython/randomimpl.py:213-225): seeds that differ by 2**32 give the same packet."""
    from tardis_b200 import synthetic as syn

    model = syn.make_model(5, 800, "scatter", mu_tau=-3.0, seed=77)
    packets = syn.make_packets(500, model.r_inner[0], base_seed=5)
    engine.set_model_from(model)
    a = engine.run_packets(packets)
    shifted = syn.Packets(packets.initial_radii, packets.initial_nus, packets.initial_mus, packets.initial_energies,
                          packets.packet_seeds + 2**32, packets.radiation_field_luminosity)
    b = engine.run_packets(shifted)
    assert np.array_equal(a["output_nus"], b["output_nus"]) and np.array_equal(a["output_energies"], b["output_energies"])


@pytest.mark.parametrize("park_min,refill_min,ctas,threads", [(1, 1, 1, 128), (32, 32, 2, 128), (7, 3, 4, 256), (16, 8, 3, 256), (2, 32, 2, 256)])
def test_pooled_kernel_scheduling_is_invisible(oracle, park_min, refill_min, ctas, threads):
    """The pooled jump kernel moves packets between lanes and shared-memory slots; how often it parks, swaps and
    refills (and so which lane finishes a packet, where its MT ring lives) must not change any trajectory.  The
    optically thick model makes every packet long-lived (hundreds of draws: ring tiers 2 and 3 migrate too)."""
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import Engine

    model = syn.make_model(4, 3000, "macroatom", mu_tau=-2.0, seed=31)
    model.electron_density[:] *= 100.0
    packets = syn.make_packets(20000, model.r_inner[0], base_seed=17)
    ref = oracle.run_oracle(model, packets, nthreads=8, n_tracked_packets=100, max_events_per_packet=8192)
    assert ref["counters"]["n_rng_draws"] / len(packets) > 100
    eng = Engine(0)
    for k, v in (("algorithm", 1), ("pooled", 1), ("park_min", park_min), ("refill_min", refill_min), ("ctas_per_sm", ctas),
                 ("threads_per_cta", threads)):
        eng.set_option(k, v)
    eng.set_model_from(model)
    res = eng.run_packets(packets, track_last_interaction=True, n_tracked_packets=100, max_events_per_packet=8192)
    eng.close()
    assert same_counters(res["counters"], ref["counters"])
    assert_close(res["output_nus"], ref["output_nus"], 1e-10, "output_nus")
    assert_close(res["output_energies"], ref["output_energies"], 1e-10, "output_energies")
    for k in ("last_interaction_type", "last_event_id", "last_shell_id", "last_line_absorb_id", "last_line_emit_id"):
        assert np.array_equal(res[k], ref[k]), k
    assert np.array_equal(res["event_counts"], ref["event_counts"])
    for k in ("j", "nu_bar", "j_blue", "edotlu"):
        assert_close(res[k], ref[k], 1e-10, k)


@pytest.mark.parametrize("vol_min", [1, 32])
def test_warp_volley_batching_does_not_change_results(oracle, vol_min):
    """The warp-cooperative volleys give the oracle's numbers whether they run for one waiting packet or for a full warp."""
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import Engine

    model = syn.make_model(12, 6000, "macroatom", mu_tau=-3.5, seed=71)
    packets = syn.make_packets(6000, model.r_inner[0], base_seed=72)
    ref = oracle.run_oracle(model, packets, number_of_vpackets=5, nthreads=4, spawn_start=2e14, spawn_end=3e15)
    eng = Engine(0)
    eng.set_option("vol_min", vol_min)
    eng.set_model_from(model, number_of_vpackets=5, vpacket_spawn_start_frequency=2e14, vpacket_spawn_end_frequency=3e15)
    res = eng.run_packets(packets)
    assert same_counters(res["counters"], ref["counters"])
    assert_close(res["vhist"], ref["vhist"], 1e-11, "vhist")
    assert_close(res["output_nus"], ref["output_nus"], 1e-11, "output_nus")
    eng.close()
