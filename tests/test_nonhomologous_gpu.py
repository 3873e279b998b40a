"""The nonhomologous kernel (nh::transport_nonhomologous_kernel) through the C-ABI, against the CPU oracle
(oracle/nonhomologous_oracle.cpp), which evaluates the line distance with the same header.  Integers (work counters, fates,
last-interaction columns, event logs) identical; floats to 1e-10 (CUDA's log / exp against glibc's, and the order of the
estimator sums); line-estimator cells that receive one term bit-identical."""
import dataclasses
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_nonhomologous_golden as mk  # noqa: E402

RTOL = 1e-10
N_TRACKED = 20
INT_KEYS = ("last_interaction_type", "last_event_id", "last_shell_id", "last_line_absorb_id", "last_line_emit_id")
FLOAT_KEYS = ("output_nus", "output_energies", "last_radius", "last_before_nu", "last_before_mu", "last_before_energy",
              "last_after_nu", "last_after_mu", "last_after_energy")
SUM_KEYS = ("j", "nu_bar", "j_blue", "edotlu", "vhist")
EVENT_INT = ("packet_id", "interaction_type", "status", "before_shell_id", "after_shell_id", "line_absorb_id", "line_emit_id")


@pytest.fixture(scope="module")
def engine():
    from tardis_b200.engine import Engine

    eng = Engine(0)
    yield eng
    eng.close()


def config(kw):
    out = dict(nonhomologous=True, number_of_vpackets=kw.get("number_of_vpackets", 0),
               survival_probability=kw.get("survival_probability", 0.0),
               disable_line_scattering=kw.get("disable_line_scattering", False))
    if "sigma_thomson" in kw:
        out["sigma_thomson"] = kw["sigma_thomson"]
    return out


def oracle_run(model, packets, kw):
    from oracle import nonhomologous_oracle

    return nonhomologous_oracle.run_oracle(model, packets, n_tracked_packets=N_TRACKED, max_events_per_packet=4096,
                                           vlog_capacity=200000 if kw.get("number_of_vpackets") else 0, **kw)


def device_run(eng, model, packets, kw):
    eng.set_model_from(dataclasses.replace(model, time_explosion=0.0), **config(kw))  # the mode never reads it
    return eng.run_packets(packets, track_last_interaction=True, n_tracked_packets=N_TRACKED, max_events_per_packet=4096,
                           vlog_capacity=200000 if kw.get("number_of_vpackets") else 0)


def assert_matches(got, ref, sums_rtol=RTOL):
    for k in INT_KEYS:
        np.testing.assert_array_equal(got[k], ref[k], err_msg=k)
    for k in FLOAT_KEYS:
        np.testing.assert_allclose(got[k], ref[k], rtol=RTOL, atol=0, equal_nan=True, err_msg=k)
    for k in SUM_KEYS:
        np.testing.assert_allclose(got[k], ref[k], rtol=sums_rtol, atol=1e-300, err_msg=k)
    for k in ("n_line_steps", "n_boundary_events", "n_line_events", "n_escat_events", "n_rng_draws", "n_macro_jumps",
              "n_macro_scanned", "n_vpackets", "n_vpacket_line_steps"):
        assert got["counters"][k] == ref["counters"][k], k
    if "events" in ref:
        for a, b in zip(got["events"], ref["events"]):
            assert len(a) == len(b)
            for k in EVENT_INT:
                np.testing.assert_array_equal(a[k], b[k], err_msg=k)
            for k in ("radius", "before_nu", "before_mu", "before_energy", "after_nu", "after_mu", "after_energy"):
                np.testing.assert_allclose(a[k], b[k], rtol=RTOL, atol=0, err_msg=k)


def case(name, n_packets=None, **extra):
    model, packets, kw = mk.case_inputs(name)
    if n_packets is not None:
        from tardis_b200 import synthetic

        packets = synthetic.make_packets(n_packets, model.r_inner[0])
    kw.update(extra)
    return model, packets, kw


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(mk.CASES))
def test_device_matches_oracle(engine, name):
    model, packets, kw = case(name, n_packets=2000)
    assert_matches(device_run(engine, model, packets, kw), oracle_run(model, packets, kw))


@pytest.mark.gpu
def test_device_matches_oracle_without_electron_scattering(engine):
    model, packets, kw = case("macroatom_vpackets", n_packets=1000, sigma_thomson=1e-200)
    assert_matches(device_run(engine, model, packets, kw), oracle_run(model, packets, kw))


@pytest.mark.gpu
def test_alternating_gradient_signs(engine):
    """Every other shell decelerates, so the line scan changes direction at every crossing."""
    model, packets, kw = case("macroatom_vpackets", n_packets=1500)
    v = np.concatenate([model.v_inner, model.v_outer[-1:]])
    v[1:-1] = np.where(np.arange(1, len(v) - 1) % 2 == 1, v[2:] * 1.02, v[1:-1])
    model = dataclasses.replace(model, v_inner=v[:-1].copy(), v_outer=v[1:].copy())
    assert np.sum(model.v_outer < model.v_inner) >= 3
    assert_matches(device_run(engine, model, packets, kw), oracle_run(model, packets, kw))


@pytest.mark.gpu
def test_options_do_not_change_results(engine):
    model, packets, kw = case("downbranch", n_packets=800)
    ref = oracle_run(model, packets, kw)
    try:
        for algorithm, pooled in ((0, 0), (1, 0), (1, 1)):
            engine.set_option("algorithm", algorithm)
            engine.set_option("pooled", pooled)
            assert_matches(device_run(engine, model, packets, kw), ref)
    finally:
        engine.set_option("algorithm", 1)
        engine.set_option("pooled", 1)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [0, 1, 2, 33, 1009])
def test_packet_counts(engine, n):
    model, packets, kw = case("scatter", n_packets=max(n, 1))
    packets = dataclasses.replace(packets, **{k: getattr(packets, k)[:n] for k in (
        "initial_radii", "initial_nus", "initial_mus", "initial_energies", "packet_seeds")})
    got = device_run(engine, model, packets, kw)
    if n == 0:
        assert len(got["output_nus"]) == 0 and not np.any(got["j_blue"])
        return
    assert_matches(got, oracle_run(model, packets, kw))


@pytest.mark.gpu
def test_single_term_cells_are_bit_identical(engine):
    """Packets that never interact (tau_Sobolev = 1e-40, sigma_T = 1e-200), each in its own frequency window, so every
    J_blue / Edotlu cell receives at most one term: the cells must equal the oracle's bit for bit -- the device evaluates
    the quartic exactly as the host does."""
    from tardis_b200 import synthetic

    model, _, kw = case("macroatom_vpackets")
    model = dataclasses.replace(model, tau_sobolev=np.full_like(model.tau_sobolev, 1e-40))
    n = 24
    packets = synthetic.make_packets(n, model.r_inner[0])
    nus = np.geomspace(model.line_list_nu[-1] * 1.05, model.line_list_nu[0] / 1.05, n)  # 4 x the largest Doppler shift apart
    packets = dataclasses.replace(packets, initial_nus=nus)
    kw = dict(sigma_thomson=1e-200)
    ref, got = oracle_run(model, packets, kw), device_run(engine, model, packets, kw)
    assert ref["counters"]["n_line_events"] == 0 and ref["counters"]["n_escat_events"] == 0
    assert np.count_nonzero(ref["j_blue"]) > 500
    np.testing.assert_array_equal(got["j_blue"], ref["j_blue"])
    np.testing.assert_array_equal(got["edotlu"], ref["edotlu"])
    np.testing.assert_array_equal(got["output_nus"], ref["output_nus"])


def _shim():
    from test_nonhomologous import build_shim

    return build_shim()


def _flip(dist, lo, hi, flipped):
    """Adjacent doubles a < b in [lo, hi] with flipped(dist(a)) != flipped(dist(b)), by bisection over the bit patterns
    (positive doubles order like their patterns); None when the ends agree."""
    fa, fb = flipped(dist(lo)), flipped(dist(hi))
    if fa == fb:
        return None
    a, b = np.float64(lo).view(np.int64), np.float64(hi).view(np.int64)
    while b - a > 1:
        m = a + (b - a) // 2
        if flipped(dist(np.int64(m).view(np.float64))) == fa:
            a = m
        else:
            b = m
    return np.int64(a).view(np.float64), np.int64(b).view(np.float64)


@pytest.mark.gpu
def test_decision_thresholds(engine):
    """Lines on both sides of the two decision thresholds of a packet's first trace, found with the header's own
    distance (the oracle's, on the CPU): the 1e-14 resonance window (MISS on one side of the pair, a root on the other) and
    distance_trace == distance_boundary (the first line of the pair ends before the boundary, the second not).  Shell 0
    accelerates, so the scan is forward.  The device and the oracle then take the same decisions."""
    from tardis_b200 import synthetic

    shim = _shim()
    model, _, kw = case("scatter")
    v_in, v_out = model.v_inner.copy(), model.v_outer.copy()
    v_out[0] = v_in[1] = v_in[0] * 1.05
    model = dataclasses.replace(model, v_inner=v_in, v_outer=v_out)
    packets = synthetic.make_packets(32, model.r_inner[0])
    ri, ro, vi, vo = model.r_inner[0], model.r_outer[0], model.v_inner[0], model.v_outer[0]
    c_inv = 1 / 2.99792458e10
    extra = []
    for r, mu, nu0 in zip(packets.initial_radii, packets.initial_mus, packets.initial_nus):
        nu = nu0 * (1.0 / (1.0 - mu * (vi * c_inv)))             # set_packet_props_partial_relativity at r = r_inner[0]
        cnu = nu * (1.0 - mu * (vi / 2.99792458e10))             # the header's comoving frequency there
        d_b = np.sqrt(ro * ro + ((mu * mu - 1.0) * r * r)) - (r * mu)

        def dist(nl, r=r, mu=mu, nu=nu):
            return shim.shim_distance_line(r, mu, nu, nl, ri, ro, vi, vo)

        window = _flip(dist, cnu * (1 - 1e-13), cnu, lambda d: d >= 1e99)
        boundary = _flip(dist, cnu * (1 - 0.2), cnu * (1 - 1e-12), lambda d, d_b=d_b: d > d_b)
        assert window is not None and boundary is not None
        assert dist(window[0]) < 1e99 <= dist(window[1])
        assert dist(boundary[1]) < d_b <= dist(boundary[0]) or dist(boundary[0]) <= d_b < dist(boundary[1])
        extra += [*window, *boundary]
    nu = np.sort(np.concatenate([model.line_list_nu, extra]))[::-1].copy()
    tau = 10.0 ** np.random.default_rng(3).normal(-4, 2, (len(nu), model.n_shells))
    model = dataclasses.replace(model, line_list_nu=nu, tau_sobolev=tau)
    assert_matches(device_run(engine, model, packets, kw), oracle_run(model, packets, kw))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(mk.RADFIELD_CASES))
def test_radiation_field_matches_reference_golden(engine, name):
    """tb200_solve_radiation_field with velocity_gradient: the nonhomologous normalisation (c / dvdr) / (4 pi t_sim V)."""
    model, _, _ = case(mk.RADFIELD_CASES[name])
    engine.set_model_from(dataclasses.replace(model, time_explosion=0.0), nonhomologous=True)
    i = mk.radfield_inputs(name)
    g = dict(np.load(os.path.join(HERE, "golden", f"nonhomologous_{name}.npz")))
    t, w, jb = engine.solve_radiation_field(time_explosion=0.0, time_of_simulation=i["time_of_simulation"], volume=i["volume"],
                                            w_epsilon=i["w_epsilon"], estimators=(i["j"], i["nu_bar"], i["j_blue"]),
                                            velocity_gradient=i["velocity_gradient"])
    np.testing.assert_allclose(t, g["t_radiative"], rtol=1e-13, atol=0)
    np.testing.assert_allclose(w, g["dilution_factor"], rtol=1e-13, atol=0)
    np.testing.assert_allclose(jb, g["j_blues"], rtol=1e-13, atol=0, equal_nan=True)


@pytest.mark.gpu
def test_radiation_field_refusals(engine):
    from tardis_b200.engine import EngineError

    model, _, _ = case("scatter")
    S = model.n_shells
    vol = np.ones(S)
    engine.set_model_from(model, nonhomologous=True)
    with pytest.raises(EngineError, match="velocity_gradient"):  # time_explosion = 0 would give an all-zero J_blue
        engine.solve_radiation_field(time_explosion=0.0, time_of_simulation=1.0, volume=vol)
    engine.set_model_from(model)
    with pytest.raises(EngineError, match="homologous"):
        engine.solve_radiation_field(time_explosion=1.0, time_of_simulation=1.0, volume=vol, velocity_gradient=np.ones(S))


@pytest.mark.gpu
def test_solver_mirror_end_to_end(engine):
    """MCTransportSolverB200Nonhomologous.run on a state whose geometry carrier is NumbaRadial1DGeometry-shaped, then the
    nonhomologous radiation-field mirror on the estimators left in HBM, against the oracle."""
    from types import SimpleNamespace

    from oracle import nonhomologous_oracle
    from tardis_b200 import montecarlo as mc

    model, packets, kw = case("macroatom_vpackets", n_packets=1500)
    mac = model.macro
    geo = SimpleNamespace(r_inner=model.r_inner, r_outer=model.r_outer, v_inner=model.v_inner, v_outer=model.v_outer,
                          velocity_gradient=(model.v_outer - model.v_inner) / (model.r_outer - model.r_inner))
    opacity = SimpleNamespace(electron_density=model.electron_density, line_list_nu=model.line_list_nu,
                              tau_sobolev=model.tau_sobolev, transition_probabilities=mac.transition_probabilities,
                              line2macro_level_upper=mac.line2macro_level_upper, macro_block_edge_index=mac.macro_block_edge_index,
                              transition_type=mac.transition_type, destination_level_id=mac.destination_level_id,
                              transition_line_id=mac.transition_line_id)
    pc = mc.PacketCollection(packets.initial_radii, packets.initial_nus, packets.initial_mus, packets.initial_energies,
                             packets.packet_seeds, packets.radiation_field_luminosity)
    state = mc.MonteCarloTransportStateB200Nonhomologous(pc, geo, opacity, (0, 0))
    cfg = mc.MonteCarloConfiguration()
    cfg.LINE_INTERACTION_TYPE = 2
    cfg.NUMBER_OF_VPACKETS = kw["number_of_vpackets"]
    cfg.SURVIVAL_PROBABILITY = kw["survival_probability"]
    cfg.VPACKET_SPAWN_START_FREQUENCY, cfg.VPACKET_SPAWN_END_FREQUENCY = 0.0, 1e200
    solver = mc.MCTransportSolverB200Nonhomologous(None, model.spectrum_frequency_grid, None, False, "macroatom", "real", None,
                                                   montecarlo_configuration=cfg)
    vhist = solver.run(state, show_progress_bars=False)
    ref = oracle_run(model, packets, kw)
    np.testing.assert_allclose(state.output_nu if not hasattr(state.output_nu, "value") else state.output_nu.value,
                               ref["output_nus"], rtol=RTOL)
    np.testing.assert_allclose(vhist, ref["vhist"], rtol=RTOL, atol=1e-300)
    np.testing.assert_allclose(state.j_blue_estimator, ref["j_blue"], rtol=RTOL, atol=1e-300)
    np.testing.assert_allclose(state.j_estimator, ref["j"], rtol=RTOL)
    np.testing.assert_array_equal(state.tracker_last_interaction_df is not None, True)
    # the radiation field on the estimators still resident in HBM
    volume = (4 / 3) * np.pi * (model.r_outer**3 - model.r_inner**3)
    rf = mc.MCRadiationFieldPropertiesSolverB200Nonhomologous(1e-10).solve(
        state.estimators_bulk, state.estimators_line, geo.velocity_gradient, pc.time_of_simulation, volume, model.line_list_nu)
    t, w, jb = nonhomologous_oracle.solve_radiation_field(ref["j"], ref["nu_bar"], ref["j_blue"], geo.velocity_gradient,
                                                          pc.time_of_simulation, volume, model.line_list_nu)
    np.testing.assert_allclose(rf.dilute_blackbody_radiationfield_state.temperature_kelvin, t, rtol=1e-9)
    np.testing.assert_allclose(rf.j_blues, jb, rtol=1e-9, atol=0)
@pytest.mark.gpu
def test_engine_group_matches_one_engine(engine):
    from tardis_b200.engine import EngineGroup

    model, packets, kw = case("macroatom_vpackets", n_packets=1200)
    ref = device_run(engine, model, packets, kw)
    g = EngineGroup([0, 0])
    try:
        res = device_run(g, model, packets, kw)
    finally:
        g.close()
    for k in INT_KEYS + ("output_nus", "output_energies"):
        np.testing.assert_array_equal(res[k], ref[k], err_msg=k)
    for k in SUM_KEYS:
        np.testing.assert_allclose(res[k], ref[k], rtol=1e-12, atol=1e-300, err_msg=k)
    assert res["counters"] == ref["counters"]


@pytest.mark.gpu
def test_device_packet_source_then_run_resident(engine):
    from tardis_b200 import synthetic

    model, _, kw = case("downbranch")
    engine.set_model_from(dataclasses.replace(model, time_explosion=0.0), **config(kw))
    engine.create_packets(1500, 1963, model.r_inner[0], 1.0e4)
    got = engine.run_resident(track_last_interaction=True)
    src = engine.download_packets()  # what the device source made (tests/test_packet_source.py pins it against numpy)
    packets = synthetic.Packets(**src, radiation_field_luminosity=1.0)
    ref = oracle_run(model, packets, kw)
    for k in INT_KEYS:
        np.testing.assert_array_equal(got[k], ref[k], err_msg=k)
    np.testing.assert_allclose(got["output_nus"], ref["output_nus"], rtol=RTOL)


@pytest.mark.gpu
def test_refusals(engine):
    from tardis_b200.engine import EngineError

    model, _, _ = case("scatter")
    with pytest.raises(NotImplementedError, match="Full relativity not supported for non-homology."):
        engine.set_model_from(model, nonhomologous=True, enable_full_relativity=True)
    with pytest.raises(ValueError, match="v_inner and v_outer"):
        engine.set_model(r_inner=model.r_inner, r_outer=model.r_outer, time_explosion=0.0,
                         electron_density=model.electron_density, line_list_nu=model.line_list_nu,
                         tau_sobolev=model.tau_sobolev, spectrum_frequency_grid=model.spectrum_frequency_grid, nonhomologous=True)
    engine.set_model_from(model, nonhomologous=True)
    with pytest.raises(EngineError, match="line accumulators"):
        engine.line_accumulators()
