"""The classic plasma on the device (tardis_b200/csrc/plasma.cuh, tb200_set_plasma_data / tb200_solve_plasma).

CPU: (1) the numpy / pandas oracle (oracle/plasma_oracle.py) reproduces the goldens of the unmodified property classes
(tests/golden/make_plasma_golden.py) bit for bit; (2) the PRODUCT's header, built for the host by tests/plasma_shim.cpp and
driven with the kernels' loops, reproduces them: identical n_e iteration counts and zero patterns, values within RTOL.
GPU: the kernels through the C-ABI against the same goldens; the resident hand-off to build_opacity / transport against the
host path, bit for bit; two iterations chained through the radiation field; engine groups; refusals.

RTOL: an ion of charge k carries a product of k Phi factors and n_e**-k.  Each Phi factor and each Boltzmann factor is a few
exp / pow results, which CUDA and glibc give within 1-2 ulp of each other (exp 1 ulp, pow 2 ulp); over k <= 30 factors and
n_e**-k that is at most ~30 x 8 ulp ~ 5e-14 relative per population pass, and the damped fixed point does not amplify it.
1e-12 leaves a margin of 20.  J_blue is W B_nu(T) cell by cell: radfield.cuh's nu * nu * nu against numpy's pow(nu, 3) and
one exp, the radiation-field tests' 1e-13."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden")
CASES = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.startswith("plasma_") and f.endswith(".npz"))
RTOL = 1e-12
RTOL_JBLUE = 1e-13
INPUTS = ("level_energy", "level_ion", "g", "metastable", "ion_atomic_number", "ion_charge", "ionization_energy", "number_density")
OPTIONS = ("ionization", "excitation", "radiative_rates_type", "link_t_rad_t_electron", "ion_zero_threshold", "delta_treatment",
           "departure_coefficient", "chi_0", "electron_densities")
OUTPUTS = ("electron_densities", "ion_number_density", "level_number_density", "j_blues")
EV = 1.602176565e-12


def load(name):
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    opts = {k: (g["opt_" + k].item() if g["opt_" + k].ndim == 0 else g["opt_" + k]) for k in OPTIONS if "opt_" + k in g}
    return g, opts


def max_rel(a, b):
    nz = b != 0
    return float(np.max(np.abs(a[nz] - b[nz]) / np.abs(b[nz]), initial=0.0))


def check(got, g, rtol=RTOL, keys=OUTPUTS):
    """identical iteration count and zero patterns, values within rtol (J_blue within RTOL_JBLUE); -> max rel. difference"""
    assert int(got["iterations"]) == int(g["iterations"])
    worst = 0.0
    for k in keys:
        a, b = np.asarray(got[k]), g[k]
        assert a.shape == b.shape, k
        assert np.array_equal(a == 0, b == 0), f"{k}: zero pattern differs"
        bar = RTOL_JBLUE if k == "j_blues" else rtol
        np.testing.assert_allclose(a, b, rtol=bar, atol=0, err_msg=k)
        worst = max(worst, max_rel(a, b))
    return worst


# ---- CPU --------------------------------------------------------------------------------------------------------------------
def test_goldens_cover_the_cases():
    """every ionisation x excitation pair, both black-body J_blue types, the options and the shapes the cases are named for"""
    seen = {(load(n)[1]["ionization"], load(n)[1]["excitation"]) for n in CASES}
    assert seen == {("nebular", "dilute-lte"), ("nebular", "lte"), ("lte", "dilute-lte"), ("lte", "lte")}
    assert {load(n)[1]["radiative_rates_type"] for n in CASES} == {"dilute-blackbody", "blackbody"}
    g, o = load("plasma_zeta_outside")
    assert ((g["t_rad"] < g["zeta_temperatures"][0]) | (g["t_rad"] > g["zeta_temperatures"][-1])).sum() == 2
    assert int(load("plasma_many_iterations")[0]["iterations"]) >= 10
    assert int(load("plasma_fixed_ne")[0]["iterations"]) == 0
    g, o = load("plasma_threshold")
    assert ((g["ion_number_density"] == 0).sum() > (load("plasma_nebular_dilute")[0]["ion_number_density"] == 0).sum())
    assert load("plasma_chi0_species")[1]["chi_0"] != load("plasma_nebular_dilute")[1]["chi_0"]
    g, _ = load("plasma_bench_shape")
    assert (len(g["level_energy"]), g["t_rad"].size, len(g["ion_charge"])) == (3000, 20, 495)


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_golden_bit_for_bit(name):
    from oracle import plasma_oracle

    g, opts = load(name)
    got = plasma_oracle.solve(*(g[k] for k in INPUTS), g["t_rad"], g["w"], zeta_temperatures=g["zeta_temperatures"], zeta=g["zeta"],
                              line_nu=g["line_nu"], **opts)
    assert got["iterations"] == int(g["iterations"])
    for k in OUTPUTS:
        assert np.array_equal(got[k], g[k], equal_nan=True), k  # NaN: the shell at n_e = 0 of plasma_fixed_ne


@pytest.fixture(scope="module")
def shim():
    out = os.path.join(HERE, "_shim", "libplasma_shim.so")
    src = os.path.join(HERE, "plasma_shim.cpp")
    csrc = os.path.join(ROOT, "tardis_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in ("plasma.cuh", "markov_build.cuh", "packet_source.cuh", "radfield.cuh", "formal_integral.cuh")]
    os.makedirs(os.path.dirname(out), exist_ok=True)
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in deps):
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", out, src], check=True)
    lib = C.CDLL(out)
    lib.shim_plasma.restype = C.c_int
    lib.shim_plasma.argtypes = [C.c_int] * 4 + [C.c_void_p] * 8 + [C.c_int] + [C.c_void_p] * 6 + [C.c_double] * 5 + [C.c_void_p] * 7

    def run(g, opts):
        from oracle import plasma_oracle as po
        from tardis_b200.engine import EXCITATION, IONIZATION, RADIATIVE_RATES_TYPE

        S, L, NL, NI = g["t_rad"].size, len(g["line_nu"]), len(g["level_energy"]), len(g["ion_charge"])
        a = dict(level_energy=g["level_energy"], level_ion=g["level_ion"].astype(np.int64), g=g["g"], metastable=g["metastable"].astype(np.uint8),
                 ion_z=g["ion_atomic_number"].astype(np.int64), ion_q=g["ion_charge"].astype(np.int64), chi=g["ionization_energy"],
                 nd=g["number_density"], zt=g["zeta_temperatures"], zeta=g["zeta"], t=g["t_rad"], w=g["w"], nu=g["line_nu"])
        a = {k: np.ascontiguousarray(v) for k, v in a.items()}
        o = np.array([IONIZATION[opts["ionization"]], EXCITATION[opts["excitation"]], RADIATIVE_RATES_TYPE[opts["radiative_rates_type"]]],
                     dtype=np.int32)
        fixed = opts.get("electron_densities")
        fixed = None if fixed is None else np.ascontiguousarray(fixed, dtype=np.float64)
        k = np.array([po.K_B, po.H, po.M_E, po.C])
        res = dict(electron_densities=np.empty(S), ion_number_density=np.empty((NI, S)), level_number_density=np.empty((NL, S)),
                   j_blues=np.empty((L, S)))
        passes = C.c_int(0)
        status = lib.shim_plasma(NL, NI, S, L, *(a[x].ctypes.data for x in ("level_energy", "level_ion", "g", "metastable", "ion_z", "ion_q",
                                                                            "chi", "nd")), len(a["zt"]), a["zt"].ctypes.data,
                                 a["zeta"].ctypes.data, a["t"].ctypes.data, a["w"].ctypes.data, a["nu"].ctypes.data, o.ctypes.data,
                                 opts["link_t_rad_t_electron"], opts.get("delta_treatment", np.nan), opts.get("departure_coefficient", np.nan),
                                 opts["chi_0"], opts["ion_zero_threshold"], None if fixed is None else fixed.ctypes.data, k.ctypes.data,
                                 *(res[x].ctypes.data for x in OUTPUTS), C.byref(passes))
        res["iterations"], res["status"] = passes.value, status
        return res

    return run


@pytest.mark.parametrize("name", CASES)
def test_product_header_matches_reference_golden(shim, name):
    g, opts = load(name)
    got = shim(g, opts)
    assert got["status"] == 0
    worst = check(got, g)
    print(f"{name}: max relative difference {worst:.2e} (bar {RTOL:g})")


def test_product_header_reports_nan_and_the_iteration_cap(shim):
    g, opts = load("plasma_nebular_dilute")
    bad = dict(g)
    bad["number_density"] = g["number_density"].copy()
    bad["number_density"][0, 2] = np.nan                     # a NaN reaches n_e: PlasmaIonizationError
    assert shim(bad, opts)["status"] == 1
    # Phi = 0 everywhere (exp underflows): every pass gives new n_e = 0, so n_e halves on every pass and never passes the
    # test; the reference would spin (down to n_e = 0 and then for ever), the header stops at its cap
    slow = dict(g, ionization_energy=np.where(g["ion_charge"] > 0, 1e-6, np.nan))
    r = shim(slow, opts)
    assert r["status"] == 2 and r["iterations"] == 1000


def frames(g):
    import pandas as pd

    lion, z, q = g["level_ion"], g["ion_atomic_number"], g["ion_charge"]
    idx = pd.MultiIndex.from_arrays([z[lion], q[lion], np.arange(len(lion))], names=["atomic_number", "ion_number", "level_number"])
    levels = pd.DataFrame({"energy": g["level_energy"], "g": g["g"], "metastable": g["metastable"]}, index=idx)
    ion_index = pd.MultiIndex.from_arrays([z, q], names=["atomic_number", "ion_number"])
    has = q > 0
    ionization = pd.Series(g["ionization_energy"][has], index=ion_index[has])
    elements = pd.unique(z)
    nd = pd.DataFrame(g["number_density"], index=pd.Index(elements, name="atomic_number"))
    zeta = pd.DataFrame(g["zeta"][has], index=ion_index[has], columns=g["zeta_temperatures"])
    return levels, ionization, nd, zeta


def test_frames_map_to_the_device_arrays():
    from tardis_b200 import plasma

    g, _ = load("plasma_bench_shape")
    levels, ionization, nd, zeta = frames(g)
    d = plasma.plasma_data(levels, ionization, nd.iloc[::-1], zeta)  # number_density rows in any order
    for k in ("level_energy", "level_ion", "ionization_energy", "number_density", "zeta_temperatures"):
        src = {"ionization_energy": g["ionization_energy"]}.get(k, g.get(k))
        assert np.array_equal(d[k], src, equal_nan=True), k
    assert np.array_equal(d["ion_atomic_number"], g["ion_atomic_number"]) and np.array_equal(d["ion_charge"], g["ion_charge"])
    assert np.array_equal(d["zeta"][g["ion_charge"] > 0], g["zeta"][g["ion_charge"] > 0])
    assert "chi_0" not in d
    assert plasma.plasma_data(levels, ionization, nd, zeta, chi_0_species=(6, 2))["chi_0"] == float(ionization.loc[(6, 2)])
    with pytest.raises(NotImplementedError):
        plasma.plasma_data(levels, ionization, nd, zeta, nlte_species=[(2, 0)])
    with pytest.raises(NotImplementedError):
        plasma.plasma_data(levels, ionization, nd, zeta, helium_treatment="recomb-nlte")
    with pytest.raises(NotImplementedError):
        plasma.plasma_data(levels, ionization, nd, zeta, continuum_interaction_species=["H I"])
    with pytest.raises(ValueError):
        plasma.plasma_data(levels, ionization, nd.iloc[1:], zeta)
    with pytest.raises(ValueError):
        plasma.plasma_data(levels, ionization, nd, zeta.iloc[1:])


# ---- GPU --------------------------------------------------------------------------------------------------------------------
def golden_engine(g, mode="macroatom", engine=None):
    """An engine on a model with the golden's line list, the golden's levels behind the lines and its plasma data."""
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import Engine

    S, L, NL = g["t_rad"].size, len(g["line_nu"]), len(g["level_energy"])
    model = syn.make_model(S, L, mode, seed=5)
    model.line_list_nu = g["line_nu"]
    atomic = syn.make_atomic_data(g["line_nu"], NL, mode, seed=6)
    atomic.lower_level, atomic.upper_level = g["lines_lower_level_index"], g["lines_upper_level_index"]
    atomic.g, atomic.metastable = g["g"], g["metastable"]
    eng = engine if engine is not None else Engine(0)
    set_tables(eng, model, atomic, mode)
    eng.set_plasma_data(**{k: g[k] for k in ("level_energy", "level_ion", "ion_atomic_number", "ion_charge", "ionization_energy",
                                             "number_density", "zeta_temperatures", "zeta")})
    return eng, model, atomic


def set_tables(eng, model, atomic, mode, electron_density=None):
    eng.set_model(r_inner=model.r_inner, r_outer=model.r_outer, time_explosion=model.time_explosion,
                  electron_density=model.electron_density if electron_density is None else electron_density,
                  line_list_nu=model.line_list_nu, tau_sobolev=None, line_interaction_type=mode, transition_probabilities=None,
                  line2macro_level_upper=atomic.line2macro_level_upper, macro_block_edge_index=atomic.macro_block_edge_index,
                  transition_type=atomic.transition_type, destination_level_id=atomic.destination_level_id,
                  transition_line_id=atomic.transition_line_idx, spectrum_frequency_grid=model.spectrum_frequency_grid)
    eng.set_atomic_data(lines_lower_level_index=atomic.lower_level, lines_upper_level_index=atomic.upper_level, g=atomic.g,
                        metastability=atomic.metastable, wavelength_cm=atomic.wavelength_cm, f_lu=atomic.f_lu, f_ul=atomic.f_ul,
                        energy_lower=atomic.energy[atomic.lower_level], energy_upper=atomic.energy[atomic.upper_level])


def solve_kwargs(opts):
    kw = {k: opts[k] for k in ("ionization", "excitation", "radiative_rates_type", "link_t_rad_t_electron", "ion_zero_threshold")}
    for k in ("delta_treatment", "departure_coefficient", "electron_densities"):
        if k in opts:
            kw[k] = opts[k]
    return kw


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_device_matches_reference_golden(name):
    g, opts = load(name)
    eng, _, _ = golden_engine(g)
    if opts["chi_0"] != 1.9020591570241798e-11:
        eng.set_plasma_data(**{k: g[k] for k in ("level_energy", "level_ion", "ion_atomic_number", "ion_charge", "ionization_energy",
                                                 "number_density", "zeta_temperatures", "zeta")}, chi_0=opts["chi_0"])
    got = eng.solve_plasma(g["t_rad"], g["w"], download=True, **solve_kwargs(opts))
    worst = check(got, g)
    print(f"{name}: max relative difference {worst:.2e} (bar {RTOL:g})")
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("ionization,excitation,rates", [(i, e, r) for i in ("nebular", "lte") for e in ("dilute-lte", "lte")
                                                          for r in ("dilute-blackbody", "blackbody")])
def test_device_matches_oracle_for_every_option_combination(ionization, excitation, rates):
    from oracle import plasma_oracle

    g, opts = load("plasma_nebular_dilute")
    opts = dict(opts, ionization=ionization, excitation=excitation, radiative_rates_type=rates)
    want = plasma_oracle.solve(*(g[k] for k in INPUTS), g["t_rad"], g["w"], zeta_temperatures=g["zeta_temperatures"], zeta=g["zeta"],
                               line_nu=g["line_nu"], **opts)
    eng, _, _ = golden_engine(g)
    got = eng.solve_plasma(g["t_rad"], g["w"], download=True, **solve_kwargs(opts))
    check(got, want)
    eng.close()


def transport_plasma(S, n_levels, L, mode, seed):
    """A model whose device-solved plasma gives tau >= 0 of order one: one element whose ion (1, 1) holds only the top level
    (which is only ever a line's upper level) and needs 100 eV, so the gas stays neutral; LTE excitation with energies
    rising with the level index makes every stimulated-emission factor non-negative."""
    from tardis_b200 import synthetic as syn

    model = syn.make_model(S, L, mode, mu_tau=-4.0, seed=seed)
    atomic = syn.make_atomic_data(model.line_list_nu, n_levels, mode, seed=seed + 1, nlte_fraction=0.0)
    st = syn.make_plasma_structure(atomic, S, (1,), seed=seed + 2, log_density=(0.0, 1.0))
    level_ion = np.zeros(n_levels, dtype=np.int64)
    level_ion[-1] = 1
    energy = atomic.energy - atomic.energy[0]
    energy[-1] = 0.0
    data = dict(level_energy=energy, level_ion=level_ion, ion_atomic_number=st.ion_atomic_number, ion_charge=st.ion_charge,
                ionization_energy=np.array([np.nan, 100 * EV]), number_density=st.number_density,
                zeta_temperatures=st.zeta_temperatures, zeta=st.zeta)
    rng = np.random.default_rng(seed + 3)
    return model, atomic, data, rng.uniform(9e3, 1.2e4, S), rng.uniform(0.1, 0.5, S)


def run_host_path(model, atomic, mode, ne, lnd, j_blues, packets):
    from tardis_b200.engine import Engine

    eng = Engine(0)
    set_tables(eng, model, atomic, mode, electron_density=ne)
    eng.build_opacity(lnd, model.time_explosion, j_blues)
    res = eng.run_packets(packets, track_last_interaction=True)
    eng.close()
    return res


PER_PACKET = ("output_nus", "output_energies", "j_blue", "edotlu", "last_interaction_type", "last_line_absorb_id", "last_line_emit_id",
              "last_shell_id")


@pytest.mark.gpu
@pytest.mark.parametrize("mode,rates", [("macroatom", "dilute-blackbody"), ("downbranch", "detailed")])
def test_resident_handoff_equals_the_host_path_bit_for_bit(mode, rates):
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import Engine

    model, atomic, data, t_rad, w = transport_plasma(10, 300, 4000, mode, seed=71)
    packets = syn.make_packets(20000, model.r_inner[0], base_seed=9)
    a = Engine(0)
    set_tables(a, model, atomic, mode)
    a.set_plasma_data(**data)
    if rates == "detailed":  # a transport on host tables first, so that the radiation field's J_blue is resident
        warm = syn.make_plasma_state(atomic, 10, model.time_explosion, seed=3, zero_fraction=0.0, inversion_fraction=0.0, noise=0.0)
        a.build_opacity(warm.level_number_density * 1e-9, model.time_explosion, warm.j_blues)
        a.run_packets(packets)
        volume = 4.0 / 3.0 * np.pi * (model.r_outer**3 - model.r_inner**3)
        _, _, rf_j_blues = a.solve_radiation_field(time_explosion=model.time_explosion, time_of_simulation=packets.time_of_simulation,
                                                   volume=volume)
        set_tables(a, model, atomic, mode)  # the order of an iteration: set_model, then the plasma
    sol = a.solve_plasma(t_rad, w, ionization="nebular", excitation="lte", radiative_rates_type=rates, download=True)
    a.build_opacity(None, model.time_explosion)
    tau = a.download_opacity()["tau_sobolev"]
    assert (tau >= 0).all() and tau.max() > 0.1
    res_a = a.run_packets(packets, track_last_interaction=True)
    a.close()
    j_blues = rf_j_blues if rates == "detailed" else sol["j_blues"]
    res_b = run_host_path(model, atomic, mode, sol["electron_densities"], sol["level_number_density"], j_blues, packets)
    assert res_a["counters"] == res_b["counters"]
    for k in PER_PACKET:
        assert np.array_equal(res_a[k], res_b[k]), k
    for k in ("j", "nu_bar"):  # f64 atomic sums: equal up to the order the atomics land in
        np.testing.assert_allclose(res_a[k], res_b[k], rtol=1e-13, err_msg=k)


@pytest.mark.gpu
def test_two_iterations_chained_through_the_radiation_field():
    """transport -> radiation field -> host damping -> solve_plasma -> build_opacity(None) -> transport, twice.  Each device
    plasma is held to the oracle on the same damped T_rad / W at RTOL.  A second chain drives the transports with the oracle's
    populations and J_blue through the host path: its tables differ from the device's by those ulps, so its estimators and
    damped T_rad / W are compared at 1e-8 (the device- against host-built-table bar of the opacity tests is 1e-9 per
    transport; the second plasma amplifies a T_rad difference by chi * beta ~ 1e2)."""
    from oracle import plasma_oracle
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import Engine

    mode = "macroatom"
    model, atomic, data, t_rad, w = transport_plasma(8, 300, 4000, mode, seed=81)
    volume = 4.0 / 3.0 * np.pi * (model.r_outer**3 - model.r_inner**3)
    engines = {"dev": Engine(0), "host": Engine(0)}
    state = {"dev": (t_rad.copy(), w.copy()), "host": (t_rad.copy(), w.copy())}
    for it in range(2):
        packets = syn.make_packets(20000, model.r_inner[0], base_seed=20 + it)
        res = {}
        for name, eng in engines.items():
            t, ww = state[name]
            want = plasma_oracle.solve(data["level_energy"], data["level_ion"], atomic.g, atomic.metastable, data["ion_atomic_number"],
                                       data["ion_charge"], data["ionization_energy"], data["number_density"], t, ww,
                                       zeta_temperatures=data["zeta_temperatures"], zeta=data["zeta"], ionization="nebular",
                                       excitation="lte", line_nu=model.line_list_nu)
            if name == "dev":
                set_tables(eng, model, atomic, mode)
                if it == 0:
                    eng.set_plasma_data(**data)
                sol = eng.solve_plasma(t, ww, ionization="nebular", excitation="lte", download=True)
                check(sol, dict(want, iterations=want["iterations"]))
                eng.build_opacity(None, model.time_explosion)
            else:
                set_tables(eng, model, atomic, mode, electron_density=want["electron_densities"])
                eng.build_opacity(want["level_number_density"], model.time_explosion, want["j_blues"])
            res[name] = eng.run_packets(packets)
            t_est, w_est, _ = eng.solve_radiation_field(time_explosion=model.time_explosion, time_of_simulation=packets.time_of_simulation,
                                                        volume=volume, want_j_blues=False)
            state[name] = (t + 0.5 * (t_est - t), ww + 0.5 * (w_est - ww))  # the reference's damped convergence, damping 0.5
        for k in ("j", "nu_bar"):
            np.testing.assert_allclose(res["dev"][k], res["host"][k], rtol=1e-8, err_msg=k)
        for a, b in zip(state["dev"], state["host"]):
            np.testing.assert_allclose(a, b, rtol=1e-8)
    for eng in engines.values():
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("peer_access", [1, 0])
def test_engine_group_gives_one_engine_s_plasma_bit_for_bit(peer_access):
    from tardis_b200.engine import EngineGroup

    g, opts = load("plasma_bench_shape")
    one, _, _ = golden_engine(g)
    want = one.solve_plasma(g["t_rad"], g["w"], download=True, **solve_kwargs(opts))
    one.close()
    grp = EngineGroup([0, 0])
    grp.set_option("peer_access", peer_access)
    golden_engine(g, engine=grp)
    got = grp.solve_plasma(g["t_rad"], g["w"], download=True, **solve_kwargs(opts))
    for k in (*OUTPUTS, "iterations"):
        assert np.array_equal(got[k], want[k]), k
    member = grp.members[1].solve_plasma(g["t_rad"], g["w"], download=True, **solve_kwargs(opts))
    for k in OUTPUTS:
        assert np.array_equal(member[k], want[k]), k
    grp.close()


@pytest.mark.gpu
def test_refusals_leave_the_engine_usable():
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import Engine, EngineError, PlasmaIonizationError

    mode = "macroatom"
    model, atomic, data, t_rad, w = transport_plasma(6, 200, 2000, mode, seed=91)
    eng = Engine(0)
    set_tables(eng, model, atomic, mode)
    with pytest.raises(EngineError, match="no tb200_solve_plasma"):  # build_opacity(None) with nothing resident
        eng.build_opacity(None, model.time_explosion)
    with pytest.raises(EngineError, match="set_plasma_data"):
        eng.solve_plasma(t_rad, w)

    def still_runs():
        set_tables(eng, model, atomic, mode)
        eng.set_plasma_data(**data)
        eng.solve_plasma(t_rad, w, excitation="lte")
        eng.build_opacity(None, model.time_explosion)
        res = eng.run_packets(syn.make_packets(2000, model.r_inner[0], base_seed=3))
        assert res["counters"]["n_boundary_events"] > 0

    still_runs()
    shuffled = dict(data, level_ion=data["level_ion"].copy())
    shuffled["level_ion"][[3, -1]] = shuffled["level_ion"][[-1, 3]]
    gap = dict(data, ion_charge=data["ion_charge"].copy())
    gap["ion_charge"][1] += 1
    missing = dict(data, ionization_energy=data["ionization_energy"].copy())
    missing["ionization_energy"][1] = np.nan
    for bad, msg in ((shuffled, "not grouped"), (gap, "not consecutive in charge"), (missing, "no ionisation energy")):
        with pytest.raises(EngineError, match=msg):
            eng.set_plasma_data(**bad)
        still_runs()
    nan_nd = dict(data, number_density=data["number_density"].copy())
    nan_nd["number_density"][0, 2] = np.nan
    eng.set_plasma_data(**nan_nd)
    with pytest.raises(PlasmaIonizationError, match="nan"):
        eng.solve_plasma(t_rad, w, excitation="lte")
    with pytest.raises(EngineError, match="no tb200_solve_plasma"):  # no populations are resident after the error
        eng.build_opacity(None, model.time_explosion)
    still_runs()
    eng.close()
    cont = syn.make_model(6, 500, "macroatom", seed=4)
    syn.add_continuum(cont)
    c = Engine(0)
    c.set_model_from(cont)
    with pytest.raises(EngineError, match="continuum"):
        c.set_plasma_data(**data)
    with pytest.raises(EngineError, match="continuum"):
        c.solve_plasma(t_rad, w)
    c.close()
    still_runs_after = Engine(0)
    set_tables(still_runs_after, model, atomic, mode)
    still_runs_after.close()
