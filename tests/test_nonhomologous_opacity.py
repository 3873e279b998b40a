"""The nonhomologous mode's opacity build on the device (opacity_line_nonhomologous_kernel, tb200_build_opacity with
tb200_plasma_state.velocity_gradient): tau = lambda f_lu COEFF / dv/dr * stim * n_lower, then the homologous mode's beta and
macro-atom probabilities.

CPU: the numpy oracle (oracle/opacity_oracle_nonhomologous.py) and the product's header, built for the host by
tests/nonhomologous_opacity_shim.cpp, against golden vectors of the reference's own functions
(tests/golden/make_nonhomologous_opacity_golden.py: tau, beta and the normalised probabilities; the stimulated-emission
factor, a restatement there too, is compared with the oracle's).  tau is four IEEE operations in numpy's order:
bit-identical.  The other tables have the bars of tests/test_opacity_build.py.
GPU: the device-built tables against the goldens (a decelerating shell with tau < 0 and beta > 1, a shell with |dv/dr|
1e-6 of the others, a shell on v = r / t), the flat shell's error, the refusals, an engine group, the bench shape, and
two iterations of transport -> radiation field -> opacity build -> transport that never leave the device, against the
same chain fed the oracle's host tables through set_model."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_nonhomologous_opacity_golden as mko  # noqa: E402

GOLDEN_DIR = os.path.join(HERE, "golden")
CASES = [n for n in mko.CASES if n != "flat_shell"]
TOL = {"stimulated_emission_factor": 1e-14, "tau_sobolev": 0.0, "beta_sobolev": 1e-11, "raw_probabilities": 1e-11,
       "transition_probabilities": 1e-11}
DEVICE_KEYS = ("stimulated_emission_factor", "tau_sobolev", "beta_sobolev", "transition_probabilities")
GOLDEN_KEYS = mko.STORED  # what the golden holds; the rest is compared with the oracle


def load(name):
    model, atomic, plasma = mko.case_inputs(name)
    return model, atomic, plasma, dict(np.load(os.path.join(GOLDEN_DIR, f"nonhomologous_opacity_{name}.npz")))


def check(got, want, keys=GOLDEN_KEYS):
    for k in keys:
        a, b = got[k], want[k]
        assert np.array_equal(a == 0, b == 0), f"{k}: zero pattern differs"
        if TOL[k] == 0.0:
            assert np.array_equal(a, b), f"{k}: not bit-identical ({np.sum(a != b)} cells differ)"
        else:
            np.testing.assert_allclose(a, b, rtol=TOL[k], atol=0, err_msg=k)


def test_golden_cases_cover_the_edge_shells():
    g = load("macroatom")[3]["velocity_gradient"]
    typical = np.median(np.abs(g))
    assert g[mko.DECELERATING] < 0
    assert 1e-7 < abs(g[mko.NEAR_FLAT]) / typical < 1e-5
    model = mko.case_inputs("macroatom")[0]
    s = mko.HOMOLOGOUS
    assert g[s] == (model.v_outer[s] - model.v_inner[s]) / (model.r_outer[s] - model.r_inner[s])
    assert np.isclose(g[s], 1 / model.time_explosion, rtol=1e-12)
    assert (load("macroatom")[3]["tau_sobolev"][:, mko.DECELERATING] < 0).any()
    assert (load("downbranch")[3]["velocity_gradient"] < 0).any()
    assert (load("flat_shell")[3]["velocity_gradient"] == 0).any()


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_golden(name):
    from oracle import opacity_oracle_nonhomologous as oon

    model, atomic, plasma, g = load(name)
    check(oon.build(atomic, plasma, g["velocity_gradient"], nlte=True), g)


def test_oracle_raises_the_reference_error_on_a_flat_shell():
    from oracle import opacity_oracle_nonhomologous as oon

    model, atomic, plasma, g = load("flat_shell")
    with pytest.raises(ValueError) as e:
        oon.build(atomic, plasma, g["velocity_gradient"], nlte=True)
    assert str(e.value) == str(g["error"])


def _shim_dir() -> str:
    """tests/_shim, where the other shims of the suite go; a fresh temporary directory where the tree is read-only."""
    d = os.path.join(HERE, "_shim")
    try:
        os.makedirs(d, exist_ok=True)
        if os.access(d, os.W_OK):
            return d
    except OSError:
        pass
    d = tempfile.mkdtemp(prefix="tb200_shim_")
    atexit.register(shutil.rmtree, d, True)
    return d


@pytest.fixture(scope="module")
def shim():
    src = os.path.join(HERE, "nonhomologous_opacity_shim.cpp")
    hdr = os.path.join(ROOT, "tardis_b200", "csrc", "opacity_build.cuh")
    out = os.path.join(_shim_dir(), "libnonhomologous_opacity_shim.so")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", out, src], check=True)
    lib = C.CDLL(out)
    lib.shim_opacity_build_nonhomologous.restype = None
    lib.shim_opacity_build_nonhomologous.argtypes = [C.c_int] * 4 + [C.c_void_p] * 23

    def run(atomic, plasma, velocity_gradient):
        from oracle import opacity_oracle as oo

        L, S, T = len(atomic.nu), plasma.level_number_density.shape[1], len(atomic.transition_type)
        out = {k: np.empty((L, S)) for k in ("stimulated_emission_factor", "tau_sobolev", "beta_sobolev")}
        out["raw_probabilities"], out["transition_probabilities"] = np.empty((T, S)), np.empty((T, S))
        k = np.array([oo.SOBOLEV_COEFFICIENT, oo.C_EINSTEIN, oo.C, oo.H])
        arrs = [np.ascontiguousarray(a) for a in (
            atomic.lower_level, atomic.upper_level, atomic.g, atomic.metastable.astype(np.uint8), atomic.nlte_line.astype(np.uint8),
            atomic.wavelength_cm * atomic.f_lu, atomic.f_lu, atomic.f_ul, atomic.energy[atomic.lower_level], atomic.energy[atomic.upper_level],
            atomic.nu, atomic.transition_type, atomic.transition_line_idx, atomic.macro_block_edge_index, plasma.level_number_density,
            plasma.j_blues, np.asarray(velocity_gradient, dtype=np.float64), k)]
        with np.errstate(all="ignore"):
            lib.shim_opacity_build_nonhomologous(L, S, T, len(atomic.macro_block_edge_index) - 1, *(a.ctypes.data for a in arrs),
                                                 *(out[n].ctypes.data for n in ("stimulated_emission_factor", "tau_sobolev", "beta_sobolev",
                                                                                "raw_probabilities", "transition_probabilities")))
        return out

    return run


@pytest.mark.parametrize("name", CASES)
def test_product_functions_match_reference_golden(shim, name):
    from oracle import opacity_oracle_nonhomologous as oon

    model, atomic, plasma, g = load(name)
    got = shim(atomic, plasma, g["velocity_gradient"])
    check(got, g)
    check(got, oon.build(atomic, plasma, g["velocity_gradient"], nlte=True), keys=("stimulated_emission_factor", "raw_probabilities"))


def test_product_functions_give_no_finite_tau_in_a_flat_shell(shim):
    model, atomic, plasma, g = load("flat_shell")
    tau = shim(atomic, plasma, g["velocity_gradient"])["tau_sobolev"]
    flat = g["velocity_gradient"] == 0
    assert not np.isfinite(tau[:, flat]).any()
    assert np.isfinite(tau[:, ~flat]).all()


# ---- on the device ---------------------------------------------------------------------------------------------------------------
def set_nonhomologous_model(eng, model, atomic, mode, tau=None, tp=None, **config):
    """set_model in the nonhomologous mode with the atomic data's macro-atom structure; tau / tp None: built on the device."""
    eng.set_model(r_inner=model.r_inner, r_outer=model.r_outer, time_explosion=0.0, electron_density=model.electron_density,
                  line_list_nu=model.line_list_nu, tau_sobolev=tau, line_interaction_type=mode, transition_probabilities=tp,
                  line2macro_level_upper=atomic.line2macro_level_upper, macro_block_edge_index=atomic.macro_block_edge_index,
                  transition_type=atomic.transition_type, destination_level_id=atomic.destination_level_id,
                  transition_line_id=atomic.transition_line_idx, spectrum_frequency_grid=model.spectrum_frequency_grid,
                  nonhomologous=True, v_inner=model.v_inner, v_outer=model.v_outer, **config)


def set_atomic(eng, atomic):
    eng.set_atomic_data(lines_lower_level_index=atomic.lower_level, lines_upper_level_index=atomic.upper_level, g=atomic.g,
                        metastability=atomic.metastable, wavelength_cm=atomic.wavelength_cm, f_lu=atomic.f_lu, f_ul=atomic.f_ul,
                        energy_lower=atomic.energy[atomic.lower_level], energy_upper=atomic.energy[atomic.upper_level],
                        nlte_line=atomic.nlte_line)


def device_tables(eng, model, atomic, plasma, mode, velocity_gradient):
    eng.set_option("keep_opacity_tables", 1)
    set_nonhomologous_model(eng, model, atomic, mode)
    set_atomic(eng, atomic)
    eng.build_opacity(plasma.level_number_density, 0.0, plasma.j_blues, velocity_gradient=velocity_gradient)
    return eng.download_opacity(transition_probabilities=True)


@pytest.fixture(scope="module")
def engine():
    from tardis_b200.engine import Engine

    eng = Engine(0)
    yield eng
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_engine_builds_the_reference_tables(engine, name):
    model, atomic, plasma, g = load(name)
    from oracle import opacity_oracle_nonhomologous as oon

    got = device_tables(engine, model, atomic, plasma, mko.CASES[name][4], g["velocity_gradient"])
    check(got, g)
    check(got, oon.build(atomic, plasma, g["velocity_gradient"], nlte=True), keys=("stimulated_emission_factor",))


@pytest.mark.gpu
def test_decelerating_and_near_flat_shells_cell_by_cell(engine):
    model, atomic, plasma, g = load("macroatom")
    got = device_tables(engine, model, atomic, plasma, "macroatom", g["velocity_gradient"])
    for s in (mko.DECELERATING, mko.NEAR_FLAT, mko.HOMOLOGOUS):
        for k in ("tau_sobolev", "beta_sobolev"):
            a, b = got[k][:, s], g[k][:, s]
            bad = ~((a == b) | (np.abs(a - b) <= TOL[k] * np.abs(b)))
            assert not bad.any(), f"shell {s} {k}: lines {np.flatnonzero(bad)[:10]}"
    s = mko.DECELERATING
    neg = got["tau_sobolev"][:, s] < 0
    assert neg.sum() > 100  # tau < 0 takes beta's series branch: beta = 1 - tau / 2 > 1, as in the reference
    assert (got["beta_sobolev"][neg, s] > 1).all()
    s = mko.NEAR_FLAT
    big = got["tau_sobolev"][:, s] > 1e3  # |dv/dr| 1e-6 of the others: beta = tau ** -1 in most cells
    assert big.sum() > 0.8 * len(big)
    assert np.array_equal(got["beta_sobolev"][big, s], 1.0 / got["tau_sobolev"][big, s])


@pytest.mark.gpu
def test_flat_shell_raises_the_reference_error(engine):
    from tardis_b200.engine import EngineError

    model, atomic, plasma, g = load("flat_shell")
    with pytest.raises(EngineError) as e:
        device_tables(engine, model, atomic, plasma, "macroatom", g["velocity_gradient"])
    assert str(g["error"]) in str(e.value)


@pytest.mark.gpu
def test_refusals(engine):
    from tardis_b200.engine import EngineError

    model, atomic, plasma, g = load("downbranch")
    set_nonhomologous_model(engine, model, atomic, "downbranch")
    set_atomic(engine, atomic)
    with pytest.raises(EngineError, match="pass velocity_gradient"):
        engine.build_opacity(plasma.level_number_density, 1.0e6, plasma.j_blues)
    with pytest.raises(ValueError, match="one entry per shell"):
        engine.build_opacity(plasma.level_number_density, 0.0, plasma.j_blues, velocity_gradient=g["velocity_gradient"][:-1])
    # a homologous model refuses the gradient (and builds as before without it)
    engine.set_model(r_inner=model.r_inner, r_outer=model.r_outer, time_explosion=model.time_explosion,
                     electron_density=model.electron_density, line_list_nu=model.line_list_nu, tau_sobolev=None,
                     line_interaction_type="downbranch", line2macro_level_upper=atomic.line2macro_level_upper,
                     macro_block_edge_index=atomic.macro_block_edge_index, transition_type=atomic.transition_type,
                     destination_level_id=atomic.destination_level_id, transition_line_id=atomic.transition_line_idx,
                     spectrum_frequency_grid=model.spectrum_frequency_grid)
    set_atomic(engine, atomic)
    with pytest.raises(EngineError, match="this model is homologous"):
        engine.build_opacity(plasma.level_number_density, model.time_explosion, plasma.j_blues, velocity_gradient=g["velocity_gradient"])
    engine.build_opacity(plasma.level_number_density, model.time_explosion, plasma.j_blues)


@pytest.mark.gpu
def test_engine_group_builds_the_tables_of_one_engine(engine):
    from tardis_b200.engine import EngineGroup

    model, atomic, plasma, g = load("macroatom")
    one = device_tables(engine, model, atomic, plasma, "macroatom", g["velocity_gradient"])
    group = EngineGroup([0, 0])
    try:
        device_tables(group, model, atomic, plasma, "macroatom", g["velocity_gradient"])
        for m in group.members:
            got = m.download_opacity(transition_probabilities=True)
            for k in DEVICE_KEYS:
                assert np.array_equal(got[k], one[k]), k
    finally:
        group.close()


@pytest.mark.gpu
def test_bench_shape_every_cell(engine):
    """5e5 lines, 20 shells, 3000 levels (1.5e6 macro-atom rows), interior velocities +-8 %: every tau and beta cell."""
    from oracle import opacity_oracle as oo
    from oracle import opacity_oracle_nonhomologous as oon
    from tardis_b200 import synthetic as syn

    model = syn.make_nonhomologous_velocities(syn.make_model(20, 500_000, "macroatom"), 0.08)
    atomic = syn.make_atomic_data(model.line_list_nu, 3000, "macroatom", seed=91)
    plasma = syn.make_plasma_state(atomic, 20, 0.0, seed=92)
    grad = (model.v_outer - model.v_inner) / (model.r_outer - model.r_inner)
    assert (grad < 0).any()
    assert len(atomic.transition_type) == 1_500_000
    got = device_tables(engine, model, atomic, plasma, "macroatom", grad)
    stim = oo.stimulated_emission_factor(atomic, plasma.level_number_density, nlte=True)
    tau = oon.tau_sobolev(atomic, plasma.level_number_density, grad, stim)
    assert np.array_equal(got["stimulated_emission_factor"], stim)
    assert np.array_equal(got["tau_sobolev"], tau)
    check(got, dict(beta_sobolev=oo.beta_sobolev(tau)), keys=("beta_sobolev",))


# ---- two iterations that stay on the device, against the same chain on host-built tables -----------------------------------------
INT_KEYS = ("last_interaction_type", "last_shell_id", "last_line_absorb_id", "last_line_emit_id")
FLOAT_KEYS = ("output_nus", "output_energies", "last_radius", "last_before_nu", "last_before_mu", "last_before_energy",
              "last_after_nu", "last_after_mu", "last_after_energy")
COUNTERS = ("n_line_steps", "n_boundary_events", "n_line_events", "n_escat_events", "n_rng_draws", "n_macro_jumps",
            "n_macro_scanned", "n_vpackets", "n_vpacket_line_steps")
RTOL = 1e-10  # the bar of tests/test_nonhomologous_gpu.py for the estimator sums


def chain_inputs(mode):
    from tardis_b200 import synthetic as syn

    model = syn.make_nonhomologous_velocities(syn.make_model(8, 4000, mode, mu_tau=-4.0, seed=61), 0.08)
    atomic = syn.make_atomic_data(model.line_list_nu, 300, mode, seed=62, nlte_fraction=0.0)
    plasmas = []
    for it in range(2):
        p = syn.make_plasma_state(atomic, 8, 0.0, seed=63 + it, zero_fraction=0.0, inversion_fraction=0.0, noise=0.0)
        p.level_number_density *= 1e-9  # optical depths of order one
        plasmas.append(p)
    grad = (model.v_outer - model.v_inner) / (model.r_outer - model.r_inner)
    packets = [syn.make_packets(20000, model.r_inner[0], base_seed=12, iteration=it) for it in range(2)]
    volume = (4 / 3) * np.pi * (model.r_outer**3 - model.r_inner**3)
    return model, atomic, plasmas, grad, packets, volume


@pytest.mark.gpu
@pytest.mark.parametrize("mode,config", [("macroatom", dict(number_of_vpackets=2)), ("downbranch", {})],
                         ids=["macroatom_vpackets", "downbranch"])
def test_two_iterations_on_the_device_equal_the_host_tables_chain(mode, config):
    from oracle import opacity_oracle_nonhomologous as oon
    from tardis_b200.engine import Engine

    model, atomic, plasmas, grad, packets, volume = chain_inputs(mode)
    assert (grad < 0).any()
    dev, host = Engine(0), Engine(0)
    try:
        set_nonhomologous_model(dev, model, atomic, mode, **config)
        set_atomic(dev, atomic)
        j_blues = plasmas[0].j_blues
        for it in range(2):
            radfield = dict(time_explosion=0.0, time_of_simulation=packets[it].time_of_simulation, volume=volume, velocity_gradient=grad)
            # the device chain: J_blue stays in HBM between the radiation field and the opacity build
            dev.build_opacity(plasmas[it].level_number_density, 0.0, plasmas[0].j_blues if it == 0 else None, velocity_gradient=grad)
            got = dev.run_packets(packets[it], track_last_interaction=True)
            dev.solve_radiation_field(want_j_blues=False, **radfield)
            # the host chain: the oracle's tables, uploaded
            plasma = dataclass_with_j_blues(plasmas[it], j_blues)
            ref_tables = oon.build(atomic, plasma, grad)
            if it == 0:
                assert (ref_tables["tau_sobolev"] < 0).any()
            set_nonhomologous_model(host, model, atomic, mode, tau=ref_tables["tau_sobolev"], tp=ref_tables["transition_probabilities"],
                                    **config)
            ref = host.run_packets(packets[it], track_last_interaction=True)
            j_blues = host.solve_radiation_field(**radfield)[2]
            for k in INT_KEYS:
                assert np.array_equal(got[k], ref[k]), f"iteration {it}: {k}"
            for k in FLOAT_KEYS:
                assert np.array_equal(got[k], ref[k], equal_nan=True), f"iteration {it}: {k}"
            for k in COUNTERS:
                assert got["counters"][k] == ref["counters"][k], f"iteration {it}: {k}"
            for k in ("j", "nu_bar", "j_blue", "edotlu", "vhist"):
                np.testing.assert_allclose(got[k], ref[k], rtol=RTOL, atol=1e-300, err_msg=f"iteration {it}: {k}")
    finally:
        dev.close()
        host.close()


def dataclass_with_j_blues(plasma, j_blues):
    import dataclasses

    return dataclasses.replace(plasma, j_blues=j_blues)
