"""The continuum (IIP) macro atom's per-iteration rows built on the device (tardis_b200/csrc/continuum_macro_build.cuh,
tb200_build_opacity in the continuum mode) and handed to tb200_build_absorbing_markov in HBM.

CPU: the oracle (oracle/continuum_macro_oracle.py) and the header, built for the host by tests/continuum_macro_build_shim.cpp,
against golden vectors of the unmodified reference ContinuumMacroAtomSolver (tests/golden/make_continuum_macro_golden.py);
the row map against the reference's own lookups where the reference tree exists.
GPU: the device tables against the goldens; the resident chain (build_opacity -> build_absorbing_markov(None) -> transport)
against the same chain fed the oracle's host tables, two iterations; an engine group [0, 0]; refusals.
Bars: continuum rows and every block without line rows bit-identical; blocks with line rows within test_opacity_build.py's
1e-11 (the device's exp in beta_Sobolev); zero patterns identical; X within 1e-13 (test_markov_build.py)."""
import ctypes as C
import hashlib
import importlib.util
import os
import subprocess
import tempfile

import numpy as np
import pytest

from golden_util import GOLDEN_DIR, assert_close

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
_spec = importlib.util.spec_from_file_location("make_continuum_macro_golden", os.path.join(GOLDEN_DIR, "make_continuum_macro_golden.py"))
gen = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(gen)
CASES = list(gen.CASES)
FULL = [n for n in CASES if gen.CASES[n][1] == "full"]
LINE_BAR = 1e-11
X_BAR = 1e-13
LINE_TYPES = (-1, 0, 1)


def golden(name):
    return gen.inputs(name), dict(np.load(os.path.join(GOLDEN_DIR, name + ".npz")))


def row_map(g):
    return dict(rate_key=g["rate_key"], energy=g["energy"], n_rate_rows=list(g["n_rate_rows"]), n_cooling_rows=list(g["n_cooling_rows"]))


def line_tables(ci, it):
    from oracle import opacity_oracle as oo

    p = ci.plasma[it]
    stim = oo.stimulated_emission_factor(ci.atomic, p.level_number_density)
    tau = oo.tau_sobolev(ci.atomic, p.level_number_density, p.time_explosion, stim)
    return tau, oo.beta_sobolev(tau), stim, p.j_blues


def oracle_tables(ci, g, it=-1):
    from oracle import continuum_macro_oracle as cmo
    from tardis_b200 import macro_atom

    tau, beta, stim, jb = line_tables(ci, it)
    raw = cmo.raw_rows(ci.atomic, g["transition_type"], g["transition_line_idx"], row_map(g), macro_atom.continuum_rates(ci.rates[it]),
                       beta, stim, jb)
    return tau, raw, cmo.normalize(raw, g["macro_block_edge_index"])


def line_blocks(g):
    """[T] bool: the row lies in a block that holds a line row"""
    e, tt = g["macro_block_edge_index"], g["transition_type"]
    block = np.repeat(np.arange(len(e) - 1), np.diff(e))
    has = np.zeros(len(e) - 1, dtype=bool)
    has[block[np.isin(tt, LINE_TYPES)]] = True
    return has[block]


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def check_table(name, got, g, key):
    """got [T, S] against the golden table `key`: bit-identical outside blocks with line rows, 1e-11 inside, same zeros"""
    lb = line_blocks(g)
    if key in g:
        want = g[key]
        assert np.array_equal(bits(got[~lb]), bits(want[~lb])), f"{name} {key}: blocks without line rows differ"
        np.testing.assert_allclose(got[lb], want[lb], rtol=LINE_BAR, atol=0, err_msg=f"{name} {key}: blocks with line rows")
        assert np.array_equal(got == 0, want == 0), f"{name} {key}: zero pattern"
    else:
        idx, want = g[key + "_sample_idx"], g[key + "_sample_val"]
        cell_lb = np.repeat(lb, got.shape[1])[idx]
        flat = got.ravel()[idx]
        assert np.array_equal(bits(flat[~cell_lb]), bits(want[~cell_lb])), f"{name} {key}: sampled cells without line rows differ"
        np.testing.assert_allclose(flat[cell_lb], want[cell_lb], rtol=LINE_BAR, atol=0)
        assert np.array_equal(flat == 0, want == 0)


def check_raw_continuum(name, raw, g):
    cont = ~np.isin(g["transition_type"], LINE_TYPES)
    if "raw" in g:
        assert np.array_equal(bits(raw[cont]), bits(g["raw"][cont])), f"{name}: continuum rows not bit-identical"
    else:
        assert hashlib.sha256(np.ascontiguousarray(raw[cont]).tobytes()).hexdigest() == str(g["raw_continuum_sha256"])


def check_x(X, g):
    if "X" in g:
        assert np.array_equal(X == 0, g["X"] == 0), "zero pattern of X"
        assert np.abs(X - g["X"]).max() <= X_BAR
    else:
        flat = X.ravel()[g["X_sample_idx"]]
        assert np.array_equal(flat == 0, g["X_sample_val"] == 0), "zero pattern of X (sampled cells)"
        assert np.abs(flat - g["X_sample_val"]).max() <= X_BAR
    assert np.abs(X.sum(axis=2) - g["row_sums"]).max() <= X_BAR


# ---- CPU -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_golden(name):
    ci, g = golden(name)
    _, raw, norm = oracle_tables(ci, g)
    check_raw_continuum(name, raw, g)
    if "raw" in g:  # the line rows too: the reference was given the oracle's beta
        assert np.array_equal(bits(raw), bits(g["raw"]))
        assert np.array_equal(bits(norm), bits(g["normalized"]))
    else:
        assert np.array_equal(bits(norm.ravel()[g["normalized_sample_idx"]]), bits(g["normalized_sample_val"]))


@pytest.fixture(scope="module")
def shim():
    src = os.path.join(HERE, "continuum_macro_build_shim.cpp")
    hdrs = [os.path.join(ROOT, "tardis_b200", "csrc", h) for h in ("continuum_macro_build.cuh", "markov_build.cuh")]
    out_dir = os.path.join(HERE, "_shim")
    try:
        os.makedirs(out_dir, exist_ok=True)
        if not os.access(out_dir, os.W_OK):
            raise OSError
    except OSError:  # read-only tree
        out_dir = tempfile.mkdtemp()
    out = os.path.join(out_dir, "libcontinuum_macro_build_shim.so")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(f) for f in [src, *hdrs]):
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", out, src], check=True)
    lib = C.CDLL(out)
    lib.shim_continuum_rows.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 7
    lib.shim_normalize.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    return lib


def shim_tables(lib, ci, g, raw_lines):
    """raw and normalised [T, S] from the header: continuum rows computed, line rows taken from `raw_lines`"""
    from tardis_b200 import macro_atom

    rates = macro_atom.continuum_rates(ci.rates[-1])
    tabs = [*rates["rate"], *rates["cooling"]]
    S = tabs[0].shape[1]
    tab = np.ascontiguousarray(np.concatenate([np.ascontiguousarray(t).reshape(-1, S) for t in tabs]))
    base = np.concatenate([[0], np.cumsum([t.shape[0] for t in tabs])]).astype(np.int64)
    shell = np.ascontiguousarray(np.stack([rates[k] for k in ("electron_densities", "ff_cool_rate", "fb_cool_rate", "coll_exc_cool_rate",
                                                                 "coll_ion_cool_rate")]))
    tt, key, en = (np.ascontiguousarray(g[k]) for k in ("transition_type", "rate_key", "energy"))
    T = len(tt)
    p = np.where(np.isin(tt, LINE_TYPES)[:, None], raw_lines, 0.0).copy()
    lib.shim_continuum_rows(T, S, tt.ctypes.data, key.ctypes.data, en.ctypes.data, base.ctypes.data, tab.ctypes.data, shell.ctypes.data,
                            p.ctypes.data)
    raw = p.copy()
    edges = np.ascontiguousarray(g["macro_block_edge_index"], dtype=np.int64)
    lib.shim_normalize(T, S, len(edges) - 1, edges.ctypes.data, p.ctypes.data)
    return raw, p


@pytest.mark.parametrize("name", CASES)
def test_header_matches_reference_golden(shim, name):
    ci, g = golden(name)
    _, oracle_raw, _ = oracle_tables(ci, g)
    raw, norm = shim_tables(shim, ci, g, oracle_raw)
    check_raw_continuum(name, raw, g)
    check_table(name, norm, g, "normalized")


def test_kahan_sum_and_nan_skip_are_the_references():
    """pandas' group sum: 1 + 1e-16 + 1e-16 ... is compensated, and a NaN addend (inf rate x zero energy) is skipped"""
    import pandas as pd

    from oracle import continuum_macro_oracle as cmo

    p = np.array([[1.0], [1e-16], [1e-16], [1e-16], [np.nan], [3.0], [np.inf], [np.nan], [2.0]])
    edges = np.array([0, 5, 9])
    want = (pd.DataFrame(p).div(pd.DataFrame(p).groupby(np.repeat([0, 1], [5, 4])).transform("sum"))).fillna(0.0).to_numpy()
    assert np.array_equal(bits(cmo.normalize(p, edges)), bits(want))


@pytest.mark.skipif(not os.path.isdir(os.environ.get("TARDIS_REFERENCE", "/root/reference")), reason="needs the reference tree")
@pytest.mark.parametrize("name", FULL)
def test_row_map_reproduces_the_reference_rows(name):
    """The map derived from the reference's solver, applied to the rates, gives the reference's raw continuum rows"""
    from oracle import reference_runner_continuum_macro as rr
    from tardis_b200 import macro_atom

    ci, g = golden(name)
    ref = rr.run(ci)
    rmap = macro_atom.continuum_row_map(ref["solver"], ref["metadata"], ci.rates[-1])
    assert np.array_equal(rmap["rate_key"], g["rate_key"]) and np.array_equal(bits(rmap["energy"]), bits(g["energy"]))
    check_raw_continuum(name, oracle_tables(ci, dict(g, **rmap))[1], dict(g, raw=ref["raw"]))


# ---- GPU -------------------------------------------------------------------------------------------------------------
def model_for(ci, g, tau=None):
    from tardis_b200 import synthetic as syn

    S = ci.plasma[0].level_number_density.shape[1]
    model = syn.add_continuum(syn.make_model(S, 200, "macroatom", seed=5), seed=6)
    model.line_list_nu = ci.atomic.nu.copy()
    model.tau_sobolev = tau
    tt, src = g["transition_type"], g["source_level_idx"]
    dst = np.where(tt >= 0, g["destination_level_idx"], -1)
    model.macro = syn.MacroAtomTables(None, g["line2macro_level_upper"], g["macro_block_edge_index"], tt, dst, g["transition_line_idx"])
    model.continuum.k_packet_idx = int(src[tt == -21][0])
    model.continuum.photo_ion_activation_idx = np.full(30, int(src[tt == -7][0]), dtype=np.int64)
    model.continuum.absorbing_markov_probabilities = None
    return model


def markov_args(g):
    tt = g["transition_type"]
    return dict(source_level_idx=g["source_level_idx"], destination_level_idx=np.where(tt >= 0, g["destination_level_idx"], -1),
                transition_type=tt)


def engine_for(ci, g, group=None, atomic=True):
    from tardis_b200.engine import Engine, EngineGroup

    eng = EngineGroup(group) if group is not None else Engine(0)
    eng.set_option("keep_opacity_tables", 1)
    eng.set_model_from(model_for(ci, g), enable_full_relativity=True)
    if atomic:
        set_atomic(eng, ci, row_map(g))
    return eng


def set_atomic(eng, ci, rows):
    a = ci.atomic
    eng.set_atomic_data(lines_lower_level_index=a.lower_level, lines_upper_level_index=a.upper_level, g=a.g, metastability=a.metastable,
                        wavelength_cm=a.wavelength_cm, f_lu=a.f_lu, f_ul=a.f_ul, energy_lower=a.energy[a.lower_level],
                        energy_upper=a.energy[a.upper_level], continuum_rows=rows)


def build(eng, ci, g, it=-1):
    from tardis_b200 import macro_atom

    p = ci.plasma[it]
    eng.build_opacity(p.level_number_density, p.time_explosion, j_blues=p.j_blues, continuum=macro_atom.continuum_rates(ci.rates[it]))
    norm = eng.download_opacity(transition_probabilities=True)["transition_probabilities"]
    eng.build_absorbing_markov(None, **markov_args(g))
    return norm, eng.download_absorbing_markov()


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_device_build_matches_reference_golden(name):
    from tardis_b200.engine import EngineError
    from tardis_b200 import synthetic as syn

    ci, g = golden(name)
    eng = engine_for(ci, g)
    p = ci.plasma[-1]
    from tardis_b200 import macro_atom
    eng.build_opacity(p.level_number_density, p.time_explosion, j_blues=p.j_blues, continuum=macro_atom.continuum_rates(ci.rates[-1]))
    pk = syn.make_packets(4, 1e15)
    eng.upload_packets(pk.initial_radii * 0 + eng_r0(ci, g), pk.initial_nus, pk.initial_mus, pk.initial_energies, pk.packet_seeds)
    with pytest.raises(EngineError, match="tb200_build_absorbing_markov"):  # the chain is pending until its build
        eng.transport(True)
    norm = eng.download_opacity(transition_probabilities=True)["transition_probabilities"]
    check_table(name, norm, g, "normalized")
    eng.build_absorbing_markov(None, **markov_args(g))
    got = eng.download_absorbing_markov()
    check_x(got["absorbing_markov_probabilities"], g)
    check_table(name, got["transition_probabilities"], g, "deactivation")
    eng.close()


def eng_r0(ci, g):
    return model_for(ci, g).r_inner[0]


@pytest.mark.gpu
def test_resident_chain_equals_the_chain_on_host_tables():
    """Two continuum iterations: build_opacity -> build_absorbing_markov(None) -> transport on the device, against set_model
    with the oracle's tau and build_absorbing_markov with the oracle's normalised table."""
    from tardis_b200 import synthetic as syn

    name = "continuum_macro_small"
    ci, g = golden(name)
    dev = engine_for(ci, g)
    host = engine_for(ci, g, atomic=False)
    packets = syn.make_packets(20000, eng_r0(ci, g), base_seed=95)
    n_events = 0
    for it in range(2):
        build(dev, ci, g, it)
        a = dev.run_packets(packets, track_last_interaction=True)
        tau, _, norm = oracle_tables(ci, g, it)
        host.set_model_from(model_for(ci, g, tau=tau), enable_full_relativity=True)
        host.build_absorbing_markov(norm, **markov_args(g))
        b = host.run_packets(packets, track_last_interaction=True)
        assert a["counters"] == b["counters"]
        n_events += a["counters"]["n_continuum_events"] + a["counters"]["n_macro_jumps"]
        for k in ("output_nus", "output_energies", "j_blue", "edotlu", "photo_ion_estimator_statistics", "last_interaction_type",
                  "last_shell_id", "last_line_absorb_id", "last_line_emit_id", "last_after_nu", "last_after_energy"):
            x, y = np.asarray(a[k]), np.asarray(b[k])
            assert np.array_equal(x.view(np.uint64) if x.dtype == np.float64 else x, y.view(np.uint64) if y.dtype == np.float64 else y), (it, k)
        for k in ("j", "nu_bar", "photo_ion_estimator", "stim_recomb_estimator", "bf_heating_estimator", "stim_recomb_cooling_estimator",
                  "ff_heating_estimator"):
            assert_close(a[k], b[k], 1e-13, k)
    assert n_events > 0
    dev.close()
    host.close()


@pytest.mark.gpu
def test_group_members_equal_one_engine():
    ci, g = golden("continuum_macro_adversarial")
    one = engine_for(ci, g)
    want_norm, want = build(one, ci, g)
    grp = engine_for(ci, g, group=[0, 0])
    build(grp, ci, g)
    for m in grp.members:
        assert np.array_equal(bits(m.download_opacity(transition_probabilities=True)["transition_probabilities"]), bits(want_norm))
        got = m.download_absorbing_markov()
        for k in want:
            assert np.array_equal(bits(got[k]), bits(want[k])), k
    one.close()
    grp.close()


@pytest.mark.gpu
def test_refusals_leave_the_engine_usable():
    from tardis_b200 import macro_atom
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import Engine, EngineError

    ci, g = golden("continuum_macro_small")
    eng = engine_for(ci, g, atomic=False)
    rows = row_map(g)
    with pytest.raises(EngineError, match="needs continuum_rows"):
        set_atomic(eng, ci, None)
    bad = dict(rows, rate_key=rows["rate_key"].copy())
    bad["rate_key"][np.flatnonzero(g["transition_type"] == 4)[0]] = rows["n_rate_rows"][3]
    with pytest.raises(EngineError, match="outside its table"):
        set_atomic(eng, ci, bad)
    with pytest.raises(EngineError, match="n_transitions"):
        set_atomic(eng, ci, dict(rows, rate_key=rows["rate_key"][:-1], energy=rows["energy"][:-1]))
    with pytest.raises(EngineError, match="has built no table"):
        eng.build_absorbing_markov(None, **markov_args(g))
    set_atomic(eng, ci, rows)
    p = ci.plasma[-1]
    with pytest.raises(EngineError, match="needs continuum"):
        eng.build_opacity(p.level_number_density, p.time_explosion, j_blues=p.j_blues)
    want_norm, want = build(eng, ci, g)
    check_table("continuum_macro_small", want_norm, g, "normalized")
    eng.close()

    plain = Engine(0)  # a model without continuum refuses both
    atomic = syn.make_atomic_data(syn.make_model(3, 300, "macroatom", seed=3).line_list_nu, 40)
    model = syn.make_model(3, 300, "macroatom", seed=3)
    model.tau_sobolev = None
    plain.set_model_from(model)
    with pytest.raises(EngineError, match="no continuum"):
        plain.set_atomic_data(lines_lower_level_index=atomic.lower_level, lines_upper_level_index=atomic.upper_level, g=atomic.g,
                              metastability=atomic.metastable, wavelength_cm=atomic.wavelength_cm, f_lu=atomic.f_lu, f_ul=atomic.f_ul,
                              energy_lower=atomic.energy[atomic.lower_level], energy_upper=atomic.energy[atomic.upper_level],
                              continuum_rows=rows)
    plain.close()


def reference_like_solver(ci, g):
    """What the reference's first iteration leaves on a ContinuumMacroAtomSolver, as far as the drop-in reads it: the
    metadata (from the golden) and the static line arrays (_precompute_static_data, macroatom_solver.py:238-274).  The
    row map is the one the golden holds (derived from the reference's own solver), cached as the drop-in caches it."""
    from types import SimpleNamespace

    import pandas as pd

    md = pd.DataFrame({k: g[k] for k in ("transition_type", "source_level_idx", "destination_level_idx", "transition_line_idx")})
    a = ci.atomic
    solver = SimpleNamespace(computed_metadata=(md, g["line2macro_level_upper"], g["macro_block_edge_index"], None),
                             _nus=ci.lines.nu.to_numpy().reshape(-1, 1), _oscillator_strength_lu=ci.lines.f_lu.to_numpy().reshape(-1, 1),
                             _oscillator_strength_ul=ci.lines.f_ul.to_numpy().reshape(-1, 1),
                             _energies_lower=a.energy[a.lower_level].reshape(-1, 1), _energies_upper=a.energy[a.upper_level].reshape(-1, 1))
    solver._b200_row_map = (md, row_map(g))
    return solver


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_drop_in_returns_what_the_golden_holds(name):
    """solve_next_macroatom_iteration with the reference's arguments (the beta / stim the reference was given) returns the
    reference's normalised probabilities and deactivation table bit for bit, X within 1e-13, and `montecarlo_transport`
    recognises the returned X."""
    import pandas as pd

    from tardis_b200 import macro_atom
    from tardis_b200.engine import Engine

    ci, g = golden(name)
    solver = reference_like_solver(ci, g)
    _, beta, stim, jb = line_tables(ci, -1)
    eng = Engine(0)
    args = {k: v for k, v in ci.rates[-1].items() if k != "delta_E_yg"}  # solve's, less what the first iteration kept
    norm, deact, X = macro_atom.solve_next_macroatom_iteration(solver, pd.DataFrame(jb), pd.DataFrame(beta), stim, **args, engine=eng)
    md = solver.computed_metadata[0]
    assert norm.index.equals(md.index) and norm.columns.equals(pd.RangeIndex(beta.shape[1])) and deact.shape == norm.shape
    for key, got in (("normalized", norm.to_numpy()), ("deactivation", deact.to_numpy())):
        if key in g:
            assert np.array_equal(bits(got), bits(g[key])), key
        else:
            assert np.array_equal(bits(got.ravel()[g[key + "_sample_idx"]]), bits(g[key + "_sample_val"])), key
    check_x(X, g)
    assert macro_atom.built_inputs(X, g["transition_type"]) is not None
    eng.close()


@pytest.mark.gpu
def test_row_map_belongs_to_its_model():
    """tb200_set_model discards the row map: a model with the same rows and fewer shells is refused until the map is given
    again, and then builds the same normalised rows as a fresh engine"""
    from tardis_b200 import macro_atom
    from tardis_b200.engine import EngineError

    ci, g = golden("continuum_macro_small")
    eng = engine_for(ci, g)
    build(eng, ci, g)
    kw = dict(gen.CASES["continuum_macro_small"][0], n_shells=3)
    ci3 = syn_inputs(kw)
    assert len(ci3.lines) == len(ci.lines)
    eng.set_model_from(model_for(ci3, g), enable_full_relativity=True)
    p = ci3.plasma[-1]
    with pytest.raises(EngineError, match="continuum_rows for this model"):
        eng.build_opacity(p.level_number_density, p.time_explosion, j_blues=p.j_blues, continuum=macro_atom.continuum_rates(ci3.rates[-1]))
    set_atomic(eng, ci3, row_map(g))
    got, _ = build(eng, ci3, g)
    fresh = engine_for(ci3, g)
    want, _ = build(fresh, ci3, g)
    assert np.array_equal(bits(got), bits(want))
    eng.close()
    fresh.close()


def syn_inputs(kw):
    from tardis_b200 import synthetic as syn

    return syn.make_continuum_rate_inputs(**kw)


@pytest.mark.gpu
def test_refusals_at_the_c_interface():
    """A NULL table that the row map reads, continuum rates on a model without continuum, a refused row map that keeps
    the previous one, and download_opacity's transition_probabilities before any continuum build"""
    from tardis_b200 import capi, macro_atom
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import Engine, EngineError

    ci, g = golden("continuum_macro_small")
    eng = engine_for(ci, g)
    host = Engine(0)  # tau from the host, no continuum build yet: download_opacity has no continuum table to return
    host.set_option("keep_opacity_tables", 1)
    host.set_model_from(model_for(ci, g, tau=line_tables(ci, -1)[0]), enable_full_relativity=True)
    tp = np.empty((len(g["transition_type"]), ci.plasma[0].level_number_density.shape[1]))
    assert host._lib.tb200_download_opacity(host._h, None, None, None, tp.ctypes.data_as(C.POINTER(C.c_double))) != 0
    assert "no kept table" in host._lib.tb200_last_error().decode()  # the deactivation table is download_absorbing_markov's
    host.close()
    rates = macro_atom.continuum_rates(ci.rates[-1])
    tabs = [np.ascontiguousarray(t) for t in (*rates["rate"], *rates["cooling"])]
    shell = [np.ascontiguousarray(rates[k]) for k in ("electron_densities", "ff_cool_rate", "fb_cool_rate", "coll_exc_cool_rate",
                                                       "coll_ion_cool_rate")]
    p = ci.plasma[-1]
    lnd, jb = np.ascontiguousarray(p.level_number_density), np.ascontiguousarray(p.j_blues)
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))  # noqa: E731
    for missing in (2, 7):  # coll_deexc_coeff, coll_exc_cool_arr.T
        cr = capi.ContinuumRates()
        for k in range(6):
            cr.rate[k] = dp(tabs[k]) if k != missing else None
        for k in range(3):
            cr.cooling[k] = dp(tabs[6 + k]) if 6 + k != missing else None
        cr.electron_densities, cr.ff_cool_rate, cr.fb_cool_rate, cr.coll_exc_cool_rate, cr.coll_ion_cool_rate = map(dp, shell)
        ps = capi.PlasmaState(level_number_density=dp(lnd), time_explosion=p.time_explosion, j_blues=dp(jb), continuum=C.pointer(cr))
        assert eng._lib.tb200_build_opacity(eng._h, C.byref(ps)) != 0
        assert "is NULL but the row map reads it" in eng._lib.tb200_last_error().decode()
    bad = dict(row_map(g), rate_key=np.full_like(g["rate_key"], 10**6))
    with pytest.raises(EngineError, match="outside its table"):
        set_atomic(eng, ci, bad)
    want_norm, _ = build(eng, ci, g)  # the refused map left the previous one in place
    check_table("continuum_macro_small", want_norm, g, "normalized")
    eng.close()

    plain = Engine(0)
    atomic = syn.make_atomic_data(syn.make_model(3, 300, "macroatom", seed=3).line_list_nu, 40)
    model = syn.make_model(3, 300, "macroatom", seed=3)
    model.tau_sobolev = None
    model.macro.transition_probabilities = None
    plain.set_model_from(model)
    plain.set_atomic_data(lines_lower_level_index=atomic.lower_level, lines_upper_level_index=atomic.upper_level, g=atomic.g,
                          metastability=atomic.metastable, wavelength_cm=atomic.wavelength_cm, f_lu=atomic.f_lu, f_ul=atomic.f_ul,
                          energy_lower=atomic.energy[atomic.lower_level], energy_upper=atomic.energy[atomic.upper_level])
    plasma = syn.make_plasma_state(atomic, 3, model.time_explosion)
    S = 3
    cont = dict(rate=[np.ones((1, S))] * 6, cooling=[np.ones((1, S))] * 3, electron_densities=np.ones(S), ff_cool_rate=np.ones(S),
                fb_cool_rate=np.ones(S), coll_exc_cool_rate=np.ones(S), coll_ion_cool_rate=np.ones(S))
    with pytest.raises(EngineError, match="no continuum"):
        plain.build_opacity(plasma.level_number_density, plasma.time_explosion, j_blues=plasma.j_blues, continuum=cont)
    plain.close()
