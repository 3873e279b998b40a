"""Device-side BlackBodyWeightedSource (packet_source/black_body_weighted.py:9-108; tardis_b200/csrc/packet_source.cuh).

CPU: the weighted restatement (oracle/weighted_source_oracle.py) against golden vectors of the unmodified reference class;
the product's header functions, built for the host by tests/weighted_source_shim.cpp and driven member by member and
chunk by chunk as engine.cu drives them, against the same; numpy's pairwise summation restated (the leaf tree both
follow) against `ndarray.sum()`; the mirror's surface against the reference class.

GPU: the kernels through the C-ABI against the goldens and the oracle; engine groups bit for bit against one engine;
weighted packets through the transport kernels against the C oracle, with J_blue / Edotlu held to the fixed-point bound
(DESIGN.md); the drop-in solver path.

Bars: seeds, radii, mus bit-identical.  nus: NU_ULPS ulps (the extremes come from one ulp of `log`).  Energies:
|d e| <= (E_ULPS * A + NU_ULPS * |3 - x A|) ulp(e), x = h nu / k T, A = e^x / (e^x - 1): A is the condition number of
exp(x) - 1 with respect to an ulp of exp (the far-red packets cancel), |3 - x A| that of I(nu) with respect to nu.
"""
from __future__ import annotations

import ctypes as C
import glob
import json
import os
import subprocess

import numpy as np
import pytest

from oracle import weighted_source_oracle as wso

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(HERE, "golden", "weighted_source_*.npz")))
EXACT = ("packet_seeds", "initial_radii", "initial_mus")
NU_ULPS = 2
E_ULPS = 6
SUM_ULPS = 4  # sum of the normalised energies against 1


def golden(name):
    return np.load(os.path.join(HERE, "golden", name + ".npz"))


def check(got, want, temperature, nu_ulps=NU_ULPS, e_ulps=E_ULPS, what=""):
    """-> (max nu ulps, max energy ulps / allowance) measured"""
    for k in EXACT:
        assert np.array_equal(got[k], want[k]), (what, k)
    nu_w, e_w = want["initial_nus"], want["initial_energies"]
    nu_err = np.abs(got["initial_nus"] - nu_w) / np.spacing(nu_w)
    assert nu_err.max() <= nu_ulps, (what, nu_err.max())
    x = wso.H * nu_w / (wso.K_B * temperature)
    A = np.exp(x) / np.expm1(x)
    allowed = e_ulps * A + nu_ulps * np.abs(3 - x * A)
    e_err = np.abs(got["initial_energies"] - e_w) / np.spacing(e_w)
    assert (e_err <= allowed).all(), (what, (e_err / allowed).max())
    total = got["initial_energies"].sum()
    assert abs(total - 1.0) <= SUM_ULPS * 2.0**-53, (what, total - 1.0)
    return float(nu_err.max()), float((e_err / allowed).max())


@pytest.fixture(scope="module")
def shim():
    out = os.path.join(HERE, "_shim", "libweighted_source_shim.so")
    src = os.path.join(HERE, "weighted_source_shim.cpp")
    hdr = os.path.join(ROOT, "tardis_b200", "csrc", "packet_source.cuh")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", out, src], check=True)
    lib = C.CDLL(out)
    lib.shim_weighted_packets.restype = C.c_int
    lib.shim_weighted_packets.argtypes = ([C.c_uint64, C.c_uint64, C.c_uint32] + [C.c_double] * 5 + [C.c_void_p, C.c_int, C.c_double, C.c_int,
                                          C.c_void_p, C.c_uint64] + [C.c_void_p] * 5 + [C.c_int, C.c_void_p, C.c_void_p])
    lib.shim_pairwise_sum.restype = C.c_double
    lib.shim_pairwise_sum.argtypes = [C.c_void_p, C.c_uint64]
    lib.shim_leaf_at.argtypes = [C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p]

    def run(seed, n, radius=1.2e15, temperature=1.0e4, bounds=None, chunk=256, normalize=True):
        l_array = np.cumsum(np.arange(1, 1000, dtype=np.float64) ** -4)
        b = np.array([0, n] if bounds is None else bounds, dtype=np.int64)
        out = {k: np.full(n, np.nan) for k in ("initial_radii", "initial_nus", "initial_mus", "initial_energies")}
        out["packet_seeds"] = np.full(n, -1, dtype=np.int64)
        total, mm = C.c_double(), (C.c_double * 2)()
        rc = lib.shim_weighted_packets(seed, n, 2**32 - 2, radius, temperature, wso.K_B, wso.H, wso.C, l_array.ctypes.data, len(l_array),
                                       np.pi**4 / 90.0, len(b) - 1, b.ctypes.data, chunk,
                                       *(out[k].ctypes.data for k in ("initial_radii", "initial_nus", "initial_mus", "initial_energies",
                                                                      "packet_seeds")), int(normalize), C.byref(total), mm)
        assert rc == 0
        out["energy_sum"], out["minmax"] = total.value, (mm[0], mm[1])
        return out

    run.lib = lib
    return run


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_golden(name):
    g = golden(name)
    got = wso.create_packets(int(g["n"]), int(g["base_seed"]) + int(g["seed_offset"]), float(g["radius"]), float(g["temperature"]))
    check(got, g, float(g["temperature"]), what=name)
    assert np.array_equal(g["self_nus"], g["initial_nus"])  # the reference leaves its nus on the source


def test_oracle_uses_the_plain_sources_stream(oracle):
    """The seeds and the Carter-Cashwell nus the weighted restatement draws are the C oracle's plain source, bit for bit
    (the extremes of those nus are the weighted source's range)."""
    n, seed, radius, temperature = 20011, 77, 1.2355e15, 1.0e4
    w = wso.create_packets(n, seed, radius, temperature)
    p = oracle.create_packets(n, seed, radius, temperature)
    assert np.array_equal(w["packet_seeds"], p["packet_seeds"])
    assert (w["nus_bb_min"], w["nus_bb_max"]) == (p["initial_nus"].min(), p["initial_nus"].max())


@pytest.mark.parametrize("name", CASES)
def test_product_functions_match_reference_golden_and_oracle(shim, name):
    g = golden(name)
    seed, n, T = int(g["base_seed"]) + int(g["seed_offset"]), int(g["n"]), float(g["temperature"])
    got = shim(seed, n, radius=float(g["radius"]), temperature=T)
    check(got, g, T, what=name)
    want = wso.create_packets(n, seed, float(g["radius"]), T)
    check(got, want, T, what=name)
    # the sum the header forms is numpy's, bit for bit, given the same addends
    raw = shim(seed, n, radius=float(g["radius"]), temperature=T, normalize=False)
    i = raw["initial_energies"]
    assert raw["energy_sum"] == i.sum() == wso.pairwise_sum(i)
    assert np.array_equal(got["initial_energies"], i / raw["energy_sum"])


@pytest.mark.parametrize("n", [1, 7, 8, 9, 127, 128, 129, 8191, 8192, 8193, 20011, 10_000_019])
def test_pairwise_restatement_matches_numpy_sum(shim, n):
    """numpy's pairwise summation restated (the oracle's leaves + combine, and the header's pw_leaf_sum / pw_combine)
    against ndarray.sum(), bit for bit, on addends spanning ~16 decades."""
    rng = np.random.default_rng(n)
    a = rng.random(n) * np.exp(rng.normal(0.0, 6.0, n))
    want = a.sum()
    assert wso.pairwise_sum(a) == want
    assert shim.lib.shim_pairwise_sum(a.ctypes.data, n) == want
    if n > 128:  # every leaf holds 64 .. 128 elements, so start >> 6 names it; the header finds the same leaves
        leaves = wso.pairwise_leaves(n)
        assert min(m for _, m in leaves) >= 64 and max(m for _, m in leaves) <= 128
        s, m = C.c_uint64(), C.c_uint64()
        for start, length in leaves[:: max(1, len(leaves) // 500)]:
            shim.lib.shim_leaf_at(n, start + length - 1, C.byref(s), C.byref(m))
            assert (s.value, m.value) == (start, length)


def random_bounds(rng, n, G):
    """G members: sorted cut points, some repeated (empty members), some inside leaves"""
    cuts = np.sort(rng.integers(0, n + 1, G - 1))
    if G > 2:
        cuts[rng.integers(0, G - 1)] = cuts[rng.integers(0, G - 1)]
    return [0, *sorted(int(c) for c in cuts), n]


def test_member_splits_give_one_engines_arrays(shim):
    """Leaf sums by "leaves that start in my range" (a leaf that runs past a member's end regenerated to its end)
    combine to the whole set's sum bit for bit, and every array equals one member's, for G = 1 .. 8 members with empty
    members, cut points inside leaves, and fewer packets than members."""
    rng = np.random.default_rng(2026)
    for n, seed in ((20011, 5), (1000, 6), (129, 7), (5, 8), (2, 9)):
        one = shim(seed, n, chunk=256)
        for G in range(1, 9):
            for trial in range(3):
                bounds = random_bounds(rng, n, G)
                got = shim(seed, n, bounds=bounds, chunk=int(rng.choice([1, 64, 100, 256])))
                assert got["energy_sum"] == one["energy_sum"], (n, bounds)
                for k in EXACT + ("initial_nus", "initial_energies"):
                    assert np.array_equal(got[k], one[k]), (n, bounds, k)


def test_mirror_keeps_the_reference_surface():
    from tardis_b200.packet_source import BlackBodySimpleSourceB200, BlackBodyWeightedSourceB200 as Src

    with open(os.path.join(HERE, "golden", "reference_interface_weighted_source.json")) as f:
        ref = json.load(f)
    assert ref["bases"] == ["BlackBodySimpleSource"] and issubclass(Src, BlackBodySimpleSourceB200)
    assert Src.hdf_name == ref["attributes"]["hdf_name"] == "black_body_weighted_source"
    assert Src.hdf_properties == ref["attributes"]["hdf_properties"]
    assert all(hasattr(Src, m) for m in ref["methods"] if not m.startswith("create_packet_"))
    assert ref["init"] == {"positional": [], "kwarg": "kwargs"}
    with pytest.raises(TypeError):
        Src(1.0e15, 1.0e4)  # keyword arguments only, as the reference class
    s = Src(radius=1.0e15, temperature=1.0e4, base_seed=1)
    with pytest.raises(ValueError):
        s.create_packets(0)  # nus.min() of zero packets
    with pytest.raises(ValueError):
        wso.create_packets(0, 1, 1.0e15, 1.0e4)
    with pytest.raises(ValueError):
        s.create_packets(10)  # no engine attached
    with pytest.raises(NotImplementedError):
        Src(radius=1.0e15, temperature=1.0e4, base_seed=1, legacy_mode_enabled=True)


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def engine():
    from tardis_b200.engine import Engine

    eng = Engine(0)
    yield eng
    eng.close()


@pytest.mark.gpu
def test_device_source_matches_goldens_and_oracle(engine):
    from tardis_b200.engine import EngineError

    measured = {}
    for name in CASES:
        g = golden(name)
        seed, n, T = int(g["base_seed"]) + int(g["seed_offset"]), int(g["n"]), float(g["temperature"])
        engine.create_packets(n, seed, float(g["radius"]), T, weighted=True)
        got = engine.download_packets()
        measured[name] = check(got, g, T, what=name)
        check(got, wso.create_packets(n, seed, float(g["radius"]), T), T, what=name)
    for n, seed in ((100_003, 11), (8192, 12), (129, 13)):
        engine.create_packets(n, seed, 1.2e15, 1.0e4, weighted=True)
        measured[n] = check(engine.download_packets(), wso.create_packets(n, seed, 1.2e15, 1.0e4), 1.0e4, what=n)
    print("measured (max nu ulps, max energy error / allowance):", measured)
    with pytest.raises((EngineError, ValueError)):
        engine.create_packets(10, 1, 1.2e15, 1.0e4, beta=0.01, weighted=True)  # no relativistic weighted source
    with pytest.raises((EngineError, ValueError)):
        engine.create_packets(0, 1, 1.2e15, 1.0e4, weighted=True)
    engine.create_packets(1000, 3, 1.2e15, 1.0e4)  # the plain source afterwards is untouched: energies 1 / N
    assert np.array_equal(engine.download_packets()["initial_energies"], np.ones(1000) / 1000)


@pytest.mark.gpu
@pytest.mark.parametrize("ids", [[0], [0, 0], [0, 0, 0]])
def test_group_weighted_source_is_one_engines(engine, ids):
    """Shard edges inside leaves (N / G is rarely a leaf edge) and fewer packets than members."""
    from tardis_b200.engine import EngineGroup

    g = EngineGroup(ids)
    try:
        for n, seed in ((100_003, 21), (20011, 22), (1000, 23), (2, 24), (1, 25)):
            engine.create_packets(n, seed, 1.2e15, 1.0e4, weighted=True)
            want = engine.download_packets()
            g.create_packets(n, seed, 1.2e15, 1.0e4, weighted=True)
            got = g.download_packets()
            for k in want:
                assert np.array_equal(got[k], want[k]), (n, k)
    finally:
        g.close()


def segments_per_shell(ref, n_shells):
    """Trace segments per shell from the oracle's event log: every straight flight inside a shell ends in exactly one
    logged event (boundary crossing or interaction) whose before_shell_id is that shell.  A segment crosses each line of
    its shell at most once, so this bounds the number of terms any cell of the shell received."""
    ev = np.concatenate(ref["events"])
    return np.bincount(ev["before_shell_id"][(ev["before_shell_id"] >= 0) & (ev["before_shell_id"] < n_shells)], minlength=n_shells)


def assert_fixed_point_bound(got, want, nu_line, scale, segments, what):
    """|d| <= segments(shell) * 0.5 * nu_i / scale + 1e-14 |want|: each term is rounded to one quantum (prefix / scale
    * nu_i is the cell), the rest is f64 rounding of the oracle's sum and of the final conversion."""
    got, want = np.asarray(got), np.asarray(want)  # [lines, shells]
    bound = segments[None, :] * 0.5 * nu_line[:, None] / scale + 1e-14 * np.abs(want)
    err = np.abs(got - want)
    assert (err <= bound).all(), (what, float((err / np.where(bound > 0, bound, 1)).max()))
    return float((err / np.where(bound > 0, bound, 1)).max())


@pytest.mark.gpu
def test_weighted_packets_through_the_transport(engine, oracle):
    """Weighted packets (energies over ~8 decades) through run_resident on a macroatom model with virtual packets,
    against the C oracle on the same packets."""
    from golden_util import assert_close

    from tardis_b200 import synthetic as syn

    model = syn.make_model(10, 4000, "macroatom", mu_tau=-4.0, seed=31, n_bins=500)
    n = 20011
    engine.set_model_from(model, number_of_vpackets=3)
    engine.create_packets(n, 1234, float(model.r_inner[0]), 1.0e4, weighted=True)
    pk = engine.download_packets()
    assert pk["initial_energies"].max() / pk["initial_energies"].min() > 1e3
    res = engine.run_resident(track_last_interaction=True)
    packets = syn.Packets(pk["initial_radii"], pk["initial_nus"], pk["initial_mus"], pk["initial_energies"], pk["packet_seeds"], 1.0)
    ref = oracle.run_oracle(model, packets, number_of_vpackets=3, nthreads=8, n_tracked_packets=n, max_events_per_packet=4096)
    assert (ref["event_counts"] < 4096).all()
    assert all(res["counters"][k] == v for k, v in ref["counters"].items())
    for k in ("last_interaction_type", "last_event_id", "last_shell_id", "last_line_absorb_id", "last_line_emit_id"):
        assert np.array_equal(res[k], ref[k]), k
    assert_close(res["output_nus"], ref["output_nus"], 1e-11, "output_nus")
    assert_close(res["output_energies"], ref["output_energies"], 1e-11, "output_energies")
    for k in ("j", "nu_bar", "vhist"):
        assert_close(res[k], ref[k], 1e-10, k)
    # numpy.histogram's bins ([grid[i], grid[i+1]), the last one closed), each bin summed on its own: np.histogram with an
    # edge array forms bin sums as differences of one cumulative sum, whose rounding (an ulp of the total) would swamp
    # the small far-tail bins that weighted packets fill
    nu, e, grid = ref["output_nus"], ref["output_energies"], model.spectrum_frequency_grid
    sel = (e >= 0) & (nu >= grid[0]) & (nu <= grid[-1])
    idx = np.minimum(np.searchsorted(grid, nu[sel], side="right") - 1, len(grid) - 2)
    em = np.bincount(idx, weights=e[sel], minlength=len(grid) - 1)
    assert_close(res["spectrum_emitted"], em, 1e-11, "spectrum_emitted", atol=1e-18)
    _, _, scale_j_blue, scale_edotlu = engine.line_accumulators()
    seg = segments_per_shell(ref, model.n_shells)
    worst = [assert_fixed_point_bound(res["j_blue"], ref["j_blue"], model.line_list_nu, scale_j_blue, seg, "j_blue"),
             assert_fixed_point_bound(res["edotlu"], ref["edotlu"], model.line_list_nu, scale_edotlu, seg, "edotlu")]
    print("J_blue / Edotlu error as a fraction of the fixed-point bound:", worst)


@pytest.mark.gpu
def test_drop_in_solver_with_the_weighted_source(engine, oracle, monkeypatch):
    """from_config -> initialize_transport_state -> run with BlackBodyWeightedSourceB200 against the oracle on the packets
    the source made."""
    from types import SimpleNamespace

    from golden_util import assert_close
    from test_host_logic import _fake_config

    from tardis_b200 import montecarlo as mc
    from tardis_b200 import synthetic as syn
    from tardis_b200.packet_source import BlackBodyWeightedSourceB200

    monkeypatch.setattr(mc, "get_engine", lambda device=0: engine)
    model = syn.make_model(8, 2500, "macroatom", mu_tau=-3.5, seed=41)
    geo = mc.HomologousGeometry(model.r_inner, model.r_outer, model.v_inner, model.v_outer, model.time_explosion)
    cfg = _fake_config()
    source = BlackBodyWeightedSourceB200(radius=float(model.r_inner[0]), temperature=1.0e4, base_seed=23111963, engine=engine)
    solver = mc.MCTransportSolverB200.from_config(cfg, source)
    sim_state = SimpleNamespace(geometry=SimpleNamespace(to_numba=lambda: geo, v_inner_boundary_idx=0, v_outer_boundary_idx=8),
                                time_explosion=model.time_explosion)
    opacity_host = SimpleNamespace(to_numba=lambda macro_atom_state, lit: mc.OpacityState.from_model(model))
    plasma = SimpleNamespace(continuum_interaction_species=SimpleNamespace(empty=True))
    state = solver.initialize_transport_state(sim_state, opacity_host, None, plasma, 3001, iteration=2)
    pc = state.packet_collection
    want = wso.create_packets(3001, 23111963 + 2, float(model.r_inner[0]), 1.0e4)
    check({k: np.asarray(getattr(pc, k)) for k in ("initial_radii", "initial_nus", "initial_mus", "initial_energies", "packet_seeds")},
          want, 1.0e4, what="drop-in")
    assert np.array_equal(source.nus, pc.initial_nus)
    solver.run(state, show_progress_bars=False)
    packets = syn.Packets(*(np.asarray(getattr(pc, k)) for k in ("initial_radii", "initial_nus", "initial_mus", "initial_energies",
                                                                  "packet_seeds")), 1.0)
    ref = oracle.run_oracle(model, packets)
    assert_close(pc.output_nus, ref["output_nus"], 1e-11, "output_nus")
    assert_close(state.j_estimator, ref["j"], 1e-10, "j")
    assert_close(state.nu_bar_estimator, ref["nu_bar"], 1e-10, "nu_bar")
