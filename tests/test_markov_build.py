"""The continuum macro atom's absorbing Markov chain on the device (tardis_b200/csrc/markov_build.cuh,
tb200_build_absorbing_markov).

CPU: (1) the oracle (oracle/markov_oracle.py) against golden vectors of the reference's own create_absorbing_probs and
normalisation (tests/golden/make_markov_golden.py); (2) the PRODUCT's functions -- the header the kernels compile, built
for the host by tests/markov_build_shim.cpp -- against the same.
GPU: the device tables against the goldens; both sides of the shared-memory dispatch (n <= 128) at odd sizes, bit for bit
against the shim; refusals followed by good runs; repeat builds and engine-group members bit-identical; continuum
transport on the device-built tables equal to transport on their downloaded copy, and to the C oracle.
Bars: X has the reference's zero pattern (see `check`) and lies within 1e-13 of it, row sums within 1e-13 (ill-conditioned
shell: at least as accurate as the reference's splu, see the comment above `all_zero_states`); the deactivation table bit-identical."""
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np
import pytest

from golden_util import GOLDEN_DIR, assert_close

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _load_generator():
    import importlib.util

    spec = importlib.util.spec_from_file_location("make_markov_golden", os.path.join(GOLDEN_DIR, "make_markov_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


gen = _load_generator()
CASES = list(gen.MARKOV_CASES)
SMALL = [n for n in CASES if gen.MARKOV_CASES[n][3] != "counts"]
BAR = 1e-13


def golden(name):
    model, cma = gen.markov_inputs(name)
    return model, cma, dict(np.load(os.path.join(GOLDEN_DIR, name + ".npz")))


# On an ill-conditioned shell (internal share 1 - 1e-6, condition ~1e6) splu and the pivoted dense solve are both ~3e-13 away
# from the solution of the same float64 system (oracle solver "extended", long double) and only 2.3e-14 from each other:
# their errors are correlated, so that distance says nothing about accuracy (the extended solution itself is 13 x it away
# from splu).  There X is held to accuracy instead: at least as close to the extended solution as splu is, cell by cell
# and in the row sums, per shell (1e-13 at least).


def all_zero_states(cma):
    """[S, n]: states whose rows are all zero in that shell (their row of I - Q is the identity row, X's row is e_i)."""
    p, e = cma.transition_probabilities, cma.macro_block_edge_index
    return np.array([[not p[e[i]:e[i + 1], s].any() for i in range(len(e) - 1)] for s in range(p.shape[1])], dtype=bool)


def check(name, cma, X, D, g, exact_zeros=True):
    """Zeros: X is zero exactly where the long-double solution of the same system is (both directions), and zero wherever
    the reference's is.  The reference may hold roundoff (|x| <= 1e-15, of either sign) where no path leads: splu's
    permuted factors leave it, e.g. in the rows of states whose probabilities are all zero (X's row is exactly e_i there)."""
    from oracle import markov_oracle as mo

    seed, _, kw, storage = gen.MARKOV_CASES[name]
    args = (cma.transition_probabilities, cma.source_level_idx, cma.destination_level_idx, cma.transition_type)
    E = mo.absorbing_probs(*args, solver="extended") if storage != "counts" else None
    if not exact_zeros:  # the oracle's splu: the reference's own roundoff, checked against the golden only
        ref = g["X"] if "X" in g else None
        if ref is not None:
            assert np.array_equal(X, ref) or np.abs(X - ref).max() <= BAR
        else:
            assert np.abs(X.ravel()[g["sample_idx"]] - g["sample_val"]).max() <= BAR
        assert np.abs(X.sum(axis=2) - g["row_sums"]).max() <= BAR
    else:
        _check_product(name, kw, storage, X, E, g, cma)
    if "deactivation" in g:
        assert np.array_equal(D.view(np.uint64), g["deactivation"].view(np.uint64)), "deactivation table not bit-identical"
    else:
        assert hashlib.sha256(np.ascontiguousarray(D).tobytes()).hexdigest() == str(g["deactivation_sha256"])


def _check_product(name, kw, storage, X, E, g, cma):
    if E is not None:
        assert np.array_equal(X == 0, E == 0), "zero pattern of X differs from the exact one"
    zs = all_zero_states(cma)
    assert (X[zs] == np.eye(X.shape[1])[np.nonzero(zs)[1]]).all(), "rows of all-zero states are not e_i"
    if kw.get("ill_conditioned_shell") is not None:
        ref = g["X"]
        cell_bar = np.maximum(BAR, np.abs(ref - E).max(axis=(1, 2)))
        row_bar = np.maximum(BAR, np.abs(ref.sum(axis=2) - E.sum(axis=2)).max(axis=1))
        assert (np.abs(X - E).max(axis=(1, 2)) <= cell_bar).all(), (np.abs(X - E).max(axis=(1, 2)), cell_bar)
        assert (np.abs(X.sum(axis=2) - E.sum(axis=2)).max(axis=1) <= row_bar).all()
    else:
        assert np.abs(X.sum(axis=2) - g["row_sums"]).max() <= BAR, f"row sums: {np.abs(X.sum(axis=2) - g['row_sums']).max():.3e}"
    if "X" in g:
        ref = g["X"]
        assert np.abs(X - ref).max() <= (BAR if kw.get("ill_conditioned_shell") is None else np.inf)
    elif "zero_bits" in g:
        ref = np.where(np.unpackbits(g["zero_bits"])[: X.size].astype(bool).reshape(X.shape), 0.0, np.nan)
    else:
        ref = None
        assert np.array_equal((X == 0).sum(axis=2), g["zero_counts"]), "zero counts of X differ"
    if ref is not None:
        assert not ((ref == 0) & (X != 0)).any(), "X is non-zero where the reference's X is zero"
    if "sample_idx" in g:
        flat = X.ravel()[g["sample_idx"]]
        sv = g["sample_val"]
        assert np.abs(flat - sv).max() <= BAR
        assert not ((sv == 0) & (flat != 0)).any()
        assert (np.abs(sv[(flat == 0) & (sv != 0)]) <= 1e-15).all()
    if "X" in g:
        assert (np.abs(g["X"][(X == 0) & (g["X"] != 0)]) <= 1e-15).all(), "X is zero where the reference holds more than roundoff"


# ---- CPU -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_golden(name):
    from oracle import markov_oracle as mo

    model, cma, g = golden(name)
    X = mo.absorbing_probs(cma.transition_probabilities, cma.source_level_idx, cma.destination_level_idx, cma.transition_type)
    D = mo.deactivation_table(cma.transition_probabilities, cma.transition_type, cma.macro_block_edge_index)
    check(name, cma, X, D, g, exact_zeros=False)


@pytest.fixture(scope="module")
def shim():
    out = os.path.join(HERE, "_shim", "libmarkov_build_shim.so")
    src = os.path.join(HERE, "markov_build_shim.cpp")
    hdr = os.path.join(ROOT, "tardis_b200", "csrc", "markov_build.cuh")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", out, src], check=True)
    lib = C.CDLL(out)
    lib.shim_markov_build.restype = C.c_longlong
    lib.shim_markov_build.argtypes = [C.c_int] * 3 + [C.c_void_p] * 6

    def run(cma, expect_error=False):
        p = np.ascontiguousarray(cma.transition_probabilities, dtype=np.float64)
        T, S = p.shape
        n = cma.n_states
        X, D = np.empty((S, n, n)), np.empty((T, S))
        arrs = [np.ascontiguousarray(a, dtype=np.int64) for a in (cma.transition_type, cma.destination_level_idx, cma.macro_block_edge_index)]
        err = lib.shim_markov_build(T, S, n, p.ctypes.data, *(a.ctypes.data for a in arrs), X.ctypes.data, D.ctypes.data)
        assert (err >= 0) == expect_error, err
        return (X, D) if not expect_error else (int(err) % S, int(err) // S)

    return run


@pytest.mark.parametrize("name", SMALL)
def test_product_functions_match_reference_golden(shim, name):
    model, cma, g = golden(name)
    check(name, cma, *shim(cma), g)


def chain(n, S=3, seed=0, singular_shell=None):
    """A model with an n-state continuum macro atom (n >= 1): every state has 0-3 internal rows and 1-2 free-free emission
    rows.  singular_shell: states 0 and 1 (n >= 2) point only at each other there -- I - Q is singular at state 1."""
    from tardis_b200 import synthetic as syn

    rng = np.random.default_rng(seed)
    model = syn.add_continuum(syn.make_model(S, 300, "macroatom", mu_tau=-4.0, seed=seed + 1), seed=seed + 2)
    src, dst, tt, edges = [], [], [], [0]
    for b in range(n):
        k = 1 if (singular_shell is not None and b < 2) else int(rng.integers(0, 4))
        for _ in range(k):
            src.append(b); dst.append((1 - b) if (singular_shell is not None and b < 2) else int(rng.integers(0, n))); tt.append(0)
        for _ in range(int(rng.integers(1, 3))):
            src.append(b); dst.append(-1); tt.append(-3)
        edges.append(len(src))
    src, dst, tt, edges = (np.array(a, dtype=np.int64) for a in (src, dst, tt, edges))
    raw = rng.random((len(src), S)) + 0.05
    share = rng.uniform(0.2, 0.9, (n, S))
    p = np.zeros_like(raw)
    for b in range(n):
        blk = slice(edges[b], edges[b + 1])
        inn = tt[blk] >= 0
        r = raw[blk]
        part = np.where(inn[:, None], r / np.maximum(r[inn].sum(axis=0), 1e-300) * share[b], r / r[~inn].sum(axis=0) * (1 - share[b]))
        if not inn.any():
            part = r / r.sum(axis=0)
        if singular_shell is not None and b < 2:
            part[:, singular_shell] = np.where(inn, 1.0, 0.0)
        p[blk] = part
    model.macro = syn.MacroAtomTables(np.ascontiguousarray(p), rng.integers(0, n, model.n_lines).astype(np.int64), edges, tt, dst,
                                      np.zeros(len(src), dtype=np.int64))
    model.continuum.k_packet_idx = 0
    model.continuum.photo_ion_activation_idx = np.full(30, n - 1, dtype=np.int64)
    model.continuum.absorbing_markov_probabilities = None
    return model, syn.ContinuumMacroAtom(np.ascontiguousarray(p), src, dst, tt, edges, n)


def test_shim_names_the_singular_state(shim):
    _, cma = chain(5, S=4, seed=3, singular_shell=2)
    assert shim(cma, expect_error=True) == (2, 1)


# ---- GPU -------------------------------------------------------------------------------------------------------------
def engine_for(model, keep=True, group=None):
    from tardis_b200.engine import Engine, EngineGroup

    eng = EngineGroup(group) if group is not None else Engine(0)
    if keep:
        eng.set_option("keep_opacity_tables", 1)
    eng.set_model_from(model, enable_full_relativity=True)
    return eng


def build(eng, cma, **kw):
    eng.build_absorbing_markov(cma.transition_probabilities, cma.source_level_idx, cma.destination_level_idx, cma.transition_type, **kw)
    return eng.download_absorbing_markov()


def tiny_packets(model):
    return (np.full(1, model.r_inner[0]), np.full(1, 1e15), np.full(1, 0.5), np.ones(1), np.ones(1, dtype=np.int64))


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_engine_builds_the_reference_tables(name):
    from tardis_b200.engine import EngineError

    model, cma, g = golden(name)
    eng = engine_for(model)
    eng.upload_packets(*tiny_packets(model))
    with pytest.raises(EngineError, match="tb200_build_absorbing_markov"):  # the macro atom is pending until the build
        eng.transport(True)
    got = build(eng, cma)
    check(name, cma, got["absorbing_markov_probabilities"], got["transition_probabilities"], g)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 63, 64, 65, 127, 128, 129, 200])
def test_sizes_on_both_sides_of_the_shared_memory_path(shim, n):
    """n <= 128: one CTA per shell in shared memory; above: one pivot + one update launch per step.  Both run the shim's
    functions in the shim's order, so the device tables equal the shim's bit for bit; and they match the oracle."""
    from oracle import markov_oracle as mo

    model, cma = chain(n, S=3, seed=n)
    eng = engine_for(model)
    got = build(eng, cma)
    X, D = shim(cma)
    assert np.array_equal(got["absorbing_markov_probabilities"].view(np.uint64), X.view(np.uint64))
    assert np.array_equal(got["transition_probabilities"].view(np.uint64), D.view(np.uint64))
    args = (cma.transition_probabilities, cma.source_level_idx, cma.destination_level_idx, cma.transition_type)
    ref = mo.absorbing_probs(*args)
    assert np.array_equal(X == 0, mo.absorbing_probs(*args, solver="extended") == 0)  # exact zeros, both ways
    assert not ((ref == 0) & (X != 0)).any() and (np.abs(ref[X == 0]) <= 1e-15).all()  # splu: roundoff where no path leads
    assert np.abs(X - ref).max() <= BAR
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [5, 200])
def test_refusals_leave_the_engine_usable(oracle, n):
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import EngineError

    model, cma = chain(n, S=4, seed=7)
    bad_model, bad = chain(n, S=4, seed=7, singular_shell=2)
    packets = syn.make_packets(3000, model.r_inner[0], base_seed=8)
    eng = engine_for(bad_model)
    with pytest.raises(EngineError, match="singular in shell 2 at state 1"):
        build(eng, bad)
    eng.upload_packets(*tiny_packets(model))
    with pytest.raises(EngineError, match="pending"):  # a failed build leaves the macro atom pending
        eng.transport(True)
    eng.set_model_from(model, enable_full_relativity=True)
    args = (cma.transition_probabilities, cma.source_level_idx, cma.destination_level_idx, cma.transition_type)
    d = cma.destination_level_idx.copy()
    d[np.flatnonzero(cma.transition_type >= 0)[0]] = n
    with pytest.raises(EngineError, match="destination_level_idx out of range"):
        eng.build_absorbing_markov(args[0], args[1], d, args[3])
    s = cma.source_level_idx.copy()
    s[0], s[-1] = s[-1], s[0]
    with pytest.raises(EngineError, match="source"):
        eng.build_absorbing_markov(args[0], s, args[2], args[3])
    with pytest.raises(EngineError, match="n_states"):
        eng.build_absorbing_markov(*args, n_states=n + 1)
    got = build(eng, cma)
    host = host_model(model, got)
    res = eng.run_packets(packets)
    ref = oracle.run_oracle(host, packets)
    compare_to_oracle(res, ref)
    eng.close()


@pytest.mark.gpu
def test_oversize_chain_is_refused_before_allocating():
    from tardis_b200.engine import EngineError

    model, cma = chain(40000, S=8, seed=11)  # 8 x 40000^2 doubles = 102 GB
    eng = engine_for(model, keep=False)
    with pytest.raises(EngineError, match="needs"):
        eng.build_absorbing_markov(cma.transition_probabilities, cma.source_level_idx, cma.destination_level_idx, cma.transition_type)
    small, scma = chain(70, S=8, seed=12)
    eng.set_option("keep_opacity_tables", 1)
    eng.set_model_from(small, enable_full_relativity=True)
    build(eng, scma)
    eng.close()


@pytest.mark.gpu
def test_two_builds_are_bit_identical():
    model, cma = gen.markov_inputs("markov_n400")
    eng = engine_for(model)
    a = build(eng, cma)
    b = build(eng, cma)
    for k in a:
        assert np.array_equal(a[k].view(np.uint64), b[k].view(np.uint64)), k
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("peer", [1, 0])
def test_group_members_are_bit_identical(peer):
    model, cma = gen.markov_inputs("markov_n400")
    one = engine_for(model)
    want = build(one, cma)
    grp = engine_for(model, group=[0, 0])
    grp.set_option("peer_access", peer)
    build(grp, cma)
    for m in grp.members:
        got = m.download_absorbing_markov()
        for k in want:
            assert np.array_equal(got[k].view(np.uint64), want[k].view(np.uint64)), k
    one.close()
    grp.close()


def host_model(model, tables):
    """`model` with the downloaded tables as host-built inputs of tb200_set_model"""
    import copy

    host = copy.deepcopy(model)
    host.macro.transition_probabilities = tables["transition_probabilities"]
    host.continuum.absorbing_markov_probabilities = tables["absorbing_markov_probabilities"]
    return host


def compare_to_oracle(res, ref):
    """test_gpu_parity.py's bars for the continuum mode"""
    assert all(res["counters"][k] == v for k, v in ref["counters"].items()), (res["counters"], ref["counters"])
    assert np.array_equal(res["output_energies"] == -99.0, ref["output_energies"] == -99.0)
    assert_close(res["output_nus"], ref["output_nus"], 1e-11, "output_nus")
    assert_close(res["j"], ref["j"], 1e-10, "j")
    assert_close(res["j_blue"], ref["j_blue"], 1e-10, "j_blue")
    for k in ("photo_ion_estimator", "stim_recomb_estimator", "bf_heating_estimator", "stim_recomb_cooling_estimator", "ff_heating_estimator"):
        assert_close(res[k], ref[k], 1e-10, k)
    assert np.array_equal(res["photo_ion_estimator_statistics"], ref["photo_ion_estimator_statistics"])


@pytest.mark.gpu
def test_transport_on_device_built_tables_equals_the_uploaded_copy(oracle):
    """Transport on the tables the engine built == transport on their downloaded copy uploaded through tb200_set_model:
    per-packet outputs, last-interaction columns, counters, J_blue / Edotlu (fixed-point) bit for bit; the estimators that
    the kernels sum with f64 atomics (J, nu_bar, the continuum estimators) vary in their last bits from run to run of one
    engine, so within 1e-13 there, with exact bound-free statistics.  And both == the C oracle on the copy."""
    from tardis_b200 import synthetic as syn

    model, cma = gen.markov_inputs("markov_n62")
    packets = syn.make_packets(20000, model.r_inner[0], base_seed=91)
    eng = engine_for(model)
    tables = build(eng, cma)
    dev = eng.run_packets(packets, track_last_interaction=True)
    host = host_model(model, tables)
    eng.set_model_from(host, enable_full_relativity=True)
    up = eng.run_packets(packets, track_last_interaction=True)
    assert dev["counters"] == up["counters"]
    assert dev["counters"]["n_continuum_events"] > 0 and dev["counters"]["n_macro_jumps"] > 0
    exact = ("output_nus", "output_energies", "j_blue", "edotlu", "photo_ion_estimator_statistics", "last_interaction_type",
             "last_shell_id", "last_line_absorb_id", "last_line_emit_id", "last_after_nu", "last_after_energy")
    for k in exact:
        assert np.array_equal(np.asarray(dev[k]).view(np.uint64) if np.asarray(dev[k]).dtype == np.float64 else dev[k],
                              np.asarray(up[k]).view(np.uint64) if np.asarray(up[k]).dtype == np.float64 else up[k]), k
    for k in ("j", "nu_bar", "photo_ion_estimator", "stim_recomb_estimator", "bf_heating_estimator", "stim_recomb_cooling_estimator",
              "ff_heating_estimator"):
        assert_close(dev[k], up[k], 1e-13, k)
    ref = oracle.run_oracle(host, packets, nthreads=8)
    compare_to_oracle(dev, ref)
    eng.close()


@pytest.mark.gpu
def test_drop_in_end_to_end_with_the_reference_pandas_objects(oracle):
    """tardis_b200.macro_atom.create_absorbing_probs with the reference's pandas objects returns the reference's values;
    the IIP mirror then recognises the returned X in the opacity state, rebuilds it in HBM instead of uploading it, and
    transports exactly as with a plain copy of the same tables uploaded."""
    from types import SimpleNamespace

    import pandas as pd

    from oracle import markov_oracle as mo
    from tardis_b200 import macro_atom
    from tardis_b200 import montecarlo as mc
    from tardis_b200 import synthetic as syn

    model, cma, g = golden("markov_n62")
    meta = pd.DataFrame({"source": cma.source_level_idx, "source_level_idx": cma.source_level_idx,
                         "destination_level_idx": cma.destination_level_idx, "transition_type": cma.transition_type})
    tp = pd.DataFrame(cma.transition_probabilities.copy())
    eng = mc.get_engine(0)
    X, deact = macro_atom.create_absorbing_probs(tp, meta, max_workers=4)
    check("markov_n62", cma, X, mo.deactivation_table(cma.transition_probabilities, cma.transition_type, cma.macro_block_edge_index), g)
    want = tp.copy()
    want[meta.transition_type >= 0] *= 0
    pd.testing.assert_frame_equal(deact, want)
    D = mo.deactivation_table(deact.to_numpy(), cma.transition_type, cma.macro_block_edge_index)

    packets = syn.make_packets(5000, model.r_inner[0], base_seed=93)
    c, m = model.continuum, model.macro

    def run(matrix):
        pc = mc.PacketCollection(packets.initial_radii, packets.initial_nus, packets.initial_mus, packets.initial_energies,
                                 packets.packet_seeds, packets.radiation_field_luminosity)
        geo = mc.HomologousGeometry(model.r_inner, model.r_outer, model.v_inner, model.v_outer, model.time_explosion)
        fields = {**{k: getattr(m, k) for k in vars(m)}, **{k: getattr(c, k) for k in vars(c)}}
        fields.update(transition_probabilities=D, absorbing_markov_probabilities=matrix)
        opa = SimpleNamespace(electron_density=model.electron_density, t_electrons=model.t_electrons,
                              line_list_nu=model.line_list_nu, tau_sobolev=model.tau_sobolev, **fields)
        cfg = mc.MonteCarloConfiguration()
        cfg.LINE_INTERACTION_TYPE = 2
        cfg.ENABLE_FULL_RELATIVITY = True
        trackers = mc.generate_tracker_last_interaction_list(len(packets))
        bulk, line, cont = mc.montecarlo_transport(pc, geo, model.time_explosion, opa, cfg, (len(c.bf_threshold_list_nu), model.n_shells),
                                                   trackers, False, engine=eng)
        return pc, line, dict(mc.montecarlo_transport.last_counters), mc.montecarlo_transport.last_markov_rebuilt

    pc_a, line_a, cnt_a, rebuilt_a = run(X)
    pc_b, line_b, cnt_b, rebuilt_b = run(X.copy())
    assert rebuilt_a and not rebuilt_b
    assert cnt_a == cnt_b and cnt_a["n_continuum_events"] > 0
    assert np.array_equal(pc_a.output_nus.view(np.uint64), pc_b.output_nus.view(np.uint64))
    assert np.array_equal(pc_a.output_energies.view(np.uint64), pc_b.output_energies.view(np.uint64))
    assert np.array_equal(line_a.mean_intensity_blueward.view(np.uint64), line_b.mean_intensity_blueward.view(np.uint64))
