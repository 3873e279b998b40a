"""The nonhomologous transport mode (tardis_b200/csrc/nonhomologous.cuh, config.nonhomologous = 1).

CPU: (1) the product's quartic / line-distance header, built for the host by tests/nonhomologous_shim.cpp, against the
reference's own known answers and against the reference's compiled functions (when the reference tree is present);
(2) the CPU oracle (oracle/nonhomologous_oracle.cpp, which compiles the same header) against golden runs of the
unmodified reference (tests/golden/nonhomologous_*.npz, tests/golden/make_nonhomologous_golden.py).
GPU: the kernel through the C-ABI against the oracle.

Bars.  Device against oracle: integers identical, floats to 1e-10 -- both evaluate the quartic with the same IEEE
operations; what remains is CUDA's log / exp against glibc's (tau_event, exp(-tau) of the virtual packets) and the order
of the estimator sums.  Oracle against reference: the reference is Numba with fastmath, and the quartic turns an ulp of
its inputs into up to ~1e-4 relative in the root (1e-2 in the far tail: 99.9th percentile / maximum over 20000 random
cases per geometry; test_header_matches_reference_distance checks 3000 per geometry).  So on the stored runs the integers (fates, counters' event sequence, line ids)
must be identical and the floats agree to FLOAT_BAR = 1e-5 relative, checked per array (worst seen: 2.9e-6, one packet's
last_before_mu in the scatter case; all other arrays of all cases within 4e-10)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden")
sys.path.insert(0, GOLDEN)
import make_nonhomologous_golden as mk  # noqa: E402

FLOAT_BAR = 1e-5
GPU_RTOL = 1e-10


def reference_available():
    from oracle import reference_loader

    return reference_loader.available()


@pytest.fixture(scope="module")
def shim():
    return build_shim()


def build_shim():
    """tests/nonhomologous_shim.cpp built with g++ -ffp-contract=off (once), loaded with its signatures declared."""
    out = os.path.join(HERE, "_shim", "libnonhomologous_shim.so")
    src = os.path.join(HERE, "nonhomologous_shim.cpp")
    hdr = os.path.join(ROOT, "tardis_b200", "csrc", "nonhomologous.cuh")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", out, src], check=True)
    lib = C.CDLL(out)
    lib.shim_depressed_quartic.argtypes = [C.c_double] * 5 + [C.c_void_p]
    lib.shim_depressed_quartic.restype = None
    lib.shim_distance_line.argtypes = [C.c_double] * 8
    lib.shim_distance_line.restype = C.c_double
    for f in ("shim_cbrt", "shim_sin", "shim_cos"):
        getattr(lib, f).argtypes, getattr(lib, f).restype = [C.c_double], C.c_double
    for f in ("shim_atan2", "shim_hypot"):
        getattr(lib, f).argtypes, getattr(lib, f).restype = [C.c_double] * 2, C.c_double
    return lib


def quartic(shim, *args):
    out = np.empty(4)
    shim.shim_depressed_quartic(*[float(a) for a in args], out.ctypes.data)
    return out


# the reference's own test_depressed_quartic cases (transport/montecarlo/tests/test_nonhomologous.py:43-63)
@pytest.mark.parametrize("coeffs, roots", [
    ((1.0, -14.0, 71.0, -154.0, 120.0), [5.0, 4.0, 3.0, 2.0]),
    ((1.0, -1.0, 0.0, 0.0, 0.0), [1.0, 0.0, 0.0, 0.0]),
    ((1.0, -10.0, 35.0, -50.0, 24.0), [4.0, 3.0, 2.0, 1.0]),
])
def test_quartic_known_answers(shim, coeffs, roots):
    np.testing.assert_almost_equal(quartic(shim, *coeffs), roots)


def test_libm_restatements_are_accurate(shim):
    """The header's own hypot / pow(x, 1./3.) / atan2 / sin / cos (no libm on the quartic's path) against CPython's."""
    import math

    rng = np.random.default_rng(5)
    xs = 10.0 ** rng.uniform(-300, 300, 4000)
    ulps = [abs(shim.shim_cbrt(x) - x ** (1.0 / 3.0)) / np.spacing(x ** (1.0 / 3.0)) for x in xs]
    assert max(ulps) <= 1.0
    ph = rng.uniform(-math.pi / 3, math.pi / 3, 4000)
    assert max(abs(shim.shim_sin(p) - math.sin(p)) for p in ph) < 2e-16 * 8
    assert max(abs(shim.shim_cos(p) - math.cos(p)) for p in ph) < 2e-16 * 8
    ys, xx = rng.normal(size=4000), rng.normal(size=4000)
    assert max(abs(shim.shim_atan2(y, x) - math.atan2(y, x)) for y, x in zip(ys, xx)) < 1e-15
    assert shim.shim_atan2(0.0, -1.0) == math.pi and shim.shim_atan2(0.0, 1.0) == 0.0
    assert max(abs(shim.shim_hypot(y, x) - math.hypot(y, x)) / math.hypot(y, x) for y, x in zip(ys, xx)) < 5e-16


def random_cases(perturbed, n, seed):
    """Random packets and lines on the bench shells: 2e14-4e15 Hz, lines 1e-9 - 3e-3 relative from resonance, on the side
    of the comoving frequency the shell's gradient reaches."""
    rng = np.random.default_rng(seed)
    S = 20
    r = np.linspace(1.1e9, 2.0e9, S + 1) * 13 * 86400.0
    v = r / (13 * 86400.0)
    if perturbed:
        v = v.copy()
        v[1:-1] *= 1 + 0.08 * rng.uniform(-1, 1, S - 1)
    cases = []
    for _ in range(n):
        s = int(rng.integers(S))
        rr, mu = rng.uniform(r[s], r[s + 1]), rng.uniform(-1, 1)
        nu = 10 ** rng.uniform(np.log10(2e14), np.log10(4e15))
        dvdr = (v[s + 1] - v[s]) / (r[s + 1] - r[s])
        vel = v[s] + dvdr * (rr - r[s])
        cnu = nu * (1.0 - mu * (vel / 2.99792458e10))
        nl = cnu * (1 - np.sign(dvdr) * 10 ** rng.uniform(-9, np.log10(3e-3)))
        cases.append((rr, mu, nu, nl, r[s], r[s + 1], v[s], v[s + 1]))
    return cases


def reference_distance(R, rr, mu, nu, nl, ri, ro, vi, vo):
    geo = R.NumbaRadial1DGeometry(np.array([ri]), np.array([ro]), np.array([vi]), np.array([vo]))
    p = R.RPacket(rr, mu, nu, 1.0, 0)
    p.current_shell_id = 0
    return R.calculate_distance_line_nonhomologous(p, geo, nl)


@pytest.mark.skipif(not reference_available(), reason="needs the reference tree")
@pytest.mark.parametrize("perturbed, bars", [
    # median, 99.9th percentile, max relative difference; measured on the CPU: 2.5e-11 / 1.6e-7 / 1.9e-6 (v = r / t) and
    # 1.9e-12 / 1.2e-4 / 5.5e-2 (perturbed), the spread of the quartic's conditioning, with a margin of ~10
    (False, (1e-9, 2e-6, 2e-5)),    # v = r / t
    (True, (1e-9, 1e-3, 2e-1)),     # interior velocities +-8 %, some shells decelerate
])
def test_header_matches_reference_distance(shim, perturbed, bars):
    """The header's line distance against the reference's compiled calculate_distance_line_nonhomologous: the same cases
    miss (MISS_DISTANCE), and the roots agree to the bars, which are those of the quartic's conditioning (a one-ulp change
    of the packet frequency moves the strict IEEE evaluation by the same amounts)."""
    from oracle.reference_runner_nonhomologous import load

    R = load()
    rel = []
    for case in random_cases(perturbed, 3000, 11 + perturbed):
        a = reference_distance(R, *case)
        b = shim.shim_distance_line(*case)
        assert (a >= 1e99) == (b >= 1e99), case
        if a < 1e99:
            rel.append(abs(a - b) / a)
    rel = np.array(rel)
    assert np.median(rel) < bars[0] and np.percentile(rel, 99.9) < bars[1] and rel.max() < bars[2], (
        np.median(rel), np.percentile(rel, 99.9), rel.max())


@pytest.mark.skipif(not reference_available(), reason="needs the reference tree")
def test_header_matches_reference_crafted(shim):
    """Crafted cases: a complex r, a negative real r (complex cube root), v0 == 0, +-2e-14 around resonance and a
    decelerating shell.  (The degenerate quartics -- the u == 0 branch and the no-real-roots fallback -- are in
    test_quartic_degenerate_branches: the reference's compiled code does not follow its source there.)"""
    from oracle.reference_runner_nonhomologous import load

    R = load()
    for coeffs in [(1.0, 0.0, -5.0, 0.0, 4.0),            # roots +-1, +-2: q2p3 < 0 (complex r)
                   (1.0, 0.0, 0.0, 1.0, 0.0),             # negative real r: principal-branch cube root
                   (1.0, -14.0, 71.0, -154.0, 120.0)]:    # q2p3 < 0 with a shift
        ref = np.array(R.depressed_quartic(*coeffs), dtype=float)
        got = quartic(shim, *coeffs)
        np.testing.assert_array_equal(np.isnan(ref), np.isnan(got))
        np.testing.assert_allclose(got[~np.isnan(got)], ref[~np.isnan(ref)], rtol=1e-12, atol=1e-14)
    r0, r1 = 1.5e14, 1.6e14
    for vi, vo in [(1.2e9, 1.2e9), (1.2e9, 1.3e9), (1.3e9, 1.2e9)]:   # flat, accelerating, decelerating
        for mu in (-0.7, 0.1, 0.9):
            rr, nu = 1.55e14, 1e15
            dvdr = (vo - vi) / (r1 - r0)
            cnu = nu * (1.0 - mu * ((vi + dvdr * (rr - r0)) / 2.99792458e10))
            # (exactly at the 1e-14 window the compiled reference -- fastmath, contracted -- may decide either way; the
            # device and the oracle share the header, and are compared there on the GPU)
            for rel in (2e-14, -2e-14, 1e-13, -1e-13, 1e-5, -1e-5):
                nl = cnu * (1 - rel)
                a = reference_distance(R, rr, mu, nu, nl, r0, r1, vi, vo)
                b = shim.shim_distance_line(rr, mu, nu, nl, r0, r1, vi, vo)
                assert (a >= 1e99) == (b >= 1e99), (vi, vo, mu, rel, a, b)
                if a < 1e99:
                    # d = r0 x - r mu cancels near resonance: the error is a fraction 1e-13 of r (the conditioned root), not of d
                    assert abs(a - b) <= 1e-6 * a + 1e-12 * rr, (vi, vo, mu, rel, a, b)


def test_quartic_degenerate_branches(shim):
    """The branches of depressed_quartic that only degenerate inputs reach, as the source states them.  The reference's
    compiled function (fastmath: no NaNs assumed) folds its np.isnan tests to False, so it returns four NaNs where the
    source's fallback forces the smaller term to zero, and differs on the all-zero quartic too; the header follows the
    source (DESIGN.md, nonhomologous mode).  In the line-distance sets of test_header_matches_reference_distance no case
    reaches these branches."""
    # x^4 + x^2 + 1: no real roots; term[0] = term[1] < 0, so the fallback zeroes term 0: x1 = x2 = w / 2
    r = quartic(shim, 1.0, 0.0, 1.0, 0.0, 1.0)
    assert r[0] == r[1] and np.isfinite(r[0]) and np.isnan(r[2]) and np.isnan(r[3])
    # x^4: p = q = 0, so r = 0 and the u == 0 branch: y = -5/6 a - q ** (1/3) = 0, w = 0, 2 b / w = NaN
    r = quartic(shim, 1.0, 0.0, 0.0, 0.0, 0.0)
    assert np.isnan(r[0]) and np.isnan(r[1]) and r[2] == 0.0 and r[3] == 0.0


def golden(name):
    return dict(np.load(os.path.join(GOLDEN, f"nonhomologous_{name}.npz")))


INT_KEYS = ("last_interaction_type", "last_event_id", "last_shell_id", "last_line_absorb_id", "last_line_emit_id")
FLOAT_KEYS = ("output_nus", "output_energies", "j", "nu_bar", "j_blue", "edotlu", "vhist", "last_radius", "last_before_nu",
              "last_before_mu", "last_before_energy", "last_after_nu", "last_after_mu", "last_after_energy")


@pytest.mark.parametrize("name", list(mk.CASES) + list(mk.SIGMA_CASES))
def test_oracle_matches_reference_golden(name):
    from oracle import nonhomologous_oracle

    model, packets, kw = mk.case_inputs(name)
    g = golden(name)
    got = nonhomologous_oracle.run_oracle(model, packets, vlog_capacity=100000 if kw.get("number_of_vpackets") else 0, **kw)
    if kw.get("survival_probability"):
        # the Russian roulette fired (tau > 10) and killed some virtual packets: the survival probability is exercised
        assert np.count_nonzero(got["vlog_energies"][: got["vlog_count"]] == 0.0) > 0
    np.testing.assert_array_equal(np.sign(got["output_energies"]), np.sign(g["output_energies"]), err_msg="fates")
    for k in INT_KEYS:
        np.testing.assert_array_equal(got[k], g[k], err_msg=k)
    for k in FLOAT_KEYS:
        np.testing.assert_allclose(got[k], g[k], rtol=FLOAT_BAR, atol=0, equal_nan=True, err_msg=k)


@pytest.mark.parametrize("name", ["macroatom_vpackets", "flat_shell"])
def test_oracle_velocity_gradient_equals_jitclass(name):
    from oracle import nonhomologous_oracle

    model, _, _ = mk.case_inputs(name)
    np.testing.assert_array_equal(nonhomologous_oracle.velocity_gradient(model), golden(name)["velocity_gradient"])


def test_synthetic_velocities_decelerate_somewhere():
    from tardis_b200 import synthetic

    base = synthetic.make_model(20, 1000)
    m = synthetic.make_nonhomologous_velocities(base, 0.08)
    assert np.array_equal(m.r_inner, base.r_inner) and np.any(m.v_outer < m.v_inner)
    assert m.v_inner[0] == base.v_inner[0] and m.v_outer[-1] == base.v_outer[-1]
    assert np.array_equal(m.v_inner[1:], m.v_outer[:-1])
    m2 = synthetic.make_nonhomologous_velocities(base, 0.08)
    assert np.array_equal(m.v_inner, m2.v_inner)


def test_oracle_matches_reference_bench_shape():
    """The bench's shape (5e5 lines, 20 shells, macroatom, 1000 packets, perturbed velocities).  One packet forks: packet
    489, whose trace about ten events in ends at line 268031 in shell 3 on the oracle and in an electron scattering in shell
    4 on the reference -- a decision that the quartic's conditioning (up to ~1e-4 relative in a root between the reference's
    fastmath evaluation and the IEEE one, test_header_matches_reference_distance) can tip either way.  Every other packet
    agrees: integers identical, floats within FLOAT_BAR.  The estimators carry the forked packet's path (J differs by 0.3 %),
    so they are checked against the reference in the six small cases only, where no packet forks."""
    from oracle import nonhomologous_oracle

    forked = [489]
    model, packets, kw = mk.case_inputs("bench_shape")
    g = golden("bench_shape")
    got = nonhomologous_oracle.run_oracle(model, packets, **kw)
    differs = np.zeros(len(packets), dtype=bool)
    for k in INT_KEYS:
        differs |= got[k] != g[k]
    assert list(np.nonzero(differs)[0]) == forked
    ok = ~differs
    np.testing.assert_array_equal(np.sign(got["output_energies"]), np.sign(g["output_energies"]))
    for k in ("output_nus", "output_energies", "last_radius", "last_before_nu", "last_before_mu", "last_before_energy",
              "last_after_nu", "last_after_mu", "last_after_energy"):
        np.testing.assert_allclose(got[k][ok], g[k][ok], rtol=FLOAT_BAR, atol=0, equal_nan=True, err_msg=k)


@pytest.mark.parametrize("name", list(mk.RADFIELD_CASES))
def test_radfield_oracle_matches_reference_golden(name):
    """The nonhomologous radiation-field solve (J_blue normalised by (c / dvdr) / (4 pi t_sim V)); the flat shell has
    dvdr = 0, so its normalisation is infinite and its untouched cells NaN, as in the reference."""
    from oracle import nonhomologous_oracle

    g = golden(name)
    t, w, jb = nonhomologous_oracle.solve_radiation_field(**mk.radfield_inputs(name))
    np.testing.assert_allclose(t, g["t_radiative"], rtol=1e-14, atol=0)
    np.testing.assert_allclose(w, g["dilution_factor"], rtol=1e-14, atol=0)
    np.testing.assert_allclose(jb, g["j_blues"], rtol=1e-13, atol=0, equal_nan=True)


def test_mirror_keeps_reference_parameters():
    """Every positional parameter of the reference's nonhomologous solver, state and radiation-field solver, same name,
    same order (parsed from the reference's sources into tests/golden/reference_interface_nonhomologous.json)."""
    import inspect
    import json

    from tardis_b200 import montecarlo as mc

    sigs = json.load(open(os.path.join(GOLDEN, "reference_interface_nonhomologous.json")))["signatures"]
    mirrors = {
        "MCTransportSolverNonhomologous": mc.MCTransportSolverB200Nonhomologous,
        "MonteCarloTransportStateNonhomologous": mc.MonteCarloTransportStateB200Nonhomologous,
        "MCRadiationFieldPropertiesSolver": mc.MCRadiationFieldPropertiesSolverB200Nonhomologous,
    }
    assert len(sigs) == 8
    for key, ref in sigs.items():
        cls, fn = key.split("::", 1)[1].split(".")
        obj = getattr(mirrors[cls], fn)
        mine = [n for n, p in inspect.signature(obj).parameters.items()
                if n not in ("self", "cls") and p.kind in (p.POSITIONAL_ONLY, p.POSITIONAL_OR_KEYWORD)]
        assert mine[:len(ref)] == ref, (key, ref, mine)


def test_host_refusals():
    """Refused in Python before the engine is reached: full relativity (the reference's NotImplementedError), continuum
    processes, missing velocities."""
    from tardis_b200.engine import Engine

    model, _, _ = mk.case_inputs("scatter")
    eng = object.__new__(Engine)  # no device: the checks come before any engine call
    base = dict(r_inner=model.r_inner, r_outer=model.r_outer, time_explosion=0.0, electron_density=model.electron_density,
                line_list_nu=model.line_list_nu, tau_sobolev=model.tau_sobolev, nonhomologous=True)
    with pytest.raises(NotImplementedError, match="Full relativity not supported for non-homology."):
        Engine.set_model(eng, **base, v_inner=model.v_inner, v_outer=model.v_outer, enable_full_relativity=True)
    with pytest.raises(ValueError, match="continuum processes"):
        Engine.set_model(eng, **base, v_inner=model.v_inner, v_outer=model.v_outer, continuum=object())
    with pytest.raises(ValueError, match="v_inner and v_outer"):
        Engine.set_model(eng, **base)


def test_transport_dispatches_on_the_geometry_carrier():
    """montecarlo_transport_with_vpackets selects the mode from the geometry: a per-shell velocity_gradient
    (NumbaRadial1DGeometry) means nonhomologous, the scalar 1 / t_exp (NumbaHomologousRadial1DGeometry) homologous."""
    from types import SimpleNamespace

    from tardis_b200 import montecarlo as mc

    model, packets, _ = mk.case_inputs("scatter")

    class Stop(Exception):
        pass

    class Recorder:
        def set_model(self, **kw):
            self.kw = kw
            raise Stop

    mac = model.macro
    opacity = SimpleNamespace(electron_density=model.electron_density, line_list_nu=model.line_list_nu,
                              tau_sobolev=model.tau_sobolev, transition_probabilities=mac.transition_probabilities,
                              line2macro_level_upper=mac.line2macro_level_upper, macro_block_edge_index=mac.macro_block_edge_index,
                              transition_type=mac.transition_type, destination_level_id=mac.destination_level_id,
                              transition_line_id=mac.transition_line_id)
    cfg = mc.MonteCarloConfiguration()
    nonhom = SimpleNamespace(r_inner=model.r_inner, r_outer=model.r_outer, v_inner=model.v_inner, v_outer=model.v_outer,
                             velocity_gradient=(model.v_outer - model.v_inner) / (model.r_outer - model.r_inner))
    homol = mc.HomologousGeometry(model.r_inner, model.r_outer, model.v_inner, model.v_outer, model.time_explosion)
    for geo, want in ((nonhom, True), (homol, False)):
        rec = Recorder()
        with pytest.raises(Stop):
            mc.montecarlo_transport_with_vpackets(None, geo, 0.0, opacity, cfg, model.spectrum_frequency_grid, None, 0,
                                                  engine=rec)
        assert rec.kw["nonhomologous"] is want
        if want:
            np.testing.assert_array_equal(rec.kw["v_inner"], model.v_inner)
