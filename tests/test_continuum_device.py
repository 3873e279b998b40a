"""The continuum (IIP) mode's bound-free opacity, bound-free estimators and continuum draw, against exact arithmetic.

What is pinned, on tables built here to be hard for the global bins of csrc/continuum_bins.cuh (`adversarial_blocks`):
breakpoint values shared between blocks (one block's first point is another's interior point), a 2-point block, nested
and overlapping blocks, 150 breakpoints inside one guide key (GUIDE_SHIFT = 44), a block over four octaves, chi_bf exactly
0 at some points, and an interval across which x_sect falls by 1e6 while chi_bf falls to 0.

* CPU, through tests/continuum_device_shim.cpp (the header the kernels compile): frequencies at, and 1..6 ulps around,
  every breakpoint (so every pi_min, pi_max, B[0] and B[-1]) and random ones.  The tie flag must be exactly
  "nu is a breakpoint", the bin exactly searchsorted(B, nu), the statistics exact, untouched cells exactly 0.0.
* CPU: packets that never interact, run through the oracle, give the exact sums below (this pins the restatement of
  the traces the GPU tests rely on).
* GPU: the same packets through the pooled, lane-resident and scan continuum kernels, through a table without the block
  structure (every trace on the literal path), through an engine group [0, 0] and through two transports accumulated
  with zero_estimators = 0.  Statistics and counters exact, zero cells exactly 0.0, f64 estimators within the bars.
* The continuum draw: packets whose first trace starts where chi_bf cancels inside a bin, with seeds whose continuum
  draw (draw 4 of the packet: tau_event, the e-scattering test, mu, the bound-free test, z) falls where the trace's
  bins value and the literal sum disagree.  The kernels must select the reference's continuum: counters, last-
  interaction columns and event logs exactly the oracle's.

Exact values: every term of the reference's literal formulas (update_estimators_bound_free,
radfield_estimator_calcs.py:57-124, and chi_continuum_calculator, opacities.py:139-172) is evaluated exactly with
Fraction from the fp64 inputs of its trace (comoving nu, comoving energy, comoving distance, the fp64 Boltzmann
factor).  Sums are kept as integers in units of 2^-(F - e_max), F = 240, which is exact to far below any bar.

Bars (u = 2^-53), derived from the expressions the kernels evaluate, not a flat rtol:
  |value - exact| <= (C_TERM + n_add) * u * A
where A is the sum, over every term the kernel's expression adds, of the absolute values of that term's products
(bins path, per (shell, bin) cell and continuum interval:  |X| M1 + |b| M2  for photo_ion,
|e X| M1 + (|X| + |e b|) M2 + |b| M3  for bf_heating, the same on the Boltzmann-weighted moments for the stimulated
pair; literal path, per trace:  |E d xs / nu|  and  |E d xs| (1 + thr / nu);  chi_bf_tot:  the interpolation products
and |D| dl), n_add is the number of additions that build the value (traces into a cell, cells and literal traces into
an estimator), C_TERM = 16 covers the roundings inside one term (at most 10: u, dl, the interpolation, the products),
and on the GPU C_INPUT = 8 more covers the trace inputs being recomputed here with the oracle's formulas rather than
read back from the device (each can differ by an ulp).  Observed distances are reported in DESIGN section 2.
"""
from __future__ import annotations

import atexit
import copy
import ctypes as C
import functools
import math
import os
import shutil
import subprocess
import tempfile
from fractions import Fraction

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
H, KB = 6.62606957e-27, 1.3806488e-16           # the oracle's and the kernels' CODATA-2010 cgs constants
M_EL, E_ESU, C_LIGHT = 9.10938291e-28, 4.80320425e-10, 2.99792458e10
FF_OPAC_CONST = math.pow(2 * math.pi / (3 * M_EL * KB), 0.5) * 4 * math.pow(E_ESU, 6) / (3 * M_EL * H * C_LIGHT)
GUIDE_SHIFT = 44
U = 2.0 ** -53
C_TERM, C_INPUT = 16, 8
F_BITS = 240
ULPS = tuple(k for k in range(-6, 7))
TRACE_KEYS = ("shell", "nu", "energy", "distance")


def _bits(x: float) -> int:
    return int(np.float64(x).view(np.int64))


def _from_bits(b: int) -> float:
    return float(np.int64(b).view(np.float64))


def _step(x: float, k: int) -> float:
    return _from_bits(_bits(x) + k)


@functools.lru_cache(maxsize=None)
def _oracle():
    from oracle import cpu_oracle

    cpu_oracle.build()
    return cpu_oracle


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


@functools.lru_cache(maxsize=None)
def _shim_lib():
    """tests/continuum_device_shim.cpp (tests/continuum_bins_shim.cpp plus the per-bin active lists), compiled as
    test_continuum_bins.py compiles its shim."""
    src = os.path.join(HERE, "continuum_device_shim.cpp")
    deps = [src, os.path.join(HERE, "continuum_bins_shim.cpp"), os.path.join(ROOT, "tardis_b200", "csrc", "continuum_bins.cuh")]
    out = os.path.join(_shim_dir(), "libcontinuum_device_shim.so")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in deps):
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", out, src], check=True)
    lib = C.CDLL(out)
    lib.shim_continuum_bins.restype = C.c_int
    lib.shim_continuum_bins.argtypes = [C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 8 + [C.c_longlong] + [C.c_void_p] * 8
    lib.shim_bin_actives.restype = C.c_longlong
    lib.shim_bin_actives.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 6 + [C.c_longlong]
    return lib


@pytest.fixture(scope="module")
def shim():
    return _shim_lib()


def run_shim(shim, cont, t_e, tr):
    nc, S, n_phot = len(cont.bf_threshold_list_nu), cont.chi_bf.shape[1], len(cont.phot_nus)
    n = len(tr["nu"])
    chi, tie, bins = np.zeros(n), np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.int32)
    est = np.zeros((5, nc, S))
    arrs = [np.ascontiguousarray(a) for a in (cont.phot_nus, cont.photo_ion_block_references.astype(np.int64),
                                              cont.photo_ion_nu_threshold_mins, cont.photo_ion_nu_threshold_maxs, cont.x_sect,
                                              cont.chi_bf, cont.bf_threshold_list_nu, t_e)]
    t = [np.ascontiguousarray(tr[k], dtype=np.int64 if k == "shell" else np.float64) for k in ("nu", "energy", "distance", "shell")]
    rc = shim.shim_continuum_bins(n_phot, nc, S, *(a.ctypes.data for a in arrs), n, *(a.ctypes.data for a in t),
                                  chi.ctypes.data, tie.ctypes.data, bins.ctypes.data, est.ctypes.data)
    assert rc == 0
    return chi, tie, bins, est


# ---------------------------------------------------------------------------------------------------------------------
# Adversarial tables
# ---------------------------------------------------------------------------------------------------------------------
def dense_key_points(nu: float, n: int) -> np.ndarray:
    """n ascending frequencies inside the guide key of nu."""
    key = _bits(nu) >> GUIDE_SHIFT
    offs = np.linspace(1, (1 << GUIDE_SHIFT) - 2, n).astype(np.int64)
    return np.array([_from_bits(int((key << GUIDE_SHIFT) + o)) for o in offs])


def adversarial_blocks():
    """[(phot_nus, x_sect, chi_bf shape factors)] per continuum, in continuum order (see the module docstring)."""
    octaves = np.geomspace(3e14, 5e15, 10)
    b1 = np.unique(np.concatenate([octaves, [1.0e15, 1.2e15, 1.7e15]]))
    blocks = [
        np.array([1.0e15, 1.7e15]),                      # 2-point block; its first point is an interior point of b1
        b1,                                              # four octaves, sharing 1e15, 1.2e15, 1.7e15 and 5e15
        np.array([1.2e15, 1.3e15, 1.45e15, 1.7e15]),     # nested in b1, first and last point shared with b1
        np.array([4.0e15, 4.5e15, 5.0e15, 7.0e15, 9.0e15]),  # overlaps b1's upper end, shares its last point
        dense_key_points(2.5e15, 150),                   # 150 breakpoints inside one guide key
        np.array([6.0e14, 6.5e14]),                      # a plain 2-point block
    ]
    out = []
    for k, nus in enumerate(blocks):
        xs = 3e-18 * (nus[0] / nus) ** 3
        shape = np.ones(len(nus))
        if k == 0:
            xs = np.array([2e-17, 2e-23])                # x_sect falls by 1e6 across the interval
            shape = np.array([1.0, 0.0])                 # chi_bf falls to exactly 0: C + D dl cancels near 1.7e15
        if k == 1:
            shape[np.searchsorted(nus, 1.2e15)] = 0.0    # chi_bf exactly 0 at an interior point
        if k == 3:
            shape[0] = 0.0                               # and at a block's first point
        out.append((nus, xs, shape))
    return out


def continuum_tables(blocks, n_shells, chi_scale, seed, ff_factor):
    """synthetic.ContinuumTables for `blocks` (reference layouts); chi_bf = x_sect * shape * level density."""
    from tardis_b200 import synthetic as syn

    rng = np.random.default_rng(seed)
    counts = [len(b[0]) for b in blocks]
    refs = np.zeros(len(blocks) + 1, dtype=np.int64)
    refs[1:] = np.cumsum(counts)
    phot_nus = np.concatenate([b[0] for b in blocks])
    x_sect = np.concatenate([b[1] for b in blocks])
    chi = np.concatenate([(b[1] * b[2])[:, None] * (10 ** rng.uniform(2, 5, (1, n_shells))) for b in blocks]) * chi_scale
    em = np.empty((len(phot_nus), n_shells))
    for k in range(len(blocks)):
        w = rng.random((counts[k], n_shells)) + 0.05
        w[0] = 0.0
        c = np.cumsum(w, axis=0)
        em[refs[k]:refs[k + 1]] = c / c[-1]
    return syn.ContinuumTables(
        bf_threshold_list_nu=phot_nus[refs[:-1]].copy(), p_fb_deactivation=np.full((len(blocks), n_shells), 1.0 / len(blocks)),
        photo_ion_nu_threshold_mins=phot_nus[refs[:-1]].copy(), photo_ion_nu_threshold_maxs=phot_nus[refs[1:] - 1].copy(),
        photo_ion_block_references=refs, chi_bf=np.ascontiguousarray(chi), x_sect=x_sect, phot_nus=phot_nus,
        ff_opacity_factor=np.full(n_shells, ff_factor), emissivities=np.ascontiguousarray(em),
        photo_ion_activation_idx=np.full(30, 0, dtype=np.int64), k_packet_idx=0, absorbing_markov_probabilities=None)


def iip_model(n_shells, n_continua, seed):
    """A synthetic IIP model (macro atom of add_continuum with n_continua continua), its continuum tables to be replaced."""
    from tardis_b200 import synthetic as syn

    model = syn.make_model(n_shells, 60, "macroatom", seed=seed, duplicate_fraction=0.0)
    syn.add_continuum(model, seed=seed + 1, n_continua=n_continua, points=(2, 4))
    return model


def with_tables(model, cont):
    m = copy.copy(model)
    c = copy.copy(cont)
    old = model.continuum
    c.photo_ion_activation_idx, c.k_packet_idx = old.photo_ion_activation_idx, old.k_packet_idx
    c.absorbing_markov_probabilities = old.absorbing_markov_probabilities
    m.continuum = c
    return m


# ---------------------------------------------------------------------------------------------------------------------
# Exact literal values and bars
# ---------------------------------------------------------------------------------------------------------------------
def boltzmann(nu, t):
    return math.exp(-(H * nu) / (KB * t))


def active_interps(cont, nu):
    """[(k, lo, hi)] of the continua active at nu, with the reference's searchsorted and [-1] wrap."""
    refs, pn = cont.photo_ion_block_references, cont.phot_nus
    out = []
    for k in range(len(refs) - 1):
        if cont.photo_ion_nu_threshold_mins[k] <= nu <= cont.photo_ion_nu_threshold_maxs[k]:
            a, b = int(refs[k]), int(refs[k + 1])
            idx = int(np.searchsorted(pn[a:b], nu, side="left"))
            assert idx < b - a
            out.append((k, a + (idx - 1 if idx > 0 else b - a - 1), a + idx))
    return out


def literal_fp64_chi(cont, nu, shell):
    """chi_bf_literal / chi_continuum_calculator in fp64, in continuum order -> list of running sums."""
    pn, chi = cont.phot_nus, cont.chi_bf
    running, out = 0.0, []
    for k, lo, hi in active_interps(cont, nu):
        hw, lw = nu - pn[lo], pn[hi] - nu
        running += (chi[hi, shell] * hw + chi[lo, shell] * lw) / (pn[hi] - pn[lo])
        out.append(running)
    return out


def exact_chi(cont, nu, shell):
    pn, chi = cont.phot_nus, cont.chi_bf
    tot = Fraction(0)
    for k, lo, hi in active_interps(cont, nu):
        f = Fraction(nu)
        tot += (Fraction(chi[hi, shell]) * (f - Fraction(pn[lo])) + Fraction(chi[lo, shell]) * (Fraction(pn[hi]) - f)) \
            / (Fraction(pn[hi]) - Fraction(pn[lo]))
    return tot


class Exact:
    """Exact literal sums of the five estimators and ff_heating over a list of traces, with the bars of the module
    docstring for the bins path (ties and n_active = 0 traces excepted) or the literal path."""

    def __init__(self, cont, t_e, ff_factor, tr, literal_everywhere=False):
        nc, S = len(cont.bf_threshold_list_nu), len(t_e)
        refs, pn, xs_t = cont.photo_ion_block_references, cont.phot_nus, cont.x_sect
        order = np.argsort(pn, kind="stable")
        B = pn[order]
        pos = np.empty(len(pn), dtype=np.int64)
        pos[order] = np.arange(len(pn))
        self.terms = [[[[] for _ in range(S)] for _ in range(nc)] for _ in range(5)]
        self.counts = np.zeros((nc, S), dtype=np.int64)
        self.abs_lit = np.zeros((4, nc, S))
        self.n_add = np.zeros((nc, S), dtype=np.int64)
        self.ff_terms = [[] for _ in range(S)]
        self.ff_abs = np.zeros(S)
        self.n_ff = np.zeros(S, dtype=np.int64)
        mom = {}
        dops = tr.get("dop", np.ones(len(tr["nu"])))
        for s, nu, e, d, dop in zip(*(tr[k] for k in TRACE_KEYS), dops):
            s = int(s)
            bz = boltzmann(nu, t_e[s])
            chi_ff = FF_OPAC_CONST * ff_factor[s] / (nu * nu * nu) * (1 - bz) * dop  # the lab-frame chi_ff, times dop
            self.ff_terms[s].append(Fraction(e) * Fraction(d) * Fraction(chi_ff))
            self.ff_abs[s] += abs(e * d * chi_ff) * (1 + abs(bz) / max(abs(1 - bz), 1e-300))
            self.n_ff[s] += 1
            acts = active_interps(cont, nu)
            g = int(np.searchsorted(B, nu, side="left"))
            tie = g < len(B) and B[g] == nu
            bins = not (tie or literal_everywhere)
            fe, fd, fn, fb = Fraction(e), Fraction(d), Fraction(nu), Fraction(bz)
            for k, lo, hi in acts:
                interval = Fraction(pn[hi]) - Fraction(pn[lo])
                xs = (Fraction(xs_t[hi]) * (fn - Fraction(pn[lo])) + Fraction(xs_t[lo]) * (Fraction(pn[hi]) - fn)) / interval
                inc = fe * fd * xs / fn
                bfh = fe * fd * xs * (1 - Fraction(cont.bf_threshold_list_nu[k]) / fn)
                for q, v in enumerate((inc, inc * fb, bfh, bfh * fb)):
                    self.terms[q][k][s].append(v)
                self.counts[k, s] += 1
                self.n_add[k, s] += 1
                if not bins:
                    fx = float(xs)
                    a_inc = abs(e * d * fx / nu)
                    a_bfh = abs(e * d * fx) * (1 + cont.bf_threshold_list_nu[k] / nu)
                    self.abs_lit[:, k, s] += (a_inc, a_inc * bz, a_bfh, a_bfh * bz)
            if bins and acts:
                uu = e * d / nu
                dl = nu - B[g - 1]
                m = mom.setdefault((s, g), np.zeros(7))
                m += (1.0, uu, uu * dl, uu * dl * dl, uu * bz, uu * bz * dl, uu * bz * dl * dl)
        # bins path: per (shell, bin) cell and continuum interval, the products of continuum_estimators_from_moments
        for (s, g), m in mom.items():
            nu_g = B[g - 1]
            for k in range(nc):
                a, b = int(refs[k]), int(refs[k + 1])
                for lo in range(a, b - 1):
                    hi = lo + 1
                    if not (pos[lo] + 1 <= g <= pos[hi]):
                        continue
                    interval = pn[hi] - pn[lo]
                    X = (xs_t[hi] * (nu_g - pn[lo]) + xs_t[lo] * (pn[hi] - nu_g)) / interval
                    bb = (xs_t[hi] - xs_t[lo]) / interval
                    ee = nu_g - cont.bf_threshold_list_nu[k]
                    for q, (m1, m2, m3) in ((0, m[1:4]), (1, m[4:7])):
                        self.abs_lit[q, k, s] += abs(X) * m1 + abs(bb) * m2
                        self.abs_lit[q + 2, k, s] += abs(ee * X) * m1 + (abs(X) + abs(ee * bb)) * m2 + abs(bb) * m3
                    self.n_add[k, s] += 1

    @staticmethod
    def fixed_sum(terms):
        """sum(terms) as a float, exact to 2^-F_BITS of the largest term."""
        if not terms:
            return 0.0
        e = max(math.frexp(float(abs(t)))[1] for t in terms)
        sh = F_BITS - e
        acc = 0
        for t in terms:
            num, den = (t.numerator << sh, t.denominator) if sh >= 0 else (t.numerator, t.denominator << -sh)
            acc += (2 * num + den) // (2 * den)
        return float(Fraction(acc, 1 << sh) if sh >= 0 else Fraction(acc << -sh))

    @functools.cached_property
    def values(self):
        nc, S = self.counts.shape
        out = np.zeros((4, nc, S))
        for q in range(4):
            for k in range(nc):
                for s in range(S):
                    out[q, k, s] = self.fixed_sum(self.terms[q][k][s])
        return out

    @functools.cached_property
    def ff_heating(self):
        return np.array([self.fixed_sum(t) for t in self.ff_terms])

    def check(self, res, c_term, what):
        """Statistics exact, zero cells exactly 0.0, the f64 estimators within their bars; -> max distance in bars."""
        names = ("photo_ion_estimator", "stim_recomb_estimator", "bf_heating_estimator", "stim_recomb_cooling_estimator")
        assert np.array_equal(res["photo_ion_estimator_statistics"], self.counts), what
        worst = 0.0
        for q, name in enumerate(names):
            got = res[name]
            zero = self.counts == 0
            assert (got[zero] == 0.0).all(), (what, name, "untouched cells")
            bar = (c_term + self.n_add) * U * self.abs_lit[q]
            err = np.abs(got - self.values[q])
            assert (err <= bar).all(), (what, name, np.argwhere(err > bar)[:5], err[err > bar][:5], bar[err > bar][:5])
            worst = max(worst, float(np.max(np.where(zero, 0.0, err / np.where(bar > 0, bar, 1.0)))))
        if "ff_heating_estimator" in res:
            ffb = (c_term + self.n_ff) * U * self.ff_abs
            ffe = np.abs(res["ff_heating_estimator"] - self.ff_heating)
            assert (ffe <= ffb).all(), (what, "ff_heating", ffe, ffb)
            assert ((res["ff_heating_estimator"] == 0.0) == (self.n_ff == 0)).all(), (what, "ff_heating zero cells")
        return worst


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the shim on every breakpoint and around it
# ---------------------------------------------------------------------------------------------------------------------
def _shim_workload(seed=7101, n_shells=3):
    cont = continuum_tables(adversarial_blocks(), n_shells, 1e-3, seed, 1e20)
    t_e = np.array([6e3, 1.1e4, 2.3e4])[:n_shells]
    B = np.unique(cont.phot_nus)
    rng = np.random.default_rng(seed)
    nu = np.concatenate([[_step(b, k) for b in B for k in ULPS],
                         np.exp(rng.uniform(np.log(2e14), np.log(1.2e16), 3000)),
                         np.geomspace(2.49e15, 2.52e15, 500)])  # through the dense guide key
    n = len(nu)
    tr = dict(shell=rng.integers(0, n_shells, n), nu=nu, energy=rng.uniform(0.5, 2.0, n) / n,
              distance=10 ** rng.uniform(12, 15, n))
    return cont, t_e, B, tr


def test_adversarial_tables_have_the_advertised_structure(shim):
    cont, t_e, B, tr = _shim_workload()
    pn, refs = cont.phot_nus, cont.photo_ion_block_references
    blocks = [pn[refs[k]:refs[k + 1]] for k in range(len(refs) - 1)]
    assert len(B) < len(pn)                                              # shared breakpoint values
    assert blocks[0][0] in blocks[1][1:-1] and blocks[2][0] in blocks[1][1:-1]
    assert min(len(b) for b in blocks) == 2
    assert blocks[1][0] < blocks[2][0] and blocks[2][-1] < blocks[1][-1]  # nested
    assert blocks[1][0] < blocks[3][0] < blocks[1][-1] < blocks[3][-1]    # overlapping
    keys = np.array([_bits(x) >> GUIDE_SHIFT for x in pn])
    assert np.bincount(keys - keys.min()).max() > 100
    assert blocks[1][-1] / blocks[1][0] > 16
    assert (cont.chi_bf == 0.0).any(axis=1).sum() >= 3
    assert (cont.x_sect[refs[0]] / cont.x_sect[refs[0] + 1]) >= 1e6
    _, tie, _, _ = run_shim(shim, cont, t_e, tr)                         # build_bins accepts it (rc == 0)
    assert tie.sum() == len(B)


def test_bins_match_exact_literal_values(shim):
    """Tie flags, bins, chi_bf_tot and the five estimators of the shim against the exact literal values."""
    cont, t_e, B, tr = _shim_workload()
    chi, tie, bins, est = run_shim(shim, cont, t_e, tr)
    nu = tr["nu"]
    assert np.array_equal(tie == 1, np.isin(nu, B))
    B = np.sort(cont.phot_nus)  # the kernels' B keeps the duplicates
    assert np.array_equal(bins, np.searchsorted(B, nu, side="left"))
    # chi_bf_tot of the bins path (ties go to the literal path and are not evaluated from the bins)
    worst = 0.0
    for i in np.flatnonzero(tie == 0):
        s, g = int(tr["shell"][i]), int(bins[i])
        acts = active_interps(cont, nu[i])
        exact = exact_chi(cont, nu[i], s)
        if g == 0 or g == len(B):
            assert chi[i] == 0.0 and not acts
            continue
        nu_g, dl = B[g - 1], nu[i] - B[g - 1]
        pn, cb = cont.phot_nus, cont.chi_bf[:, s]
        a = sum((abs(cb[hi]) * (nu_g - pn[lo]) + abs(cb[lo]) * (pn[hi] - nu_g)) / (pn[hi] - pn[lo])
                + (abs(cb[hi]) + abs(cb[lo])) / (pn[hi] - pn[lo]) * dl for _, lo, hi in acts)
        bar = (C_TERM + 2 * len(acts)) * U * a
        err = abs(Fraction(chi[i]) - exact)
        assert err <= bar, (i, nu[i], chi[i], float(exact), bar)
        worst = max(worst, float(err) / bar if bar else 0.0)
    # the moments skip ties (the kernels send them to the literal path)
    ex = Exact(cont, t_e, cont.ff_opacity_factor, {k: tr[k][tie == 0] for k in TRACE_KEYS})
    res = {"photo_ion_estimator": est[0], "stim_recomb_estimator": est[1], "bf_heating_estimator": est[2],
           "stim_recomb_cooling_estimator": est[3], "photo_ion_estimator_statistics": est[4].astype(np.int64)}
    assert np.array_equal(est[4], est[4].round())
    worst_est = ex.check(res, C_TERM, "shim")
    print(f"shim: chi_bf_tot worst {worst:.3g} bars, estimators worst {worst_est:.3g} bars")


def test_bin_active_lists_are_the_reference_selection(shim):
    """HostBins::act, which the continuum event reads to form the literal sum on the bins path: for every frequency
    strictly inside a bin, its bin's list is the reference's active continua and interpolation intervals, in order."""
    cont, t_e, B, tr = _shim_workload()
    pn, refs = cont.phot_nus, cont.photo_ion_block_references.astype(np.int64)
    act_start = np.zeros(len(pn) + 2, dtype=np.int32)
    act = np.zeros(2 * len(pn) * len(refs), dtype=np.int32)
    n = shim.shim_bin_actives(len(pn), len(refs) - 1, pn.ctypes.data, refs.ctypes.data,
                              np.ascontiguousarray(cont.photo_ion_nu_threshold_mins).ctypes.data,
                              np.ascontiguousarray(cont.photo_ion_nu_threshold_maxs).ctypes.data, act_start.ctypes.data,
                              act.ctypes.data, len(act))
    assert 0 < n <= len(act) and act_start[-1] * 2 == n
    Bs = np.sort(pn)
    inside = tr["nu"][~np.isin(tr["nu"], B)]
    for nu in inside:
        g = int(np.searchsorted(Bs, nu, side="left"))
        lst = act[2 * act_start[g]:2 * act_start[g + 1]].reshape(-1, 2)
        assert [tuple(x) for x in lst] == [(k, lo) for k, lo, hi in active_interps(cont, nu)], nu
        assert all(hi == lo + 1 for _, lo, hi in active_interps(cont, nu))


def test_cancellation_inside_an_interval_is_the_documented_fork(shim):
    """chi_bf 0.1 -> 0 over [1e15, 1.7e15], at 1e-12 of the interval below its top: C + D (nu - B[g-1]) is ~1e-4 off
    the exact value, the literal interpolation ~1e-16.  The trace distance uses the bins value (DESIGN section 2);
    the continuum event uses the literal sum."""
    blocks = [(np.array([1.0e15, 1.7e15]), np.array([1e-17, 1e-18]), np.array([1.0, 0.0]))]
    cont = continuum_tables(blocks, 1, 1.0, 1, 1e20)
    cont.chi_bf = np.array([[0.1], [0.0]])
    nu = 1.7e15 - 1e-12 * 0.7e15
    chi, tie, _, _ = run_shim(shim, cont, np.array([1e4]), dict(shell=[0], nu=[nu], energy=[1.0], distance=[1.0]))
    exact = exact_chi(cont, nu, 0)
    lit = literal_fp64_chi(cont, nu, 0)[-1]
    bins_err = float(abs(Fraction(chi[0]) - exact) / exact)
    lit_err = float(abs(Fraction(lit) - exact) / exact)
    assert tie[0] == 0 and bins_err > 1e-6 and lit_err < 1e-15 and bins_err > 1e8 * lit_err


# ---------------------------------------------------------------------------------------------------------------------
# Packets that never interact: straight flights from r_inner[0] to the outer boundary
# ---------------------------------------------------------------------------------------------------------------------
N_SHELLS_FLIGHT = 4
SIGMA_TINY = 1e-200
OFFSETS = (0, 0, -1, 1)   # breakpoint placed on a first trace, twice as often as one ulp below / above it


def flight_traces(model, packets):
    """Every trace of every packet (IIP propagation: full relativity), restated from the oracle's
    packet_propagation_iip / move_r_packet with its own doppler_factor and distance_boundary."""
    o = _oracle()
    t = model.time_explosion
    out = {k: [] for k in TRACE_KEYS + ("dop", "packet", "index")}
    for i in range(len(packets)):
        r, mu = float(packets.initial_radii[i]), float(packets.initial_mus[i])
        beta = (r / t) / C_LIGHT
        idf = o.inverse_doppler_factor(r / t, mu, True)
        nu, e = float(packets.initial_nus[i]) * idf, float(packets.initial_energies[i]) * idf
        mu = (mu + beta) / (1 + beta * mu)
        s, j = 0, 0
        while s < model.n_shells:
            dop = o.doppler_factor(r / t, mu, True)
            d, delta = o.distance_boundary(r, mu, float(model.r_inner[s]), float(model.r_outer[s]))
            assert delta == 1
            for k, v in zip(TRACE_KEYS + ("dop", "packet", "index"), (s, nu * dop, e * dop, d * dop, dop, i, j)):
                out[k].append(v)
            new_r = math.sqrt(r * r + d * d + 2.0 * r * d * mu)
            mu = (mu * r + d) / new_r
            r = new_r
            s += 1
            j += 1
    return {k: np.array(v) for k, v in out.items()}


@functools.lru_cache(maxsize=None)
def flight_workload(seed=7202, n_random=600):
    """-> (model, packets, traces, exact sums).  The tables are built after the traces: every distinct breakpoint of
    adversarial_blocks() is moved onto the first comoving frequency of its own packet (OFFSETS), and no other trace
    comes within 1e-12 of a breakpoint."""
    from tardis_b200 import synthetic as syn

    S = N_SHELLS_FLIGHT
    model = iip_model(S, 6, seed)
    model.tau_sobolev = np.full_like(model.tau_sobolev, 1e-40)
    rng = np.random.default_rng(seed)
    blocks = adversarial_blocks()
    values = np.unique(np.concatenate([b[0] for b in blocks]))
    nu0 = np.concatenate([values, np.exp(rng.uniform(np.log(2e14), np.log(1.2e16), n_random))])
    n = len(nu0)
    r0 = float(model.r_inner[0])
    packets = syn.Packets(np.full(n, r0), nu0, rng.uniform(0.2, 1.0, n), np.full(n, 1.0 / n),
                          rng.integers(1, 2**32 - 1, n).astype(np.int64), 1.0)
    tr = flight_traces(model, packets)
    first = tr["nu"][tr["index"] == 0]
    moved = {v: _step(first[i], OFFSETS[i % len(OFFSETS)]) for i, v in enumerate(values)}
    placed = [(np.array([moved[x] for x in b[0]]), b[1], b[2]) for b in blocks]
    for p, _, _ in placed:
        assert (np.diff(p) > 0).all()
    cont = continuum_tables(placed, S, 1e-60, seed, 1e-30)
    B = np.unique(cont.phot_nus)
    designated = (tr["index"] == 0) & (tr["packet"] < len(values))
    near = np.abs(tr["nu"][:, None] / B[None, :] - 1).min(axis=1) < 1e-12
    assert not (near & ~designated).any()
    assert np.isin(tr["nu"][designated], B).sum() == sum(OFFSETS[i % len(OFFSETS)] == 0 for i in range(len(values)))
    m = with_tables(model, cont)
    return m, packets, tr, Exact(cont, m.t_electrons, cont.ff_opacity_factor, tr)


def unstructured(model):
    """The same tables with one pi_max lowered by an ulp: build_bins refuses them, every trace takes the literal path."""
    m = copy.copy(model)
    c = copy.copy(model.continuum)
    c.photo_ion_nu_threshold_maxs = c.photo_ion_nu_threshold_maxs.copy()
    c.photo_ion_nu_threshold_maxs[3] = _step(c.photo_ion_nu_threshold_maxs[3], -1)
    m.continuum = c
    return m


@functools.lru_cache(maxsize=None)
def unstructured_workload():
    model, packets, tr, _ = flight_workload()
    m = unstructured(model)
    return m, Exact(m.continuum, m.t_electrons, m.continuum.ff_opacity_factor, tr, literal_everywhere=True)


def assert_no_interaction(res, n_updates, what):
    c = res["counters"]
    for k in ("n_line_events", "n_escat_events", "n_continuum_events"):
        assert c[k] == 0, (what, k, c[k])
    assert c["n_bf_estimator_updates"] == n_updates, (what, c["n_bf_estimator_updates"], n_updates)
    assert (res["output_energies"] > 0).all(), what


def test_straight_flights_restate_the_oracle():
    """The oracle's run of the flight workload: no interaction, and its estimators equal the exact sums over the
    restated traces (literal bars: the oracle adds the reference's terms one by one)."""
    model, packets, tr, ex = flight_workload()
    ref = _oracle().run_oracle(model, packets, sigma_thomson=SIGMA_TINY)
    assert_no_interaction(ref, int(ex.counts.sum()), "oracle")
    lit = Exact(model.continuum, model.t_electrons, model.continuum.ff_opacity_factor, tr, literal_everywhere=True)
    lit.check(ref, C_TERM, "oracle")
    assert np.isin(tr["nu"], np.unique(model.continuum.phot_nus)).sum() >= 80  # traces exactly on a breakpoint


def engine_run(model, packets, options, group=None):
    from tardis_b200.engine import Engine, EngineGroup

    eng = EngineGroup(group) if group else Engine(0)
    try:
        for k, v in options.items():
            eng.set_option(k, v)
        eng.set_model_from(model, sigma_thomson=SIGMA_TINY)
        return eng.run_packets(packets)
    finally:
        eng.close()


KERNELS = {"pooled": {"algorithm": 1, "pooled": 1}, "lane": {"algorithm": 1, "pooled": 0}, "scan": {"algorithm": 0}}


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", list(KERNELS))
def test_straight_flights_match_exact_sums(kernel):
    model, packets, tr, ex = flight_workload()
    res = engine_run(model, packets, KERNELS[kernel])
    assert_no_interaction(res, int(ex.counts.sum()), kernel)
    worst = ex.check(res, C_TERM + C_INPUT, kernel)
    print(f"{kernel}: worst distance {worst:.3g} bars")


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["pooled", "scan"])
def test_straight_flights_on_the_literal_path_match_exact_sums(kernel):
    _, packets, tr, _ = flight_workload()
    model, ex = unstructured_workload()
    res = engine_run(model, packets, KERNELS[kernel])
    assert_no_interaction(res, int(ex.counts.sum()), kernel)
    worst = ex.check(res, C_TERM + C_INPUT, kernel + " literal")
    print(f"{kernel} literal: worst distance {worst:.3g} bars")


@pytest.mark.gpu
def test_straight_flights_through_an_engine_group():
    model, packets, tr, ex = flight_workload()
    res = engine_run(model, packets, {}, group=[0, 0])
    assert_no_interaction(res, int(ex.counts.sum()), "group")
    ex.check(res, C_TERM + C_INPUT + 1, "group [0, 0]")  # + 1: the members' sums are added once more


@pytest.mark.gpu
def test_straight_flights_accumulated_over_two_transports():
    """The two halves of the packets in two transports, the second with zero_estimators = 0."""
    from tardis_b200.engine import Engine

    model, packets, tr, ex = flight_workload()
    n = len(packets)
    halves = [np.arange(n) < n // 2, np.arange(n) >= n // 2]
    eng = Engine(0)
    try:
        eng.set_model_from(model, sigma_thomson=SIGMA_TINY)
        for h, zero in zip(halves, (True, False)):
            eng.upload_packets(packets.initial_radii[h], packets.initial_nus[h], packets.initial_mus[h],
                               packets.initial_energies[h], packets.packet_seeds[h])
            eng.transport(zero_estimators=zero)
            eng.sync()
        res = eng.download()
    finally:
        eng.close()
    ex.check(res, C_TERM + C_INPUT, "zero_estimators = 0")


# ---------------------------------------------------------------------------------------------------------------------
# The continuum draw where the trace's bins value and the literal sum disagree
# ---------------------------------------------------------------------------------------------------------------------
DRAW_Z = 4   # tau_event, the e-scattering test, mu, the bound-free test, z
DRAW_ION = 5
IT_CONTINUUM_PROCESS = 8


def draw_blocks():
    """Two continua that fall to chi_bf = 0 at a shared top point 1.7e15 (their sum cancels in the bin (1.2e15, 1.7e15]),
    and one that is not active there."""
    return [(np.array([1.0e15, 1.7e15]), np.array([1e-17, 5e-18]), np.array([1.0, 0.0])),
            (np.array([1.2e15, 1.7e15]), np.array([2e-17, 1e-17]), np.array([0.5, 0.0])),
            (np.array([2.0e15, 3.0e15]), np.array([1e-17, 5e-18]), np.array([1.0, 1.0]))]


@functools.lru_cache(maxsize=None)
def draw_workload(seed=7303, n_per_kind=8):
    """-> (model, {kind: (packets, rtol of the event point)}) with kind 'beyond' (z in [sum / bins value, 1): the parent
    found no continuum) and 'between' (z between running_k / bins value and running_k / literal sum: the parent picked
    another continuum).  The first trace's distance tau_event / chi uses the bins value (DESIGN section 2), so the event
    point moves by |bins value / sum - 1| tau_event / sum against the reference's; the rtol is twice that over r."""
    from tardis_b200 import synthetic as syn

    model = iip_model(3, 3, seed)
    model.tau_sobolev = np.full_like(model.tau_sobolev, 1e-40)
    cont = continuum_tables(draw_blocks(), 3, 1.0, seed, 1e-30)
    cont.chi_bf = np.ascontiguousarray(np.repeat(np.array([[1e8], [0.0], [5e7], [0.0], [1e7], [1e7]]), 3, axis=1))
    model = with_tables(model, cont)
    model.continuum.photo_ion_activation_idx = (np.arange(30) * 2 + 1).astype(np.int64)  # a distinct state per continuum
    rng = np.random.default_rng(seed)
    r0, t = float(model.r_inner[0]), model.time_explosion
    o = _oracle()
    beta = (r0 / t) / C_LIGHT
    cands = []
    for j in range(16, 3000):  # first comoving frequencies j ulps below the top point, where C + D dl cancels
        nu0, mu0 = _step(1.7e15, -j), float(rng.uniform(0.3, 1.0))
        mu = (mu0 + beta) / (1 + beta * mu0)
        cands.append((nu0, mu0, (nu0 * o.inverse_doppler_factor(r0 / t, mu0, True)) * o.doppler_factor(r0 / t, mu, True)))
    tr = dict(shell=np.zeros(len(cands), dtype=np.int64), nu=np.array([c[2] for c in cands]),
              energy=np.ones(len(cands)), distance=np.ones(len(cands)))
    chi_bins, tie, _, _ = run_shim(_shim_lib(), cont, model.t_electrons, tr)
    assert not tie.any() and (tr["nu"] < 1.7e15).all()
    runs = [literal_fp64_chi(cont, c[2], 0) for c in cands]
    assert all(len(r) == 2 for r in runs)
    gaps = np.array([cb / r[-1] - 1 for cb, r in zip(chi_bins, runs)])
    kinds = {"beyond": [], "between": []}
    for i in np.argsort(-np.abs(gaps)):
        (nu0, mu0, _), cb, lit = cands[i], chi_bins[i], runs[i][-1]
        gap = [(r / cb, r / lit) for r in runs[i]]  # (the parent's, the reference's) normalised running sums
        taken = {"beyond": 0, "between": 0}
        for seed_ in rng.integers(1, 2**32 - 1, min(100000, int(40 / abs(gaps[i])))):
            z = o.rng_double(int(seed_), DRAW_Z)
            parent = next((k for k, (a, _) in enumerate(gap) if not (a < z)), -1)
            fixed = next(k for k, (_, b) in enumerate(gap) if not (b < z))
            kind = "beyond" if parent < 0 else ("between" if parent != fixed else None)
            if kind and taken[kind] < 2 and len(kinds[kind]) < n_per_kind and o.rng_double(int(seed_), DRAW_ION) < 0.5:
                fork = 2.0 * abs(gaps[i]) * -math.log(o.rng_double(int(seed_), 0)) / lit / r0
                kinds[kind].append((nu0, mu0, int(seed_), fork))
                taken[kind] += 1
        if all(len(v) == n_per_kind for v in kinds.values()):
            break
    out = {}
    for kind, rows in kinds.items():
        assert len(rows) == n_per_kind, (kind, len(rows))
        a = np.array(rows)
        n = len(a)
        out[kind] = (syn.Packets(np.full(n, r0), a[:, 0].copy(), a[:, 1].copy(), np.full(n, 1.0 / n),
                                 np.array([r[2] for r in rows], dtype=np.int64), 1.0), float(a[:, 3].max()))
    return model, out


MAX_EVENTS = 4096


@functools.lru_cache(maxsize=None)
def draw_reference(kind):
    model, packets = draw_workload()
    p, fork = packets[kind]
    ref = _oracle().run_oracle(model, p, sigma_thomson=SIGMA_TINY, n_tracked_packets=len(p), max_events_per_packet=MAX_EVENTS)
    return model, p, ref, fork


@pytest.mark.parametrize("kind", ["beyond", "between"])
def test_draw_seeds_hit_the_gap(kind):
    """Every packet's first event is a continuum event in its first trace, and its draw z lies where a normalisation by
    the bins value finds no continuum ('beyond') or another one than the reference's ('between'): draw_workload picks
    the seeds by that test, here every packet is checked to reach that draw."""
    model, p, ref, fork = draw_reference(kind)
    assert fork < 1e-10  # the per-packet floats stay compared to 1e-10 or better
    assert (ref["event_counts"] < MAX_EVENTS).all()
    first = np.array([(e[1]["interaction_type"], e[1]["before_shell_id"]) for e in ref["events"]])
    assert (first[:, 0] == IT_CONTINUUM_PROCESS).all() and (first[:, 1] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["beyond", "between"])
@pytest.mark.parametrize("kernel", list(KERNELS))
def test_continuum_draw_matches_the_oracle(kernel, kind):
    from golden_util import assert_close
    from tardis_b200.engine import Engine

    model, p, ref, fork = draw_reference(kind)
    eng = Engine(0)
    try:
        for k, v in KERNELS[kernel].items():
            eng.set_option(k, v)
        eng.set_model_from(model, sigma_thomson=SIGMA_TINY)
        res = eng.run_packets(p, track_last_interaction=True, n_tracked_packets=len(p), max_events_per_packet=MAX_EVENTS)
    finally:
        eng.close()
    for k, v in ref["counters"].items():
        assert res["counters"][k] == v, (kernel, kind, k, res["counters"][k], v)
    for k in ("last_interaction_type", "last_event_id", "last_shell_id", "last_line_absorb_id", "last_line_emit_id"):
        assert np.array_equal(res[k], ref[k]), (kernel, kind, k)
    assert np.array_equal(res["event_counts"], ref["event_counts"])
    a, b = np.concatenate(res["events"]), np.concatenate(ref["events"])
    for k in ("packet_id", "interaction_type", "status", "before_shell_id", "after_shell_id", "line_absorb_id", "line_emit_id"):
        assert np.array_equal(a[k], b[k]), (kernel, kind, "event " + k)
    for k in ("output_nus", "output_energies", "last_radius", "last_after_nu", "last_after_energy"):
        assert_close(res[k], ref[k], 1e-11 + fork, f"{kernel} {kind}: {k}")
