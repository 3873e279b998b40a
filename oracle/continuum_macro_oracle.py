"""CPU restatement of the continuum (IIP) macro atom's per-iteration rows and their normalisation.

TEST INFRASTRUCTURE ONLY.  numpy restatement of, paths relative to /root/reference/tardis/:
    the continuum rows of ContinuumMacroAtomSolver._solve_next_macroatom_iteration
                                        opacities/macro_atom/macroatom_solver.py:1533-1631, macroatom_continuum_transitions.py
    normalize_cooling_block_by_rate_fractions (existing cooling block)   macroatom_solver.py:1817-1833
    normalize_transition_probabilities  macroatom_solver.py:709-739 (pandas' group_sum: Kahan, NaN addends skipped)
The line rows are oracle/opacity_oracle.py's.  Which table row and energy a continuum row reads comes from the row map
(tardis_b200.macro_atom.continuum_row_map), pinned against the reference by tests/golden/continuum_macro_*.npz."""
from __future__ import annotations

import numpy as np

from oracle import opacity_oracle as oo

RATE_TYPES = {2: 0, 3: 1, -7: 1, 11: 2, 5: 2, 4: 3, 6: 4, 7: 5, 14: 5}
COOL_TYPES = {-20: ("fb_cool_rate", 0), 21: ("coll_exc_cool_rate", 1), 22: ("coll_ion_cool_rate", 2)}


def raw_rows(atomic, transition_type, transition_line_idx, row_map, rates, beta, stim, j_blues):
    """[T, S] unnormalised probabilities.  `atomic`: synthetic.AtomicData of the line list; `rates`: the dict of
    tardis_b200.macro_atom.continuum_rates."""
    tt = np.asarray(transition_type)
    T, S = len(tt), beta.shape[1]
    nu = atomic.nu[:, None]
    e_lower = atomic.energy[atomic.lower_level][:, None]
    e_upper = atomic.energy[atomic.upper_level][:, None]
    f_ul, f_lu, C, H, CE = atomic.f_ul[:, None], atomic.f_lu[:, None], oo.C, oo.H, oo.C_EINSTEIN
    line = {-1: beta * (2 * nu**2 * f_ul / C**2 * (e_upper - e_lower)) * CE,
            0: beta * (2 * nu**2 * f_ul / C**2 * e_lower) * CE,
            1: beta * (f_lu / (H * nu) * stim * j_blues * e_lower) * CE}
    out = np.zeros((T, S))
    key, energy, n_e = row_map["rate_key"], row_map["energy"], rates["electron_densities"]
    with np.errstate(invalid="ignore", over="ignore"):
        for t, p in line.items():
            rows = np.flatnonzero(tt == t)
            out[rows] = p[transition_line_idx[rows]]
        for t, k in RATE_TYPES.items():
            rows = np.flatnonzero(tt == t)
            r = rates["rate"][k][key[rows]]
            out[rows] = r * energy[rows, None] if t in (2, 3, -7) else (r * n_e) * energy[rows, None]
        out[tt == -21] = rates["ff_cool_rate"]
        for t, (rate, k) in COOL_TYPES.items():
            rows = np.flatnonzero(tt == t)
            out[rows] = rates[rate] * rates["cooling"][k][key[rows]]
    return out


def group_sums(p, edges):
    """pandas' group_sum per source block: Kahan in row order, NaN addends skipped, a NaN compensation reset"""
    sums = np.zeros((len(edges) - 1, p.shape[1]))
    for b in range(len(edges) - 1):
        s, c = np.zeros(p.shape[1]), np.zeros(p.shape[1])
        for t in range(edges[b], edges[b + 1]):
            v = p[t]
            ok = ~np.isnan(v)
            with np.errstate(invalid="ignore"):
                y = v - c
                u = s + y
                cn = (u - s) - y
            cn[np.isnan(cn)] = 0.0
            s, c = np.where(ok, u, s), np.where(ok, cn, c)
        sums[b] = s
    return sums


def normalize(p, edges):
    """probabilities / group sum, NaN -> 0"""
    block = np.repeat(np.arange(len(edges) - 1), np.diff(edges))
    with np.errstate(divide="ignore", invalid="ignore"):
        q = p / group_sums(p, edges)[block]
    q[np.isnan(q)] = 0.0
    return q
