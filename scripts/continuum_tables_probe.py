"""Time the continuum (IIP) mode's per-iteration macro-atom tables: built on the device against today's host path.

    python scripts/continuum_tables_probe.py [--shells 50] [--levels 1000] [--repeats 10]
    python scripts/continuum_tables_probe.py --reference [--h-levels 60 --he-levels 40]

GPU mode (default), on one synthetic continuum macro atom of `--levels` levels + a k- and an i-packet state:
  device: tb200_build_opacity (tau / beta / stim, every row, normalisation) + tb200_build_absorbing_markov(NULL);
  host tables: tb200_set_model with the host-built tau and tb200_build_absorbing_markov with the host-built normalised
  [T, S] table (what a continuum iteration uploads today; building those tables on the host is not included).
Both are synchronous calls, timed with a host clock and the median of `--repeats` taken.  The card's name and power
limit are read in the same run.  Writes profiles/continuum_tables_gpu.json.
--reference (where the reference tree exists, no GPU): the unmodified ContinuumMacroAtomSolver's second iteration,
_solve_next_macroatom_iteration, with create_absorbing_probs replaced by a stub returning at once, on
synthetic.make_continuum_rate_inputs; writes profiles/continuum_tables_reference_host.json."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tardis_b200 import synthetic as syn  # noqa: E402


def macro_atom(S, n_levels, n_lines, seed=3):
    """Line rows of synthetic.make_atomic_data plus continuum rows of every kind, grouped by source state; a row map with
    random keys into tables of `n_levels` rows; rates that keep every probability positive and the chain absorbing."""
    rng = np.random.default_rng(seed)
    model = syn.add_continuum(syn.make_model(S, n_lines, "macroatom", seed=seed), seed=seed + 1)
    atomic = syn.make_atomic_data(model.line_list_nu, n_levels, seed=seed + 2)
    k_idx, i_idx = n_levels, n_levels + 1
    blocks = {b: [] for b in range(n_levels + 2)}
    for t, tl in zip(atomic.transition_type, atomic.transition_line_idx):  # states are levels: source / destination by level
        up, lo = int(atomic.upper_level[tl]), int(atomic.lower_level[tl])
        blocks[up if t <= 0 else lo].append((int(t), int(tl), lo if t <= 0 else up))
    lev = lambda: int(rng.integers(0, n_levels))  # noqa: E731
    for b in range(n_levels):
        blocks[b] += [(2, 0, i_idx), (11, 0, k_idx), (5, 0, lev()), (4, 0, lev()), (6, 0, i_idx)]
    blocks[i_idx] = [(3, 0, lev()), (3, 0, lev()), (-7, 0, -1), (-7, 1, -1), (7, 0, lev()), (14, 0, k_idx)]
    blocks[k_idx] = [(-21, 0, -1), (-20, 0, -1), (-20, 1, -1), (21, 0, lev()), (21, 0, lev()), (22, 0, i_idx)]
    rows = [(b, *r) for b in range(n_levels + 2) for r in blocks[b]]
    src = np.array([r[0] for r in rows], dtype=np.int64)
    tt = np.array([r[1] for r in rows], dtype=np.int64)
    tline = np.array([r[2] for r in rows], dtype=np.int64)
    dst = np.where(tt >= 0, np.array([r[3] for r in rows], dtype=np.int64), -1)
    edges = np.concatenate([[0], np.cumsum(np.bincount(src, minlength=n_levels + 2))]).astype(np.int64)
    H = n_levels
    row_map = dict(rate_key=rng.integers(0, H, len(rows)).astype(np.int64), energy=rng.uniform(1e-12, 2e-11, len(rows)),
                   n_rate_rows=[H] * 6, n_cooling_rows=[H] * 3)
    rates = dict(rate=[rng.uniform(0.5, 1.5, (H, S)) * 1e-2 for _ in range(6)], cooling=[rng.uniform(0.5, 1.5, (H, S)) for _ in range(3)],
                 electron_densities=np.full(S, 1e2), **{k: np.full(S, 1e-13) for k in ("ff_cool_rate", "fb_cool_rate",
                                                                                     "coll_exc_cool_rate", "coll_ion_cool_rate")})
    model.macro = syn.MacroAtomTables(None, np.zeros(model.n_lines, dtype=np.int64), edges, tt, dst, tline)
    model.continuum.k_packet_idx, model.continuum.absorbing_markov_probabilities = k_idx, None
    model.continuum.photo_ion_activation_idx = np.full(30, i_idx, dtype=np.int64)
    plasma = syn.make_plasma_state(atomic, S, model.time_explosion, seed=seed + 3, zero_fraction=0.0, inversion_fraction=0.0, noise=0.0)
    return model, atomic, plasma, row_map, rates, dict(source_level_idx=src, destination_level_idx=dst, transition_type=tt)


def gpu(args):
    from tardis_b200.engine import Engine

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    model, atomic, plasma, row_map, rates, chain = macro_atom(args.shells, args.levels, args.lines)
    eng = Engine(0)
    eng.set_option("keep_opacity_tables", 1)
    model.tau_sobolev = None
    eng.set_model_from(model, enable_full_relativity=True)
    eng.set_atomic_data(lines_lower_level_index=atomic.lower_level, lines_upper_level_index=atomic.upper_level, g=atomic.g,
                        metastability=atomic.metastable, wavelength_cm=atomic.wavelength_cm, f_lu=atomic.f_lu, f_ul=atomic.f_ul,
                        energy_lower=atomic.energy[atomic.lower_level], energy_upper=atomic.energy[atomic.upper_level], continuum_rows=row_map)

    def device():
        eng.build_opacity(plasma.level_number_density, plasma.time_explosion, j_blues=plasma.j_blues, continuum=rates)
        eng.build_absorbing_markov(None, **chain)

    device()
    tables = eng.download_opacity(transition_probabilities=True)
    host_model = model
    host_model.tau_sobolev = tables["tau_sobolev"]
    tp = tables["transition_probabilities"]

    def host():
        eng.set_model_from(host_model, enable_full_relativity=True)
        eng.build_absorbing_markov(tp, **chain)

    out = {"card": card, "shells": args.shells, "levels": args.levels, "states": args.levels + 2, "lines": int(model.n_lines),
           "rows": int(len(chain["transition_type"])), "repeats": args.repeats}
    for name, fn in (("host_tables_ms", host), ("device_ms", device)):
        if name == "device_ms":  # the device path needs its model and row map again
            model.tau_sobolev = None
            eng.set_model_from(model, enable_full_relativity=True)
            eng.set_atomic_data(lines_lower_level_index=atomic.lower_level, lines_upper_level_index=atomic.upper_level, g=atomic.g,
                                metastability=atomic.metastable, wavelength_cm=atomic.wavelength_cm, f_lu=atomic.f_lu, f_ul=atomic.f_ul,
                                energy_lower=atomic.energy[atomic.lower_level], energy_upper=atomic.energy[atomic.upper_level],
                                continuum_rows=row_map)
        fn()
        ts = []
        for _ in range(args.repeats):
            t0 = time.perf_counter()
            fn()
            ts.append((time.perf_counter() - t0) * 1e3)
        out[name] = float(np.median(ts))
        out[name + "_all"] = ts
    eng.close()
    return "continuum_tables_gpu.json", out


def reference(args):
    import pandas as pd

    from oracle import reference_runner_continuum_macro as rr

    ms = rr.load_solver_module()
    ci = syn.make_continuum_rate_inputs(args.shells, n_h_levels=args.h_levels, n_he_levels=args.he_levels, seed=11, n_iterations=2)
    solver = ms.ContinuumMacroAtomSolver(ci.levels, ci.lines, ci.photoionization_data, ci.ionization_energies)
    jb, beta, stim = rr.line_inputs(ci, 0)
    solver.solve(jb, beta, stim, **ci.rates[0])
    ms.create_absorbing_probs = lambda tp, md, max_workers=1: (None, tp * 0)
    jb, beta, stim = rr.line_inputs(ci, 1)
    ts = []
    for _ in range(args.repeats):
        t0 = time.perf_counter()
        solver._solve_next_macroatom_iteration(jb, beta, stim, **{k: v for k, v in ci.rates[1].items() if k != "delta_E_yg"})
        ts.append((time.perf_counter() - t0) * 1e3)
    return "continuum_tables_reference_host.json", {"shells": args.shells, "states": int(solver.computed_metadata[0].source_level_idx.max() + 1),
                                                    "rows": int(len(solver.computed_metadata[0])), "ms": float(np.median(ts)), "all_ms": ts,
                                                    "pandas": pd.__version__, "note": "create_absorbing_probs stubbed out"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shells", type=int, default=50)
    ap.add_argument("--levels", type=int, default=1000)
    ap.add_argument("--lines", type=int, default=20000)
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--reference", action="store_true")
    ap.add_argument("--h-levels", type=int, default=60)
    ap.add_argument("--he-levels", type=int, default=40)
    args = ap.parse_args()
    name, out = reference(args) if args.reference else gpu(args)
    os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)
    path = os.path.join(ROOT, "profiles", name)
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps({k: v for k, v in out.items() if not k.endswith("all") and k != "all_ms"}))


if __name__ == "__main__":
    main()
