"""Golden vectors of the continuum (IIP) macro atom's per-iteration rows (tests/test_continuum_macro_build.py), computed by
the UNMODIFIED reference ContinuumMacroAtomSolver.solve run twice (oracle/reference_runner_continuum_macro.py): the second
iteration takes _solve_next_macroatom_iteration.  Runs where the reference exists:

    python tests/golden/make_continuum_macro_golden.py [--case NAME]

Inputs are regenerated from seeds (tardis_b200.synthetic.make_continuum_rate_inputs).  Each case stores the reference's
metadata as arrays (the rows' types, source / destination states, line rows, block edges, line2macro_level_upper), the row
map that tardis_b200.macro_atom.continuum_row_map derives from the reference's own solver, and of the second iteration: the
unnormalised and normalised probabilities, the normalised deactivation table and X: whole, or (config-5-sized case) as
sampled cells, row sums of X and the SHA-256 of the continuum rows' unnormalised values."""
from __future__ import annotations

import argparse
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from tardis_b200 import synthetic as syn  # noqa: E402

# name: (make_continuum_rate_inputs keyword arguments, X storage)
CASES = {
    # every row type, 4 shells
    "continuum_macro_small": (dict(n_shells=4, n_h_levels=6, n_he_levels=5, seed=81), "full"),
    # rate frames in another row order than the metadata, repeated cooling destinations, all-zero blocks, an infinite rate
    "continuum_macro_adversarial": (dict(n_shells=5, n_h_levels=9, n_he_levels=6, seed=82, shuffle_rates=True, zero_levels=2,
                                         infinite_rate=True), "full"),
    # config-5-sized: 50 shells
    "continuum_macro_s50": (dict(n_shells=50, n_h_levels=20, n_he_levels=12, seed=83, n_lines=150), "sampled"),
}
N_SAMPLE = 6000


def inputs(name):
    return syn.make_continuum_rate_inputs(**CASES[name][0])


def metadata_arrays(solver):
    md, line2macro, edges, _ = solver.computed_metadata
    return dict(transition_type=md.transition_type.to_numpy().astype(np.int64),
                source_level_idx=md.source_level_idx.to_numpy().astype(np.int64),
                destination_level_idx=md.destination_level_idx.to_numpy().astype(np.int64),
                transition_line_idx=md.transition_line_idx.to_numpy().astype(np.int64),
                macro_block_edge_index=np.asarray(edges, dtype=np.int64),
                line2macro_level_upper=np.asarray(line2macro, dtype=np.int64))


def generate(name):
    from oracle import reference_runner_continuum_macro as rr
    from tardis_b200 import macro_atom

    ci = inputs(name)
    ref = rr.run(ci)
    out = metadata_arrays(ref["solver"])
    rmap = macro_atom.continuum_row_map(ref["solver"], ref["metadata"], ci.rates[-1])
    out.update(rate_key=rmap["rate_key"], energy=rmap["energy"], n_rate_rows=np.array(rmap["n_rate_rows"]),
               n_cooling_rows=np.array(rmap["n_cooling_rows"]))
    X = ref["state"].absorbing_probability_matrix
    out["row_sums"] = X.sum(axis=2)
    if CASES[name][1] == "full":
        out.update(raw=ref["raw"], normalized=ref["normalized"], deactivation=ref["deactivation"], X=X)
    else:  # the continuum rows' raw values as a digest of their bytes, the rest as sampled cells
        cont = ~np.isin(out["transition_type"], (-1, 0, 1))
        out["raw_continuum_sha256"] = np.array(hashlib.sha256(np.ascontiguousarray(ref["raw"][cont]).tobytes()).hexdigest())
        rng = np.random.default_rng(7)
        for key, table in (("raw", ref["raw"]), ("normalized", ref["normalized"]), ("deactivation", ref["deactivation"]), ("X", X)):
            idx = np.sort(rng.choice(table.size, min(N_SAMPLE, table.size), replace=False))
            out[key + "_sample_idx"], out[key + "_sample_val"] = idx, table.ravel()[idx]
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, **out)
    print(f"{name}: T = {len(out['transition_type'])}, S = {X.shape[0]}, n = {X.shape[1]}; wrote {os.path.getsize(path) / 1e3:.0f} kB")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--case", default=None)
    args = ap.parse_args()
    for name in [args.case] if args.case else CASES:
        generate(name)


if __name__ == "__main__":
    main()
