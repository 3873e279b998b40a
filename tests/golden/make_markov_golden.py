"""Golden vectors of the continuum macro atom's absorbing Markov chain (tests/test_markov_build.py), computed by the
UNMODIFIED reference function create_absorbing_probs (/root/reference/tardis/opacities/macro_atom/absorbing_markov_chain.py,
loaded from its file: it imports only numpy, pandas and scipy) and the reference's normalisation,
normalize_transition_probabilities (opacities/macro_atom/macroatom_solver.py:709-739).  That function's module pulls the
atomic-data stack, so `normalize` restates what it does with pandas: divide by the group-by-source sum, NaN -> 0, so that
pandas' own group sum produces the golden.  Runs where the reference exists:

    python tests/golden/make_markov_golden.py [--case NAME]

Inputs are regenerated from seeds by `markov_inputs` (tardis_b200.synthetic.add_continuum_macro_atom).  Small cases store X
and the deactivation table whole; the others store X as row sums, sampled cells and its zero pattern (packed bits, or zero
counts per row for the bench-shape case), and the deactivation table whole or as the SHA-256 of its bytes."""
from __future__ import annotations

import argparse
import hashlib
import importlib.util
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from tardis_b200 import synthetic as syn  # noqa: E402

# name: (seed, n_shells, add_continuum_macro_atom keyword arguments, storage)
MARKOV_CASES = {
    "markov_n62": (71, 8, dict(n_levels=60), "full"),
    "markov_illcond": (72, 4, dict(n_levels=128, ill_conditioned_shell=2), "full"),
    "markov_n400": (73, 8, dict(n_levels=398, n_groups=3, duplicate_fraction=0.25, self_loop_fraction=0.1, zero_blocks=4), "packed"),
    "markov_n1000": (74, 50, dict(n_levels=998, internal_rows=(12, 12), deactivation_rows=(4, 4)), "counts"),
}
N_SAMPLE = 8000


def markov_inputs(name):
    """-> (model, ContinuumMacroAtom) of the case."""
    seed, S, kw, _ = MARKOV_CASES[name]
    model = syn.add_continuum(syn.make_model(S, 2000, "macroatom", seed=seed), seed=seed + 1)
    return model, syn.add_continuum_macro_atom(model, seed=seed + 2, **kw)


def sample_idx(shape, seed):
    return np.sort(np.random.default_rng(seed).choice(int(np.prod(shape)), min(N_SAMPLE, int(np.prod(shape))), replace=False))


def compress(name, X, D):
    seed, _, _, storage = MARKOV_CASES[name]
    out = {"row_sums": X.sum(axis=2), "max_abs": np.abs(X).max()}
    if storage == "full":
        out["X"] = X
    else:
        idx = sample_idx(X.shape, seed)
        out["sample_idx"], out["sample_val"] = idx, X.ravel()[idx]
        if storage == "packed":
            out["zero_bits"] = np.packbits((X == 0).ravel())
        else:
            out["zero_counts"] = (X == 0).sum(axis=2).astype(np.int32)
    if storage == "counts":
        out["deactivation_sha256"] = np.array(hashlib.sha256(np.ascontiguousarray(D).tobytes()).hexdigest())
    else:
        out["deactivation"] = D
    return out


def reference_functions():
    import pandas as pd

    ref = os.environ.get("TARDIS_REFERENCE", "/root/reference")
    path = os.path.join(ref, "tardis", "opacities", "macro_atom", "absorbing_markov_chain.py")
    spec = importlib.util.spec_from_file_location("reference_absorbing_markov_chain", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)

    def normalize(probabilities, metadata):  # restates macroatom_solver.py:709-739
        sums = probabilities.groupby(metadata["source"].to_numpy()).transform("sum")
        return (probabilities / sums).fillna(0.0)

    return pd, mod.create_absorbing_probs, normalize


def reference_tables(cma):
    pd, create_absorbing_probs, normalize = reference_functions()
    meta = pd.DataFrame({"source": cma.source_level_idx, "source_level_idx": cma.source_level_idx,
                         "destination_level_idx": cma.destination_level_idx, "transition_type": cma.transition_type})
    tp = pd.DataFrame(cma.transition_probabilities.copy())
    t0 = time.perf_counter()
    X, deact = create_absorbing_probs(tp, meta, max_workers=1)
    t1 = time.perf_counter()
    D = normalize(deact, meta).to_numpy()
    return X, D, t1 - t0


def generate(name):
    model, cma = markov_inputs(name)
    X, D, dt = reference_tables(cma)
    out = compress(name, X, D)
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, **out)
    print(f"{name}: n = {cma.n_states}, S = {X.shape[0]}, reference {dt:.2f} s; wrote {os.path.getsize(path) / 1e3:.0f} kB")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--case", default=None)
    args = ap.parse_args()
    for name in [args.case] if args.case else MARKOV_CASES:
        generate(name)


if __name__ == "__main__":
    main()
