"""Time tb200_build_absorbing_markov (the continuum macro atom's absorbing Markov chain, tardis_b200/csrc/markov_build.cuh) at
S = 50 shells and n = 62, 300, 1000, 2000 states, with the oracle's host solve (scipy splu, as the reference) beside it.

    python scripts/markov_build_probe.py [--sizes 62,300,1000,2000] [--host-max 1000] [--out DIR]

Prints one JSON line.  `wall_s`: host clock around the whole call, which ends in a device synchronise (host checks, upload
of the [T, S] input, assembly, solve, cumulative sums, deactivation table), median of the repeats after a warm-up build.
It is wall time, not kernel time: at small n the host checks and the upload dominate it.
FLOP/s: the Gauss-Jordan inversion's 2 n^3 per shell over that time, against the H100 SXM data sheet's 67 TFLOP/s FP64
tensor core and 34 TFLOP/s FP64 peaks.  The card's name and power limit are read in the same run."""
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

from oracle import markov_oracle as mo  # noqa: E402
from tardis_b200 import synthetic as syn  # noqa: E402
from tardis_b200.engine import Engine  # noqa: E402

PEAK_FP64_TC, PEAK_FP64 = 67e12, 34e12


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="62,300,1000,2000")
    ap.add_argument("--shells", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--host-max", type=int, default=1000, help="largest n whose host solve is timed")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    S = args.shells
    eng = Engine(0)
    rows = []
    for n in (int(x) for x in args.sizes.split(",")):
        model = syn.add_continuum(syn.make_model(S, 2000, "macroatom", seed=81), seed=82)
        cma = syn.add_continuum_macro_atom(model, seed=83, n_levels=n - 2, internal_rows=(12, 12), deactivation_rows=(4, 4))
        eng.set_model_from(model, enable_full_relativity=True)
        a = (cma.transition_probabilities, cma.source_level_idx, cma.destination_level_idx, cma.transition_type)
        eng.build_absorbing_markov(*a)
        times = []
        for _ in range(args.repeats):
            t0 = time.perf_counter()
            eng.build_absorbing_markov(*a)
            times.append(time.perf_counter() - t0)
        wall = float(np.median(times))
        flops = 2.0 * n ** 3 * S
        row = dict(n=n, shells=S, wall_s=wall, wall_s_all=times, fp64_flops_per_s=flops / wall,
                   share_of_fp64_tc_peak=flops / wall / PEAK_FP64_TC, share_of_fp64_peak=flops / wall / PEAK_FP64)
        if n <= args.host_max:
            t0 = time.perf_counter()
            mo.absorbing_probs(*a)
            mo.deactivation_table(cma.transition_probabilities, cma.transition_type, cma.macro_block_edge_index)
            row["host_oracle_splu_s"] = time.perf_counter() - t0
        rows.append(row)
    eng.close()
    line = json.dumps(dict(probe="markov_build", gpu=gpu_info(), results=rows))
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "markov_build_probe.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
