"""Cost of the nonhomologous mode's opacity tables per iteration at the bench shape (5e5 lines, 20 shells, 3000 levels,
1.5e6 macro-atom rows, interior velocities +-8 %, macroatom), two ways, in one process:

  device: `Engine.build_opacity(level_number_density, 0.0, velocity_gradient=...)` on the J_blue table the radiation-field
          solve left in HBM (tb200_build_opacity: tau, beta, probabilities, normalisation, running sums, prefix sums);
  host:   what a nonhomologous iteration did before: `set_model` with the host-built [L, S] tau and [T, S] probability tables
          (the upload, transposes and the same running sums / prefix sums).  The host build of those tables is not timed
          here (pass --with-oracle-build to add the numpy oracle's time; the reference's pandas path is slower still).

Host clocks around synchronised calls, after a warm-up of each path; the card's name and power limit are read in the same
process.  Writes one JSON line to stdout (and to --out when given).

    python scripts/nonhomologous_opacity_probe.py --repeats 5 --out profiles/nonhomologous_opacity_h100.json
"""
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


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except (OSError, subprocess.CalledProcessError):
        return dict(gpu="unknown", power_limit="unknown", max_sm_clock="unknown")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--with-oracle-build", action="store_true", help="also time the numpy oracle's host build of the tables")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    from oracle import opacity_oracle_nonhomologous
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import Engine

    S = 20
    model = syn.make_nonhomologous_velocities(syn.make_model(S, 500_000, "macroatom"), 0.08)
    atomic = syn.make_atomic_data(model.line_list_nu, 3000, "macroatom", seed=91)
    plasma = syn.make_plasma_state(atomic, S, 0.0, seed=92, zero_fraction=0.0, inversion_fraction=0.0)
    grad = (model.v_outer - model.v_inner) / (model.r_outer - model.r_inner)
    t0 = time.perf_counter()
    tables = opacity_oracle_nonhomologous.build(atomic, plasma, grad, nlte=True)
    oracle_s = time.perf_counter() - t0
    tau, tp = tables["tau_sobolev"], tables["transition_probabilities"]
    del tables

    def set_model(eng, tau=None, tp=None):
        eng.set_model(r_inner=model.r_inner, r_outer=model.r_outer, time_explosion=0.0, electron_density=model.electron_density,
                      line_list_nu=model.line_list_nu, tau_sobolev=tau, line_interaction_type="macroatom", transition_probabilities=tp,
                      line2macro_level_upper=atomic.line2macro_level_upper, macro_block_edge_index=atomic.macro_block_edge_index,
                      transition_type=atomic.transition_type, destination_level_id=atomic.destination_level_id,
                      transition_line_id=atomic.transition_line_idx, spectrum_frequency_grid=model.spectrum_frequency_grid,
                      nonhomologous=True, v_inner=model.v_inner, v_outer=model.v_outer)

    dev, host = Engine(0), Engine(0)
    set_model(dev)
    dev.set_atomic_data(lines_lower_level_index=atomic.lower_level, lines_upper_level_index=atomic.upper_level, g=atomic.g,
                        metastability=atomic.metastable, wavelength_cm=atomic.wavelength_cm, f_lu=atomic.f_lu, f_ul=atomic.f_ul,
                        energy_lower=atomic.energy[atomic.lower_level], energy_upper=atomic.energy[atomic.upper_level],
                        nlte_line=atomic.nlte_line)
    # J_blue resident in HBM, as after a transport: the radiation-field solve on the host-given estimators
    volume = (4 / 3) * np.pi * (model.r_outer**3 - model.r_inner**3)
    dev.solve_radiation_field(time_explosion=0.0, time_of_simulation=1.0, volume=volume, velocity_gradient=grad, want_j_blues=False,
                              estimators=(np.full(S, 1e40), np.full(S, 1e55), plasma.j_blues))
    lnd = plasma.level_number_density

    def device():
        dev.build_opacity(lnd, 0.0, velocity_gradient=grad)
        dev.sync()

    def host_path():
        set_model(host, tau, tp)
        host.sync()

    device(); host_path()  # warm-up of both paths
    dev_s, host_s = [], []
    for _ in range(args.repeats):  # alternating
        t0 = time.perf_counter(); device(); dev_s.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); host_path(); host_s.append(time.perf_counter() - t0)
    got = dev.download_opacity()
    parity = dict(tau_bit_identical=bool(np.array_equal(got["tau_sobolev"], tau)),
                  negative_tau_cells=int((tau < 0).sum()))
    res = dict(info=gpu_info(), shape=dict(lines=len(atomic.nu), shells=S, levels=atomic.n_levels, rows=len(atomic.transition_type)),
               device_build_ms=[1e3 * s for s in dev_s], set_model_host_tables_ms=[1e3 * s for s in host_s],
               device_build_ms_min=1e3 * min(dev_s), set_model_host_tables_ms_min=1e3 * min(host_s), parity=parity)
    if args.with_oracle_build:
        res["numpy_oracle_host_build_ms"] = 1e3 * oracle_s
    dev.close(); host.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
