"""Time the classic plasma solved on the device (tb200_solve_plasma) against the numpy / pandas restatement of the reference's
chain on the host, and the opacity build on the resident populations against the build from host arrays.

Sizes: 20 shells / 3000 levels and 50 shells / 30000 levels, 5e5 lines, 30 elements (495 ions), nebular ionisation,
dilute-LTE excitation, dilute-blackbody J_blue.  Per stage:
  * the kernels of one solve (torch.profiler with CUDA activities, in a run of its own): Boltzmann factors, partition
    functions, Phi, the n_e fixed point (one launch; its iteration count is reported), level populations, the J_blue write;
  * the whole tb200_solve_plasma call (host clock around the call, which ends in a device synchronise);
  * build_opacity(None) (resident populations and J_blue) against build_opacity(host populations, host J_blue);
  * the oracle on the host (oracle/plasma_oracle.py: the reference's operations in numpy / pandas), J_blue included.
The card's name and power limit are read in the same run.

    python scripts/plasma_probe.py --repeats 5 --out profiles/plasma_h100.json
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
                             capture_output=True, text=True, check=True).stdout.splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception:  # noqa: BLE001
        return dict(gpu="unknown", power_limit="unknown", max_sm_clock="unknown")


def timed(f, repeats):
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        f()
        ts.append((time.perf_counter() - t0) * 1e3)
    return dict(min_ms=min(ts), median_ms=float(np.median(ts)))


def probe(S, n_levels, L, repeats):
    from oracle import plasma_oracle
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import Engine

    model = syn.make_model(S, L, "macroatom", seed=31)
    atomic = syn.make_atomic_data(model.line_list_nu, n_levels, seed=32)
    st = syn.make_plasma_structure(atomic, S, seed=33)
    rng = np.random.default_rng(34)
    t_rad, w = rng.uniform(8e3, 1.3e4, S), rng.uniform(0.05, 0.5, S)
    eng = Engine(0)
    eng.set_model(r_inner=model.r_inner, r_outer=model.r_outer, time_explosion=model.time_explosion,
                  electron_density=model.electron_density, line_list_nu=model.line_list_nu, tau_sobolev=None,
                  line_interaction_type="macroatom", transition_probabilities=None, line2macro_level_upper=atomic.line2macro_level_upper,
                  macro_block_edge_index=atomic.macro_block_edge_index, transition_type=atomic.transition_type,
                  destination_level_id=atomic.destination_level_id, transition_line_id=atomic.transition_line_idx,
                  spectrum_frequency_grid=model.spectrum_frequency_grid)
    eng.set_atomic_data(lines_lower_level_index=atomic.lower_level, lines_upper_level_index=atomic.upper_level, g=atomic.g,
                        metastability=atomic.metastable, wavelength_cm=atomic.wavelength_cm, f_lu=atomic.f_lu, f_ul=atomic.f_ul,
                        energy_lower=atomic.energy[atomic.lower_level], energy_upper=atomic.energy[atomic.upper_level])
    data = dict(level_energy=st.level_energy, level_ion=st.level_ion, ion_atomic_number=st.ion_atomic_number, ion_charge=st.ion_charge,
                ionization_energy=st.ionization_energy, number_density=st.number_density, zeta_temperatures=st.zeta_temperatures,
                zeta=st.zeta)
    eng.set_plasma_data(**data)
    host = eng.solve_plasma(t_rad, w, download=True)  # warm-up, and the host copies for the host-array build
    solve = timed(lambda: eng.solve_plasma(t_rad, w), repeats)
    eng.build_opacity(None, model.time_explosion)
    build_resident = timed(lambda: eng.build_opacity(None, model.time_explosion), repeats)
    lnd, jb = host["level_number_density"], host["j_blues"]
    eng.build_opacity(lnd, model.time_explosion, jb)
    build_host = timed(lambda: eng.build_opacity(lnd, model.time_explosion, jb), repeats)
    eng.solve_plasma(t_rad, w)  # resident again
    kernels = {}
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(repeats):
                eng.solve_plasma(t_rad, w)
            torch.cuda.synchronize()
        for e in prof.key_averages():
            if e.key.startswith(("plasma_", "_GLOBAL__N__")) or "plasma_" in e.key:
                name = e.key.split("(")[0].split("::")[-1]
                kernels[name] = kernels.get(name, 0.0) + e.device_time_total / 1e3 / repeats
    except Exception as ex:  # noqa: BLE001
        kernels = {"error": repr(ex)}
    t0 = time.perf_counter()
    ref = plasma_oracle.solve(st.level_energy, st.level_ion, atomic.g, atomic.metastable, st.ion_atomic_number, st.ion_charge,
                              st.ionization_energy, st.number_density, t_rad, w, zeta_temperatures=st.zeta_temperatures, zeta=st.zeta,
                              line_nu=model.line_list_nu)
    oracle_ms = (time.perf_counter() - t0) * 1e3
    agree = float(np.max(np.abs(host["electron_densities"] / ref["electron_densities"] - 1)))
    eng.close()
    return dict(n_shells=S, n_levels=n_levels, n_ions=len(st.ion_charge), n_lines=L, ne_iterations=int(host["iterations"]),
                solve_plasma_ms=solve, kernels_ms=kernels, build_opacity_resident_ms=build_resident, build_opacity_host_arrays_ms=build_host,
                host_oracle_ms=oracle_ms, max_rel_ne_vs_oracle=agree)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--lines", type=int, default=500000)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    res = dict(**gpu_info(), repeats=a.repeats, sizes=[probe(20, 3000, a.lines, a.repeats), probe(50, 30000, a.lines, a.repeats)])
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
