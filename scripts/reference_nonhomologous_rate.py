"""Packets/s of the UNMODIFIED reference's nonhomologous Numba loop (`montecarlo_transport_with_vpackets` with the
nonhomologous `packet_propagation`, time_explosion = 0.0) on the model of scripts/nonhomologous_probe.py: the bench model
(20 shells, 5e5 lines, macroatom) with the interior velocities perturbed by +-8 %.  Run where the reference tree exists (it
does not travel to the GPU machines).  Protocol of scripts/reference_numba_rate.py: one warm-up call (JIT), then best of 3,
at 1 thread and at --threads threads.

    python scripts/reference_nonhomologous_rate.py [--packets 2000] [--threads 8] [--out profiles/reference_nonhomologous_rate.json]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import reference_runner, reference_runner_nonhomologous as rrn  # noqa: E402
from tardis_b200 import synthetic as syn  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--packets", type=int, default=2000)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numba

    model = syn.make_nonhomologous_velocities(syn.make_model(20, 500_000, "macroatom"), 0.08)
    packets = syn.make_packets(args.packets, model.r_inner[0], base_seed=11)
    R = rrn.load()
    _, _, opacity, cfg, pc = reference_runner.build_reference_objects(model, packets)
    geo = rrn.geometry(model)
    n = len(packets)
    results = {}
    for nthreads in (1, args.threads):
        numba.set_num_threads(nthreads)
        best = None
        for rep in range(4):  # rep 0 = JIT warm-up
            trackers = R.generate_tracker_last_interaction_list(n)
            t0 = time.perf_counter()
            R.montecarlo_transport_with_vpackets(pc, geo, 0.0, opacity, cfg, model.spectrum_frequency_grid, trackers, 0, False,
                                                 R.nonhomologous_packet_propagation)
            dt = time.perf_counter() - t0
            if rep > 0:
                best = dt if best is None else min(best, dt)
        results[str(nthreads)] = {"threads": nthreads, "packets_per_s_loop_only": n / best, "seconds_loop_only": best}
        print(nthreads, results[str(nthreads)], flush=True)
    out = {"what": "unmodified reference nonhomologous Numba loop, bench model (5e5 lines, 20 shells, macroatom) with interior "
                   "velocities x (1 + 0.08 U(-1, 1)), no virtual packets, JIT excluded",
           "packets": n, "host": {"cpu_count": os.cpu_count(), "numba": numba.__version__, "where": "CPU build host (no GPU)"},
           "results": results}
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
