"""Rate of the nonhomologous transport kernel on the bench model (20 shells, 5e5 lines, macroatom) with the interior
velocities perturbed by +-8 % (synthetic.make_nonhomologous_velocities: some shells decelerate).

Reports the GPU's name and power limit (read in the same process as the timing), packets/s and line-steps/s from the CUDA
events of tb200_transport after a warm-up, and the parity of the work counters and estimators against the CPU oracle on a
sample of packets.  Writes one JSON line to stdout (and to --out when given).

    python scripts/nonhomologous_probe.py --packets 10000000 --sample 20000
"""
from __future__ import annotations

import argparse
import dataclasses
import json
import os
import subprocess
import sys

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
    ap.add_argument("--packets", type=int, default=10_000_000)
    ap.add_argument("--sample", type=int, default=20_000, help="packets compared with the CPU oracle")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    from oracle import nonhomologous_oracle
    from tardis_b200 import synthetic
    from tardis_b200.engine import Engine

    model = synthetic.make_nonhomologous_velocities(synthetic.make_model(20, 500_000, "macroatom"), 0.08)
    model = dataclasses.replace(model, time_explosion=0.0)
    eng = Engine(0)
    eng.set_model_from(model, nonhomologous=True)

    # parity on a sample
    sample = synthetic.make_packets(args.sample, model.r_inner[0], base_seed=7)
    got = eng.run_packets(sample, track_last_interaction=True)
    ref = nonhomologous_oracle.run_oracle(model, sample)
    parity = dict(
        counters_identical=all(got["counters"][k] == v for k, v in ref["counters"].items() if k in got["counters"]),
        last_interaction_identical=all(np.array_equal(got[k], ref[k]) for k in ("last_interaction_type", "last_line_absorb_id",
                                                                                "last_line_emit_id", "last_shell_id")),
        max_rel_output_nus=float(np.max(np.abs(got["output_nus"] - ref["output_nus"]) / np.abs(ref["output_nus"]))),
        max_rel_j_blue=float(np.max(np.abs(got["j_blue"] - ref["j_blue"]) / np.maximum(np.abs(ref["j_blue"]), 1e-300))),
    )

    packets = synthetic.make_packets(args.packets, model.r_inner[0], base_seed=11)
    eng.upload_packets(packets.initial_radii, packets.initial_nus, packets.initial_mus, packets.initial_energies, packets.packet_seeds)
    eng.transport(); eng.sync()  # warm-up
    ms = []
    for _ in range(args.steps):
        eng.transport(); eng.sync()
        ms.append(eng.last_kernel_ms())
    c = eng.counters()
    best = min(ms)
    res = dict(info=gpu_info(), packets=args.packets, kernel_ms=ms, packets_per_s=args.packets / (best * 1e-3),
               line_steps_per_s=c["n_line_steps"] / (best * 1e-3), line_steps_per_packet=c["n_line_steps"] / args.packets,
               events_per_packet=(c["n_line_events"] + c["n_escat_events"]) / args.packets, parity_sample=args.sample, parity=parity)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
