"""Time of the device-side packet source at the bench's packet count: `Engine.create_packets` for BlackBodyWeightedSource
(three passes, the leaf sums combined on the host) and for BlackBodySimpleSource, after a warm-up, and what the
reference-equivalent numpy code takes on the host for the same N (oracle/weighted_source_oracle.py restates it operation
by operation; its sum is np.sum itself here).

Reports the GPU's name and power limit (read in the same process as the timing).  Device times are CUDA events recorded
around the call on the default stream; the call returns after its own stream has finished, so they span the whole
create_packets, host work between the passes included.  Writes one JSON line to stdout (and to --out when given).

    python scripts/weighted_source_probe.py --packets 100000000 --out profiles/weighted_source_h100.json
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


def numpy_weighted(n, seed, radius, temperature):
    """BlackBodyWeightedSource.create_packets in the reference's numpy calls (base.py:229-236, black_body_weighted.py)"""
    from oracle.weighted_source_oracle import H, K_B, intensity_black_body

    rng = np.random.default_rng(seed)
    seeds = rng.choice(2**32 - 1, n, replace=True)
    l_array = np.cumsum(np.arange(1, 1000, dtype=np.float64) ** -4)
    xis = rng.random((5, n))
    l_ = l_array.searchsorted(xis[0] * (np.pi**4 / 90.0)) + 1.0
    nus_bb = (-np.log(np.prod(xis[1:], 0)) / l_) * (K_B * temperature) / H
    del xis, l_
    nus = rng.uniform(nus_bb.min(), nus_bb.max(), n)
    del nus_bb
    mus = np.sqrt(rng.random(n))
    intensity = intensity_black_body(nus, temperature)
    energies = intensity / intensity.sum()
    return np.full(n, radius), nus, mus, energies, seeds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--packets", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--numpy-packets", type=int, default=None, help="N of the host numpy run (default: --packets)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    from tardis_b200.engine import Engine

    n, radius, temperature, seed = args.packets, 1.23552e15, 1.0e4, 23111963
    eng = Engine(0)
    times = {}
    for label, kw in (("weighted", dict(weighted=True)), ("plain", {})):
        eng.create_packets(n, seed, radius, temperature, **kw)  # warm-up (allocations, first launches)
        ms = []
        for rep in range(args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            eng.create_packets(n, seed + 1 + rep, radius, temperature, **kw)
            b.record()
            b.synchronize()
            ms.append(a.elapsed_time(b))
        times[label] = dict(median_ms=float(np.median(ms)), min_ms=float(np.min(ms)), all_ms=ms)
    eng.create_packets(n, seed, radius, temperature, weighted=True)  # the plain source ran last: one more weighted set to check
    pk = eng.download_packets()
    checks = dict(energy_sum_minus_1=float(pk["initial_energies"].sum() - 1.0),
                  energy_max_over_min=float(pk["initial_energies"].max() / pk["initial_energies"].min()))
    del pk
    eng.close()

    nn = args.numpy_packets or n
    t0 = time.perf_counter()
    numpy_weighted(nn, seed, radius, temperature)
    host_s = time.perf_counter() - t0

    res = dict(probe="weighted_source", packets=n, **gpu_info(), torch_device=torch.cuda.get_device_name(0),
               create_packets_weighted_ms=times["weighted"], create_packets_plain_ms=times["plain"],
               weighted_over_plain=times["weighted"]["median_ms"] / times["plain"]["median_ms"],
               weighted_packets_per_s=n / (times["weighted"]["median_ms"] * 1e-3),
               numpy_reference_equivalent=dict(packets=nn, seconds=host_s, cpu_count=os.cpu_count(),
                                               note="single-threaded numpy on the host of the same run"),
               checks=checks)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
