"""Packets per second of one Engine(0) against an EngineGroup, on the bench model, and the time of the group's collective.

Strong scaling: the same total number of packets on one engine and on the group.  Weak scaling: `--packets` per member.
Packets come from the device-side packet source (tb200_group_create_packets: each member generates its own range), and
every timed call is `run_resident` without per-packet outputs: transport, collective and the estimators to the host.
Times are host clocks around calls that end in a device synchronise; the collective's time is the group's own
(tb200_group_allreduce_ms), which covers the whole step: waiting for the members' streams, the reductions, the
finalisation of the line estimators on every member and the final synchronise.  The byte count is every member's
fixed-point words (n_shells x (line_pitch + 1) x 4 x 8 B) plus the f64 prefix of its estimator buffer, read from every
member and written to every member; bytes over the step's time ("step_GB_per_s") is a lower bound on the bandwidth of
the reduction kernels themselves.

With one GPU the default group is [0, 0]: two engines on the same device, which shows the group's overhead (the members
transport one after the other, and the collective runs on that device's HBM).  Prints one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tardis_b200 import synthetic as syn  # noqa: E402
from tardis_b200.engine import Engine, EngineGroup  # noqa: E402


def timed(eng, model, n, reps, seed):
    """Median seconds of run_resident over `reps` calls (after one warm-up), with fresh packets each time."""
    radius, temp = float(model.r_inner[0]), 10000.0
    times = []
    for rep in range(reps + 1):
        eng.create_packets(n, seed + rep, radius, temp)
        t0 = time.perf_counter()
        eng.run_resident(per_packet=False)
        if rep:
            times.append(time.perf_counter() - t0)
    times.sort()
    return times[len(times) // 2]


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out
    except Exception as e:  # the numbers still stand; say what could not be read
        return [f"nvidia-smi unavailable: {e}"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--packets", type=int, default=100_000_000, help="total packets (strong) / packets per member (weak)")
    ap.add_argument("--devices", default=None, help="comma-separated device ids of the group (default: every device; 0,0 on one GPU)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--lines", type=int, default=500_000)
    ap.add_argument("--shells", type=int, default=20)
    ap.add_argument("--mode", default="macroatom")
    ap.add_argument("--mu-tau", type=float, default=-7.5)
    ap.add_argument("--no-weak", action="store_true")
    args = ap.parse_args()
    import torch

    n_dev = torch.cuda.device_count()
    if n_dev < 1:
        raise SystemExit("no CUDA device: this script measures the GPU")
    devices = [int(d) for d in args.devices.split(",")] if args.devices else (list(range(n_dev)) if n_dev > 1 else [0, 0])
    model = syn.make_model(args.shells, args.lines, args.mode, mu_tau=args.mu_tau)
    out = {"gpus": gpu_info(), "devices": devices, "model": {"shells": args.shells, "lines": args.lines, "mode": args.mode,
                                                              "mu_tau": args.mu_tau}}
    one = Engine(0)
    one.set_model_from(model)
    t1 = timed(one, model, args.packets, args.reps, 1000)
    out["engine0"] = {"packets": args.packets, "s": t1, "packets_per_s": args.packets / t1}
    lay = one.estimator_layout()
    one.close()

    group = EngineGroup(devices)
    group.set_model_from(model)
    g = len(devices)
    ts = timed(group, model, args.packets, args.reps, 2000)
    coll_ms = group.allreduce_ms()
    out["strong"] = {"packets": args.packets, "s": ts, "packets_per_s": args.packets / ts, "speedup": t1 / ts}
    if not args.no_weak:
        tw = timed(group, model, args.packets * g, args.reps, 3000)
        out["weak"] = {"packets": args.packets * g, "s": tw, "packets_per_s": args.packets * g / tw,
                       "efficiency": (args.packets * g / tw) / (g * args.packets / t1)}
        coll_ms = group.allreduce_ms()
    words_bytes = lay["n_shells"] * (lay["line_pitch"] + 1) * 4 * 8
    member_bytes = words_bytes + lay["off_j_blue"] * 8
    moved = 2 * g * member_bytes  # every member's copy read once and written once
    out["collective"] = {"ms": coll_ms, "bytes_per_member": member_bytes, "bytes_read_and_written": moved,
                         "step_GB_per_s": moved / (coll_ms * 1e-3) / 1e9}
    group.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
