"""Golden vectors of the unmodified `BlackBodyWeightedSource.create_packets`
(tardis/transport/montecarlo/packet_source/black_body_weighted.py:9-108 on base.py:195-253).

    python tests/golden/make_weighted_source_golden.py      # writes tests/golden/weighted_source_*.npz

Runs where the reference tree is available (oracle/reference_loader.py), with the stand-ins oracle/reference_runner.py
already installs: `numexpr` evaluated by numpy (so the goldens carry numpy's `log`, `**` and `exp`) and a
`tardis.util.base` holding only `intensity_black_body`.  The Quantity stand-in also needs what this class calls on its
frequencies: `.min()`, `.max()` and `.unit`.  The output is a pure function of the cases below: rerunning gives
byte-identical files.  (Named weighted_source_*, not packet_source_*: that prefix is the plain source's case list.)
"""
from __future__ import annotations

import io
import os
import sys
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

# name -> (no_of_packets, base_seed, seed_offset, radius [cm], temperature [K])
CASES = {
    "weighted_source_basic": (4001, 23111963, 0, 1.2355e15, 1.0e4),
    "weighted_source_iteration5": (2500, 23111963, 5, 1.2355e15, 9.974969e3),
    "weighted_source_big_seed": (1024, 2**32 - 6, 10, 8.0e14, 2.5e4),  # base_seed + seed_offset >= 2**32
    "weighted_source_single": (1, 1963, 0, 1.0e15, 1.0e4),
    "weighted_source_20011": (20011, 77, 0, 1.2355e15, 1.0e4),  # > 8192 packets, not a multiple of 8
    "weighted_source_bench_model": (12289, 23111963, 1, 1.23552e15, 1.0e4),  # synthetic.make_model's r_inner[0], bench's T
}


def install_stand_ins():
    from oracle import reference_loader
    from oracle.reference_runner import run_reference_packet_source, run_reference_radfield

    run_reference_packet_source(1, 1, 0, 1.0e15, 1.0e4)  # numexpr, hdf_writer_mixin, the packet_source package
    run_reference_radfield(np.ones(1), np.full(1, 1e15), np.ones((1, 1)), 1.0e6, 1.0, np.full(1, 1e45), np.full(1, 1e15))  # tardis.util.base
    Q = reference_loader._Q
    Q.min = lambda self: Q(self.value.min())
    Q.max = lambda self: Q(self.value.max())
    Q.unit = property(lambda self: Q(1.0))
    return Q


def generate(name, Q):
    from tardis.transport.montecarlo.packet_source.black_body_weighted import BlackBodyWeightedSource

    n, base_seed, off, radius, temperature = CASES[name]
    src = BlackBodyWeightedSource(radius=Q(float(radius)), temperature=Q(float(temperature)), base_seed=int(base_seed))
    pc = src.create_packets(int(n), seed_offset=int(off))
    out = dict(initial_radii=np.asarray(pc.initial_radii, dtype=np.float64), initial_nus=np.asarray(pc.initial_nus, dtype=np.float64),
               initial_mus=np.asarray(pc.initial_mus, dtype=np.float64), initial_energies=np.asarray(pc.initial_energies, dtype=np.float64),
               packet_seeds=np.asarray(pc.packet_seeds, dtype=np.int64),
               radiation_field_luminosity=np.float64(pc.radiation_field_luminosity),
               self_nus=np.asarray(src.nus.value, dtype=np.float64))
    arrays = dict(n=np.int64(n), base_seed=np.uint64(base_seed), seed_offset=np.int64(off), radius=np.float64(radius),
                  temperature=np.float64(temperature), **out)
    # np.savez_compressed stamps the zip members with the current time; fixed stamps make the file reproducible
    path = os.path.join(HERE, name + ".npz")
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k, v in arrays.items():
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(v), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())
    print(f"{name}: wrote {os.path.getsize(path) / 1e3:.0f} kB; energies {out['initial_energies'].min():.3e} .. "
          f"{out['initial_energies'].max():.3e}, sum - 1 = {out['initial_energies'].sum() - 1:.2e}")


def write_interface():
    """The reference class's public surface, parsed (not imported) from black_body_weighted.py, for the mirror's test."""
    import ast
    import json

    from oracle import reference_loader

    path = os.path.join(reference_loader.REF, "tardis", "transport", "montecarlo", "packet_source", "black_body_weighted.py")
    cls = next(n for n in ast.parse(open(path).read()).body if isinstance(n, ast.ClassDef) and n.name == "BlackBodyWeightedSource")
    attrs, methods, init = {}, [], None
    for node in cls.body:
        if isinstance(node, ast.Assign) and isinstance(node.targets[0], ast.Name):
            attrs[node.targets[0].id] = ast.literal_eval(node.value)
        elif isinstance(node, ast.FunctionDef):
            methods.append(node.name)
            if node.name == "__init__":
                init = {"positional": [a.arg for a in node.args.args[1:]], "kwarg": node.args.kwarg.arg if node.args.kwarg else None}
    out = {"bases": [ast.unparse(b) for b in cls.bases], "attributes": attrs, "methods": sorted(methods), "init": init}
    with open(os.path.join(HERE, "reference_interface_weighted_source.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


def main():
    Q = install_stand_ins()
    for name in CASES:
        generate(name, Q)
    write_interface()


if __name__ == "__main__":
    main()
