"""Golden vectors of the reference's nonhomologous mode (oracle/reference_runner_nonhomologous.py).

Run from the repository root where the reference tree exists:  python tests/golden/make_nonhomologous_golden.py
Writes tests/golden/nonhomologous_<case>.npz: the case's inputs are rebuilt from the synthetic generators by
`case_inputs`, the outputs are the reference's.
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from tardis_b200 import synthetic  # noqa: E402

# name -> (model kwargs, velocity law, n_packets, run kwargs).  Velocity laws: "perturbed" = make_nonhomologous_velocities
# (some shells decelerate), "homologous" = v = r / t as the model has it, "flat" = perturbed with one shell of
# v_inner == v_outer.
CASES = {
    "macroatom_vpackets": (dict(n_shells=10, n_lines=4000, line_interaction_type="macroatom", mu_tau=-4.0), "perturbed", 300,
                           dict(number_of_vpackets=2, survival_probability=0.5)),
    "scatter": (dict(n_shells=10, n_lines=4000, line_interaction_type="scatter", mu_tau=-4.0), "perturbed", 300, {}),
    "downbranch": (dict(n_shells=10, n_lines=4000, line_interaction_type="downbranch", mu_tau=-4.0), "perturbed", 300, {}),
    "homologous": (dict(n_shells=10, n_lines=4000, line_interaction_type="macroatom", mu_tau=-4.0), "homologous", 300, {}),
    "flat_shell": (dict(n_shells=10, n_lines=4000, line_interaction_type="macroatom", mu_tau=-4.0), "flat", 300, {}),
    "nolines": (dict(n_shells=10, n_lines=4000, line_interaction_type="scatter", mu_tau=-4.0), "perturbed", 300,
                dict(disable_line_scattering=True)),
}


# cases stored with compress_line_table (the [L, S] tables of the bench shape are 80 MB each)
BENCH_CASES = {
    "bench_shape": (dict(n_shells=20, n_lines=500_000, line_interaction_type="macroatom"), "perturbed", 1000, {}),
}
# cases run in a subprocess of their own: SIGMA_THOMSON is frozen into the compiled loop at its first compile
SIGMA_CASES = {
    "sigma_1e-200": (dict(n_shells=10, n_lines=4000, line_interaction_type="macroatom", mu_tau=-4.0), "perturbed", 300,
                     dict(sigma_thomson=1e-200)),
}
# the nonhomologous radiation-field solve on the estimators of a stored transport case
RADFIELD_CASES = {"radfield_macroatom_vpackets": "macroatom_vpackets", "radfield_flat_shell": "flat_shell"}
ALL = {**CASES, **BENCH_CASES, **SIGMA_CASES}


def case_inputs(name):
    """(model, packets, run kwargs) of a case."""
    mk, law, n, kw = ALL[name]
    model = synthetic.make_model(**mk)
    if law in ("perturbed", "flat"):
        model = synthetic.make_nonhomologous_velocities(model, 0.08)
    if law == "flat":
        model.v_outer[4] = model.v_inner[4]
        model.v_inner[5] = model.v_inner[4]
    packets = synthetic.make_packets(n, model.r_inner[0])
    return model, packets, dict(kw)


def radfield_inputs(name):
    """Inputs of a radiation-field case: the stored transport case's estimators and geometry, t_sim = 1 / L_inner."""
    src = RADFIELD_CASES[name]
    model, packets, _ = case_inputs(src)
    g = np.load(os.path.join(HERE, f"nonhomologous_{src}.npz"))
    volume = (4 / 3) * np.pi * (model.r_outer**3 - model.r_inner**3)
    return dict(j=g["j"], nu_bar=g["nu_bar"], j_blue=g["j_blue"], velocity_gradient=g["velocity_gradient"],
                time_of_simulation=packets.time_of_simulation, volume=volume, line_list_nu=model.line_list_nu, w_epsilon=1e-10)


INTERFACE = {  # reference file (relative to transport/montecarlo/modes/) -> functions whose positional parameters are mirrored
    "nonhomologous/solver.py": ["MCTransportSolverNonhomologous.__init__", "MCTransportSolverNonhomologous.from_config",
                                "MCTransportSolverNonhomologous.initialize_transport_state", "MCTransportSolverNonhomologous.run",
                                "MCTransportSolverNonhomologous.run_nonhomologous"],
    "nonhomologous/montecarlo_transport_state.py": ["MonteCarloTransportStateNonhomologous.__init__"],
    "nonhomologous/mc_rad_field_solver.py": ["MCRadiationFieldPropertiesSolver.__init__", "MCRadiationFieldPropertiesSolver.solve"],
}


def write_interface():
    """tests/golden/reference_interface_nonhomologous.json: the positional parameter names (self excluded) of INTERFACE,
    parsed from the reference's sources."""
    import ast
    import json

    from oracle.reference_loader import REF

    sigs = {}
    for rel, names in INTERFACE.items():
        tree = ast.parse(open(os.path.join(REF, "tardis", "transport", "montecarlo", "modes", rel)).read())
        for cls in (n for n in tree.body if isinstance(n, ast.ClassDef)):
            for fn in (n for n in cls.body if isinstance(n, ast.FunctionDef)):
                key = f"{cls.name}.{fn.name}"
                if key in names:
                    sigs[f"{rel}::{key}"] = [a.arg for a in fn.args.posonlyargs + fn.args.args if a.arg not in ("self", "cls")]
    assert len(sigs) == sum(len(v) for v in INTERFACE.values()), sorted(sigs)
    with open(os.path.join(HERE, "reference_interface_nonhomologous.json"), "w") as f:
        json.dump({"signatures": sigs}, f, indent=1, sort_keys=True)


def main(names):
    from oracle import reference_runner_nonhomologous as rrn
    from oracle.reference_runner import set_sigma_thomson

    for name in names:
        if name == "interface":
            write_interface()
            continue
        if name in RADFIELD_CASES:
            out = rrn.run_reference_radfield_nonhomologous(**radfield_inputs(name))
        else:
            model, packets, kw = case_inputs(name)
            sigma = kw.pop("sigma_thomson", None)
            if sigma is not None:
                set_sigma_thomson(sigma)
                import tardis.transport.montecarlo.modes.nonhomologous.virtual_packet as nh_vp

                nh_vp.SIGMA_THOMSON = sigma
            out = rrn.run_reference_nonhomologous(model, packets, **kw)
            print(name, "emitted", int((out["output_energies"] > 0).sum()), "reabsorbed", int((out["output_energies"] < 0).sum()))
            if name in BENCH_CASES:
                from make_golden import compress_table

                for k in ("j_blue", "edotlu"):
                    for kk, v in compress_table(out.pop(k)).items():
                        out[f"{k}__{kk}"] = v
        np.savez_compressed(os.path.join(HERE, f"nonhomologous_{name}.npz"), **out)


if __name__ == "__main__":
    names = sys.argv[1:] or [*CASES, *BENCH_CASES, *SIGMA_CASES, *RADFIELD_CASES, "interface"]
    for n in names:  # one process per case: the sigma cases need a fresh compile
        if len(names) == 1:
            main(names)
        else:
            import subprocess

            subprocess.run([sys.executable, os.path.abspath(__file__), n], check=True)
