"""Golden vectors of the nonhomologous mode's opacity build (oracle/reference_runner_nonhomologous.py::
run_reference_opacity in oracle/reference_runner_nonhomologous_opacity.py): tau_Sobolev divided by the velocity gradient, beta_Sobolev and the macro-atom
probabilities.

Run from the repository root where the reference tree exists:  python tests/golden/make_nonhomologous_opacity_golden.py
Writes tests/golden/nonhomologous_opacity_<case>.npz: the inputs are rebuilt from the synthetic generators by
`case_inputs`; the velocity gradient is the reference's NumbaRadial1DGeometry's, stored with the outputs.  A case whose
build raises stores the reference's message under `error`.  Stored: the tables the reference's own functions compute
(tau, beta) and the normalised probabilities the device keeps (STORED); the stimulated-emission factor is a restatement
(oracle/opacity_oracle.py) in the reference runner as well, so it is not stored.
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from tardis_b200 import synthetic  # noqa: E402

# name -> (seed, shells, lines, levels, line_interaction_type, velocity law)
CASES = {
    "macroatom": (71, 8, 1000, 400, "macroatom", "edge_cases"),
    "downbranch": (75, 6, 1500, 150, "downbranch", "perturbed"),
    "flat_shell": (79, 6, 1500, 150, "macroatom", "flat"),
}
DECELERATING, NEAR_FLAT, HOMOLOGOUS = 6, 4, 1  # shells of the "edge_cases" law
STORED = ("tau_sobolev", "beta_sobolev", "transition_probabilities")


def velocities(model, law, seed):
    """Shell-edge velocities of a case.  "perturbed": interior edges * (1 + 0.08 U(-1, 1)) (make_nonhomologous_velocities,
    which leaves at least one shell decelerating).  "edge_cases": the same, then one shell on v = r / t, one with |dv/dr|
    about 1e-6 of the others and one decelerating.  "flat": perturbed, one shell with v_inner == v_outer (dv/dr = 0)."""
    m = synthetic.make_nonhomologous_velocities(model, 0.08, seed=seed)
    v = np.concatenate([m.v_inner, m.v_outer[-1:]])
    r = np.concatenate([m.r_inner, m.r_outer[-1:]])
    t = model.time_explosion
    if law == "edge_cases":
        s = HOMOLOGOUS
        v[s], v[s + 1] = r[s] / t, r[s + 1] / t
        s = NEAR_FLAT
        v[s + 1] = v[s] + 1e-6 * (r[s + 1] - r[s]) / t
        s = DECELERATING
        v[s + 1] = v[s] * 0.95
    elif law == "flat":
        v[3] = v[2]
    return v[:-1].copy(), v[1:].copy()


def case_inputs(name):
    """(model, atomic, plasma) of a case; the model carries the case's v_inner / v_outer (its time_explosion is the t of the
    v = r / t shell; the build does not read it)."""
    import dataclasses

    seed, S, L, n_levels, mode, law = CASES[name]
    model = synthetic.make_model(S, L, mode, mu_tau=-4.0, seed=seed)
    v_inner, v_outer = velocities(model, law, seed + 3)
    atomic = synthetic.make_atomic_data(model.line_list_nu, n_levels, mode, seed=seed + 1)
    plasma = synthetic.make_plasma_state(atomic, S, 0.0, seed=seed + 2)
    return dataclasses.replace(model, v_inner=v_inner, v_outer=v_outer), atomic, plasma


def main(names):
    from oracle import reference_runner_nonhomologous as rrn
    from oracle import reference_runner_nonhomologous_opacity as rro

    for name in names:
        model, atomic, plasma = case_inputs(name)
        g = np.asarray(rrn.geometry(model).velocity_gradient, dtype=np.float64).copy()
        out = dict(velocity_gradient=g)
        try:
            tables = rro.run_reference_opacity(atomic, plasma, g, nlte=True)
            out.update({k: tables[k] for k in STORED})
        except ValueError as e:
            out["error"] = np.array(str(e))
        path = os.path.join(HERE, f"nonhomologous_opacity_{name}.npz")
        np.savez_compressed(path, **out)
        tau = out.get("tau_sobolev")
        print(name, f"{os.path.getsize(path) / 1e3:.0f} kB", "dvdr", g,
              out["error"] if tau is None else f"tau in [{tau.min():.3e}, {tau.max():.3e}]")


if __name__ == "__main__":
    main(sys.argv[1:] or list(CASES))
