"""Run the UNMODIFIED reference's nonhomologous opacity functions on synthetic atomic data and populations.

TEST INFRASTRUCTURE ONLY (see oracle/reference_loader.py).  Used by tests/golden/make_nonhomologous_opacity_golden.py.
"""
from __future__ import annotations

import numpy as np

from . import reference_loader


def run_reference_opacity(atomic, plasma, velocity_gradient, nlte=False):
    """The nonhomologous mode's opacity build (OpacitySolver.legacy_solve, modes/nonhomologous/opacity_solver.py): tau_Sobolev
    and beta_Sobolev from the UNMODIFIED `calculate_sobolev_line_opacity` / `calculate_beta_sobolev`
    (modes/nonhomologous/tau_sobolev.py:21-110), handed `velocity_gradient` as a quantity whose `.to(1 / u.s).value` is the
    plain [S] array; the raw macro-atom probabilities from the unmodified `probability_*` functions that
    BoundBoundMacroAtomSolver calls (macroatom_line_transitions.py).  As in oracle.reference_runner.run_reference_opacity, the
    stimulated-emission factor (oracle/opacity_oracle.py) and the normalisation (the solver's pandas expression,
    macroatom_solver.py:731-739) are evaluated next to them: their modules pull the atomic-data / HDF stack.
    A shell with velocity_gradient == 0 raises the reference's ValueError."""
    import sys
    import types

    import pandas as pd

    from . import opacity_oracle
    from .reference_loader import REF, _Q

    reference_loader.load()
    for name, sub in (("tardis.plasma.properties", "plasma/properties"), ("tardis.opacities.macro_atom", "opacities/macro_atom")):
        if name not in sys.modules:
            m = types.ModuleType(name)
            m.__path__ = [REF + "/tardis/" + sub]
            sys.modules[name] = m
    from tardis.opacities.macro_atom.macroatom_line_transitions import (
        probability_emission_down,
        probability_internal_down,
        probability_internal_up,
    )
    from tardis.transport.montecarlo.modes.nonhomologous.tau_sobolev import calculate_beta_sobolev, calculate_sobolev_line_opacity

    L = len(atomic.nu)
    stim = opacity_oracle.stimulated_emission_factor(atomic, plasma.level_number_density, nlte)
    # one species (Z = 14, ion 1): lines indexed (Z, ion, lower, upper), levels (Z, ion, level) as in atom_data
    lines = pd.DataFrame({"wavelength_cm": atomic.wavelength_cm, "f_lu": atomic.f_lu},
                         index=pd.MultiIndex.from_arrays([np.full(L, 14), np.full(L, 1), atomic.lower_level, atomic.upper_level],
                                                         names=["atomic_number", "ion_number", "level_number_lower", "level_number_upper"]))
    lnd = pd.DataFrame(plasma.level_number_density,
                       index=pd.MultiIndex.from_arrays([np.full(atomic.n_levels, 14), np.full(atomic.n_levels, 1), np.arange(atomic.n_levels)],
                                                       names=["atomic_number", "ion_number", "level_number"]))
    with np.errstate(divide="ignore", invalid="ignore"):
        tau_df = calculate_sobolev_line_opacity(lines, lnd, _Q(np.asarray(velocity_gradient, dtype=np.float64)), stim)
    beta = calculate_beta_sobolev(tau_df).to_numpy()
    tau = tau_df.to_numpy()
    nu, f_ul, f_lu = atomic.nu.reshape(-1, 1), atomic.f_ul.reshape(-1, 1), atomic.f_lu.reshape(-1, 1)
    e_lo, e_up = atomic.energy[atomic.lower_level].reshape(-1, 1), atomic.energy[atomic.upper_level].reshape(-1, 1)
    p_em = np.asarray(probability_emission_down(beta, nu, f_ul, e_up, e_lo))
    p_dn = np.asarray(probability_internal_down(beta, nu, f_ul, e_lo))
    p_up = np.asarray(probability_internal_up(beta, nu, f_lu, stim, plasma.j_blues, e_lo))
    rows = atomic.transition_line_idx
    raw = np.where((atomic.transition_type == -1)[:, None], p_em[rows], np.where((atomic.transition_type == 0)[:, None], p_dn[rows], p_up[rows]))
    df = pd.DataFrame(raw)
    df["source"] = atomic.source_block
    norm = df.div(df.groupby("source").transform("sum"))
    norm.replace(np.nan, 0.0, inplace=True)
    norm = norm.drop(columns=["source"]).to_numpy()
    return dict(stimulated_emission_factor=stim, tau_sobolev=tau, beta_sobolev=beta, raw_probabilities=raw, transition_probabilities=norm)
