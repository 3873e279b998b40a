"""CPU restatement of the nonhomologous mode's opacity build.

TEST INFRASTRUCTURE ONLY.  numpy restatement of, paths relative to /root/reference/tardis/:
    calculate_sobolev_line_opacity     transport/montecarlo/modes/nonhomologous/tau_sobolev.py:21-75
and, unchanged from the homologous build (oracle/opacity_oracle.py), the stimulated-emission factor, beta_Sobolev
(modes/nonhomologous/tau_sobolev.py:77-110 is the homologous function) and the macro-atom probabilities of the same
BoundBoundMacroAtomSolver.  Pinned by tests/golden/nonhomologous_opacity_*.npz
(tests/golden/make_nonhomologous_opacity_golden.py)."""
from __future__ import annotations

import numpy as np

from .opacity_oracle import SOBOLEV_COEFFICIENT, beta_sobolev, macro_atom_probabilities, stimulated_emission_factor


def tau_sobolev(atomic, level_number_density, velocity_gradient, stim):
    """modes/nonhomologous/tau_sobolev.py:55-67: ((((lambda f_lu) * COEFF) / dvdr) * stim) * n_lower, numpy's order -- divided
    by the per-shell velocity gradient [S] (1/s) where the homologous mode multiplies by time_explosion"""
    with np.errstate(divide="ignore", invalid="ignore"):
        tau = ((atomic.wavelength_cm * atomic.f_lu)[np.newaxis].T * SOBOLEV_COEFFICIENT / np.asarray(velocity_gradient, dtype=np.float64)
               * stim * level_number_density.take(atomic.lower_level, axis=0))
    if np.any(np.isnan(tau)) or np.any(np.isinf(np.abs(tau))):
        raise ValueError("Some tau_sobolevs are nan, inf, -inf in tau_sobolevs. Something went wrong!")
    return tau


def build(atomic, plasma, velocity_gradient, nlte=False):
    """The mode's tables: its own tau, the rest as oracle.opacity_oracle.build"""
    stim = stimulated_emission_factor(atomic, plasma.level_number_density, nlte)
    tau = tau_sobolev(atomic, plasma.level_number_density, velocity_gradient, stim)
    beta = beta_sobolev(tau)
    raw, norm = macro_atom_probabilities(atomic, beta, stim, plasma.j_blues)
    return dict(stimulated_emission_factor=stim, tau_sobolev=tau, beta_sobolev=beta, raw_probabilities=raw, transition_probabilities=norm)
