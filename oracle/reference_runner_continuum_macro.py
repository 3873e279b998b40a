"""Run the UNMODIFIED reference ContinuumMacroAtomSolver.solve (opacities/macro_atom/macroatom_solver.py:861-1020) on
synthetic inputs: the first iteration (metadata, sorting, cooling block), then the second, which takes
_solve_next_macroatom_iteration (:1358-1668) -- the step tb200_build_opacity replaces in the continuum mode.

TEST INFRASTRUCTURE ONLY (needs the reference tree).  macroatom_solver.py and macroatom_continuum_transitions.py are
imported unmodified through oracle/reference_loader.py plus three stand-in modules for imports the solver does not use
here: tardis.io.atom_data (AtomData, a type hint), tardis.opacities.macro_atom.base (get_macro_atom_data /
initialize_transition_probabilities, used by the legacy solver only) and tardis.io.hdf_writer_mixin (HDFWriterMixin, a
base class of MacroAtomState).  Every step runs as the reference wrote it under pandas 3; nothing is restated.
beta_Sobolev and the stimulated-emission factor given to `solve` are oracle/opacity_oracle.py's on the case's populations."""
from __future__ import annotations

import sys
import types

import numpy as np
import pandas as pd

from oracle import opacity_oracle as oo
from oracle import reference_loader


def load_solver_module():
    reference_loader.load()
    stand_ins = {"tardis.io.atom_data": {"AtomData": object},
                 "tardis.opacities.macro_atom.base": {"get_macro_atom_data": None, "initialize_transition_probabilities": None},
                 "tardis.io.hdf_writer_mixin": {"HDFWriterMixin": object}}
    for name, attrs in stand_ins.items():
        if name not in sys.modules:
            m = types.ModuleType(name)
            m.__dict__.update(attrs)
            sys.modules[name] = m
    import tardis.opacities.macro_atom.macroatom_solver as ms

    return ms


def line_inputs(ci, it):
    p = ci.plasma[it]
    stim = oo.stimulated_emission_factor(ci.atomic, p.level_number_density)
    tau = oo.tau_sobolev(ci.atomic, p.level_number_density, p.time_explosion, stim)
    return pd.DataFrame(p.j_blues), pd.DataFrame(oo.beta_sobolev(tau)), stim


def run(ci):
    """-> dict: the solver after its second iteration, the metadata, the unnormalised probabilities of the second iteration
    (the input of its first normalize_transition_probabilities call), the normalised ones, the normalised deactivation
    table and X."""
    ms = load_solver_module()
    solver = ms.ContinuumMacroAtomSolver(ci.levels, ci.lines, ci.photoionization_data, ci.ionization_energies)
    seen = []
    cls = ms.BoundBoundMacroAtomSolver
    original = cls.__dict__["normalize_transition_probabilities"]

    def recording(probabilities_df, metadata):
        seen.append(probabilities_df.drop(columns=["source"], errors="ignore").to_numpy(copy=True))
        return original.__func__(probabilities_df, metadata)

    states = []
    for it in range(len(ci.rates)):
        jb, beta, stim = line_inputs(ci, it)
        seen.clear()
        cls.normalize_transition_probabilities = staticmethod(recording)
        try:
            states.append(solver.solve(jb, beta, stim, **ci.rates[it]))
        finally:
            cls.normalize_transition_probabilities = original
    st = states[-1]
    return dict(solver=solver, metadata=solver.computed_metadata[0], raw=seen[0],
                normalized=st.transition_probabilities.to_numpy(), deactivation=st.normalized_deactivating_probs.to_numpy()
                if hasattr(st, "normalized_deactivating_probs") else None, state=st)
