"""The classic plasma on the device (`tb200_set_plasma_data` / `tb200_solve_plasma`) from the reference's own frames.

`plasma_data` maps the frames the reference's plasma reads -- atomic_data.levels (MultiIndex atomic_number, ion_number,
level_number; columns energy, g, metastable), ionization_data (Series on (atomic_number, ion_number): the energy into the ion),
zeta_data (DataFrame on (atomic_number, ion_number), columns the temperatures) and number_density (DataFrame on atomic_number,
columns the shells) -- to the arrays of `Engine.set_plasma_data`; `as_frames` turns what `Engine.solve_plasma(download=True)`
returns into frames indexed as the reference's (ion_number_density on (atomic_number, ion_number), level_number_density on the
levels' index).  Only the graphs the device builds are accepted: no NLTE species, helium_treatment "none", no
continuum-interaction species (their plasmas solve rate equations: plasma/properties/nlte_rate_equation_solver.py,
helium_nlte.py, the IIP properties)."""
from __future__ import annotations

import numpy as np
import pandas as pd


def check_supported(nlte_species=(), helium_treatment="none", continuum_interaction_species=()):
    if len(nlte_species):
        raise NotImplementedError(f"NLTE species {list(nlte_species)}: the device solves the classic plasma without NLTE only")
    if helium_treatment != "none":
        raise NotImplementedError(f"helium_treatment {helium_treatment!r}: the device solves helium_treatment 'none' only")
    if len(continuum_interaction_species):
        raise NotImplementedError("continuum-interaction species: the continuum mode's plasma is not built on the device")


def plasma_data(levels: pd.DataFrame, ionization_data: pd.Series, number_density: pd.DataFrame, zeta_data: pd.DataFrame | None = None,
                chi_0_species=(20, 2), nlte_species=(), helium_treatment="none", continuum_interaction_species=()) -> dict:
    """-> keyword arguments of `Engine.set_plasma_data` (the level rows must be those of `Engine.set_atomic_data`)."""
    check_supported(nlte_species, helium_treatment, continuum_interaction_species)
    idx = levels.index
    z, q = idx.get_level_values("atomic_number").values, idx.get_level_values("ion_number").values
    ion_index = pd.MultiIndex.from_arrays([z, q], names=["atomic_number", "ion_number"]).unique()  # the partition function's rows
    level_ion = ion_index.get_indexer(pd.MultiIndex.from_arrays([z, q]))
    ion_z = ion_index.get_level_values(0).values.astype(np.int64)
    ion_q = ion_index.get_level_values(1).values.astype(np.int64)
    chi = ionization_data.reindex(ion_index).values.astype(np.float64)  # PhiSahaLTE's reindex (ion_population.py:74-76)
    chi[ion_q == 0] = np.nan
    elements = pd.unique(ion_z)
    missing = set(elements) - set(number_density.index)
    if missing:
        raise ValueError(f"number_density has no row for atomic numbers {sorted(missing)}")
    out = dict(level_energy=levels["energy"].values.astype(np.float64), level_ion=level_ion.astype(np.int64), ion_atomic_number=ion_z,
               ion_charge=ion_q, ionization_energy=chi, number_density=number_density.loc[elements].values.astype(np.float64))
    if zeta_data is not None:
        phi_index = ion_index[ion_q > 0]
        absent = phi_index.difference(zeta_data.index)
        if len(absent):
            raise ValueError(f"zeta_data has no row for ions {list(absent)[:5]} (the reference's .loc would raise)")
        zeta = np.full((len(ion_index), zeta_data.shape[1]), np.nan)
        zeta[ion_q > 0] = zeta_data.loc[phi_index].values.astype(np.float64)
        out.update(zeta_temperatures=zeta_data.columns.values.astype(np.float64), zeta=zeta)
    if tuple(chi_0_species) != (20, 2):  # RadiationFieldCorrection._set_chi_0 (ion_population.py:211-215)
        out["chi_0"] = float(ionization_data.loc[tuple(chi_0_species)])
    return out


def as_frames(result: dict, levels_index: pd.MultiIndex) -> dict:
    """The downloaded arrays of `Engine.solve_plasma(download=True)` as the reference's frames."""
    z = levels_index.get_level_values("atomic_number").values
    q = levels_index.get_level_values("ion_number").values
    ion_index = pd.MultiIndex.from_arrays([z, q], names=["atomic_number", "ion_number"]).unique()
    return dict(electron_densities=pd.Series(result["electron_densities"]),
                ion_number_density=pd.DataFrame(result["ion_number_density"], index=ion_index),
                level_number_density=pd.DataFrame(result["level_number_density"], index=levels_index),
                j_blues=result.get("j_blues"), iterations=result.get("iterations"))
