"""CPU restatement of the classic plasma update (nebular / LTE ionisation, dilute-LTE / LTE excitation, n_e fixed point,
dilute black-body J_blue).

TEST INFRASTRUCTURE ONLY (tests/test_plasma.py, scripts/plasma_probe.py).  numpy / pandas restatement of, paths relative to
the reference's tardis/:
    BetaRadiation, ElectronTemperature, BetaElectron, GElectron      plasma/properties/general.py:20-121
    LevelBoltzmannFactorLTE / ...DiluteLTE                           plasma/properties/partition_function.py:50-60, 107-114
    PartitionFunction (pandas group sum)                             partition_function.py:350-353
    PhiSahaLTE                                                       plasma/properties/ion_population.py:56-86
    PhiSahaNebular (+ get_zeta_values: interp1d, NaN -> 1.0)          ion_population.py:141-182
    RadiationFieldCorrection                                         ion_population.py:199-258
    IonNumberDensity                                                 ion_population.py:296-390
    LevelNumberDensity                                               plasma/properties/level_population.py:33-68
    radiative_rates_type dilute-blackbody / blackbody                simulation/base.py:378-401, plasma/radiation_field/planck_rad_field.py:56-72
Inputs are the arrays of tb200_set_plasma_data (tardis_b200.plasma.plasma_data builds them from the reference's frames).
Pinned by tests/golden/plasma_*.npz, produced by the unmodified property classes (tests/golden/make_plasma_golden.py).
Unlike the reference the loop stops after `max_iterations` (the device's cap) with PlasmaIonizationError."""
from __future__ import annotations

import numpy as np
import pandas as pd
from scipy import interpolate

K_B, H, M_E, C = 1.3806488e-16, 6.62606957e-27, 9.10938291e-28, 2.99792458e10  # CODATA-2010 cgs (tardis/constants.py:1)
CHI_0_CA_II = 1.9020591570241798e-11  # ion_population.py:212-213
MAX_ITERATIONS = 1000                 # tbp::MAX_NE_ITERATIONS


class PlasmaIonizationError(Exception):
    pass


def solve(level_energy, level_ion, g, metastable, ion_atomic_number, ion_charge, ionization_energy, number_density, t_rad, w, *,
          zeta_temperatures=None, zeta=None, ionization="nebular", excitation="dilute-lte", radiative_rates_type="dilute-blackbody",
          link_t_rad_t_electron=0.9, delta_treatment=None, departure_coefficient=None, chi_0=CHI_0_CA_II, ion_zero_threshold=1e-20,
          electron_densities=None, line_nu=None, max_iterations=MAX_ITERATIONS):
    """-> dict(electron_densities [S], ion_number_density [n_ions, S], level_number_density [n_levels, S],
    j_blues [L, S] or None, iterations)"""
    t_rad, w = np.asarray(t_rad, dtype=np.float64), np.asarray(w, dtype=np.float64)
    S = len(t_rad)
    ion_index = pd.MultiIndex.from_arrays([np.asarray(ion_atomic_number), np.asarray(ion_charge)], names=["atomic_number", "ion_number"])
    level_ion = np.asarray(level_ion)
    level_index = pd.MultiIndex.from_arrays([ion_index.get_level_values(0)[level_ion], ion_index.get_level_values(1)[level_ion],
                                             np.arange(len(level_ion))], names=["atomic_number", "ion_number", "level_number"])
    # general.py
    beta_rad = 1 / (K_B * t_rad)
    t_e = t_rad * link_t_rad_t_electron
    beta_e = 1 / (K_B * t_e)
    g_e = ((2 * np.pi * M_E / beta_rad) / (H**2)) ** 1.5
    # partition_function.py: g exp(outer(E, -beta)), non-metastable rows times W (dilute-lte)
    lbf = pd.DataFrame(np.asarray(g)[np.newaxis].T * np.exp(np.outer(np.asarray(level_energy), -beta_rad)), index=level_index,
                       columns=np.arange(S), dtype=np.float64)
    if excitation == "dilute-lte":
        lbf[~np.asarray(metastable, dtype=bool)] *= w
    Z = lbf.groupby(level=["atomic_number", "ion_number"]).sum()
    # PhiSahaLTE: Z_j / Z_{j-1} per element block, times 2 g_e exp(chi * -beta) of the ions that have an ionisation energy
    zv = Z.values
    first = np.asarray(ion_charge) == 0
    phi_rows = np.flatnonzero(~first)
    chi = np.asarray(ionization_energy, dtype=np.float64)[phi_rows]
    phis = zv[phi_rows] / zv[phi_rows - 1]
    phi = phis * (2 * g_e * np.exp(np.outer(chi, -beta_rad)))
    if ionization == "nebular":
        zt = np.asarray(zeta_temperatures, dtype=np.float64)
        zeta_v = interpolate.interp1d(zt, np.asarray(zeta, dtype=np.float64)[phi_rows], bounds_error=False, fill_value=np.nan)(t_rad)
        zeta_v = zeta_v.astype(float)
        zeta_v[np.isnan(zeta_v)] = 1.0
        if delta_treatment is None:  # RadiationFieldCorrection
            dep = 1.0 / w if departure_coefficient is None else departure_coefficient
            delta = -np.ones((len(chi), S))
            less = chi < chi_0
            factor_a = t_e / (dep * w * t_rad)
            delta[~less] = factor_a * np.exp(np.outer(chi[~less], beta_rad - beta_e))
            delta[less] = 1 - np.exp(np.outer(chi[less], beta_rad) - beta_rad * chi_0)
            delta[less] += factor_a * np.exp(np.outer(chi[less], beta_rad) - chi_0 * beta_e)
        else:
            delta = np.ones((len(chi), S)) * delta_treatment
        phi = phi * w * ((zeta_v * delta) + w * (1 - zeta_v)) * (t_e / t_rad) ** 0.5
    # IonNumberDensity.calculate_with_n_electron: blocks of Phi rows per element (calculate_block_ids_from_dataframe).  The
    # reference's frames hand numpy Fortran-ordered .values, so its axis-0 sums are numpy's pairwise sums down the rows.
    phi = np.asfortranarray(phi)
    nd_frame = pd.DataFrame(np.asarray(number_density, dtype=np.float64))
    nd = nd_frame.values
    phi_z = np.asarray(ion_atomic_number)[phi_rows]
    block_ids = np.hstack(([0], np.where(np.diff(phi_z) != 0.0)[0] + 1, [len(phi_z)]))
    charges = np.asarray(ion_charge).reshape(-1, 1)

    def populations(n_e):
        pops = np.empty_like(np.asfortranarray(zv))
        phi_e = np.nan_to_num(phi / n_e)
        for i, start in enumerate(block_ids[:-1]):
            end = block_ids[i + 1]
            prod = np.cumprod(phi_e[start:end], 0)
            tmp = np.empty((prod.shape[0] + 1, prod.shape[1]))
            tmp[0] = nd[i] / (1 + np.sum(prod, axis=0))
            tmp[1:] = tmp[0] * prod
            pops[start + i:end + 1 + i] = tmp
        pops[pops < ion_zero_threshold] = 0.0
        return pops

    iterations = 0
    if electron_densities is None:
        n_e = nd_frame.sum(axis=0).values
        while True:
            pops = populations(n_e)
            new = (pops * charges).sum(axis=0)
            if np.any(np.isnan(new)):
                raise PlasmaIonizationError('n_electron just turned "nan" - aborting')
            iterations += 1
            if np.all(np.abs(new - n_e) / n_e < 0.05):
                break
            if iterations >= max_iterations:
                raise PlasmaIonizationError(f"n_electron did not converge within {max_iterations} iterations")
            n_e = 0.5 * (new + n_e)
    else:
        n_e = np.asarray(electron_densities, dtype=np.float64)
        pops = populations(n_e)
    # LevelNumberDensity
    lnd = lbf.values / zv[level_ion] * pops[level_ion]
    j_blues = None
    if line_nu is not None and radiative_rates_type != "detailed":
        nu = np.asarray(line_nu, dtype=np.float64)[np.newaxis].T
        intensity = 2 * H / C**2 * nu**3 / (np.exp(H * nu * (1 / (K_B * t_rad))) - 1)  # util/base.py:299-302
        j_blues = w * intensity if radiative_rates_type == "dilute-blackbody" else intensity
    return dict(electron_densities=np.asarray(n_e, dtype=np.float64), ion_number_density=pops, level_number_density=lnd, j_blues=j_blues,
                iterations=iterations)

