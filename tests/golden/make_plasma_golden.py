"""Golden vectors of the unmodified classic plasma chain (the reference's tardis/plasma/properties/, no NLTE, no helium NLTE,
no continuum-interaction species):

    BetaRadiation -> ElectronTemperature -> BetaElectron -> GElectron                       general.py:20-121
    LevelBoltzmannFactorLTE | LevelBoltzmannFactorDiluteLTE -> PartitionFunction             partition_function.py:32-353
    PhiSahaLTE | RadiationFieldCorrection + PhiSahaNebular -> IonNumberDensity               ion_population.py:37-390
    LevelNumberDensity                                                                       level_population.py:13-70
    DilutePlanckianRadiationField / PlanckianRadiationField.calculate_mean_intensity         planck_rad_field.py:56-129

    python tests/golden/make_plasma_golden.py      # writes tests/golden/plasma_*.npz

Runs where the reference tree is available, through oracle/reference_loader.py and the stand-ins
oracle/reference_runner.py::run_reference_radfield installs (`tardis.util.base` holding only `intensity_black_body`, its
numexpr expression evaluated by numpy).  Stand-ins added here, for imports the chain never calls:
  * `tardis.plasma.properties` as a bare namespace package (its __init__ imports every property module, NLTE solvers included);
  * `tardis.plasma.electron_energy_distribution`, `tardis.plasma.equilibrium.level_populations`, `.rate_matrix`, `.rates`:
    empty modules whose attributes are placeholder classes (partition_function.py imports them for the NLTE factors only).
`LevelNumberDensity` is created without its __init__ (which wires it into a plasma graph) and with `initialize_indices` set,
as its __init__ sets it.  `IonNumberDensity` does not report its iteration count: the count is read by wrapping its
`calculate_with_n_electron` on the instance.  Each file holds the inputs (as the arrays tb200_set_plasma_data takes) and the
reference's outputs; rerunning gives byte-identical files.
"""
from __future__ import annotations

import importlib
import io
import os
import sys
import types
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

SMALL = dict(n_shells=8, n_levels=150, n_lines=400, atomic_numbers=(1, 2, 6, 8, 14))
# name -> sizes, seed and plasma options (the keyword arguments of oracle.plasma_oracle.solve, chi_0 by species)
CASES = {
    "plasma_nebular_dilute": dict(SMALL, seed=1),
    "plasma_nebular_lte": dict(SMALL, seed=2, excitation="lte", radiative_rates_type="blackbody"),
    "plasma_lte_dilute": dict(SMALL, seed=3, ionization="lte"),
    "plasma_lte_lte": dict(SMALL, seed=4, ionization="lte", excitation="lte", radiative_rates_type="blackbody"),
    "plasma_delta_treatment": dict(SMALL, seed=5, delta_treatment=0.7),
    "plasma_departure": dict(SMALL, seed=6, departure_coefficient=2.5),
    "plasma_chi0_species": dict(SMALL, seed=7, chi_0_species=(6, 2)),
    "plasma_zeta_outside": dict(SMALL, seed=8, t_rad_override={0: 1500.0, 5: 45000.0}),
    "plasma_fixed_ne": dict(SMALL, seed=9, fixed_ne=True),
    "plasma_threshold": dict(SMALL, seed=10, ion_zero_threshold=100.0),
    # a cool, nearly neutral gas: n_e starts at the number of nuclei and has to fall by orders of magnitude
    "plasma_many_iterations": dict(n_shells=6, n_levels=120, n_lines=200, atomic_numbers=(6, 8, 14), seed=11, ionization="lte",
                                   excitation="lte", t_range=(3e3, 4e3), w_range=(0.9, 1.0), log_density=(8.0, 8.5)),
    "plasma_bench_shape": dict(n_shells=20, n_levels=3000, n_lines=2000, atomic_numbers=tuple(range(1, 31)), seed=12),
}


def case_inputs(name):
    """The arrays of tb200_set_plasma_data / tb200_solve_plasma for one case, from tardis_b200.synthetic."""
    from tardis_b200 import synthetic as syn

    c = CASES[name]
    S, n_levels, L, seed = c["n_shells"], c["n_levels"], c["n_lines"], c["seed"]
    model = syn.make_model(S, L, "macroatom", seed=100 + seed)
    atomic = syn.make_atomic_data(model.line_list_nu, n_levels, seed=200 + seed)
    st = syn.make_plasma_structure(atomic, S, c["atomic_numbers"], seed=300 + seed, log_density=c.get("log_density", (3.0, 9.0)))
    rng = np.random.default_rng(400 + seed)
    t_rad = rng.uniform(*c.get("t_range", (8e3, 1.3e4)), S)
    w = rng.uniform(*c.get("w_range", (0.05, 0.5)), S)
    for s, t in c.get("t_rad_override", {}).items():
        t_rad[s] = t
    inp = dict(level_energy=st.level_energy, level_ion=st.level_ion, g=atomic.g, metastable=atomic.metastable,
               ion_atomic_number=st.ion_atomic_number, ion_charge=st.ion_charge, ionization_energy=st.ionization_energy,
               number_density=st.number_density, zeta_temperatures=st.zeta_temperatures, zeta=st.zeta, t_rad=t_rad, w=w,
               line_nu=model.line_list_nu, lines_lower_level_index=atomic.lower_level, lines_upper_level_index=atomic.upper_level)
    opts = dict(ionization=c.get("ionization", "nebular"), excitation=c.get("excitation", "dilute-lte"),
                radiative_rates_type=c.get("radiative_rates_type", "dilute-blackbody"), link_t_rad_t_electron=0.9,
                ion_zero_threshold=c.get("ion_zero_threshold", 1e-20))
    for k in ("delta_treatment", "departure_coefficient"):
        if k in c:
            opts[k] = c[k]
    chi_0 = 1.9020591570241798e-11
    if "chi_0_species" in c:
        z, q = c["chi_0_species"]
        chi_0 = float(st.ionization_energy[(st.ion_atomic_number == z) & (st.ion_charge == q)][0])
    opts["chi_0"] = chi_0
    if c.get("fixed_ne"):  # one shell at n_e = 0: Phi / n_e is inf or 0 / 0 there, which np.nan_to_num maps to DBL_MAX and 0
        opts["electron_densities"] = 10 ** rng.uniform(7.0, 9.0, S)
        opts["electron_densities"][1] = 0.0
    return inp, opts


def install_stand_ins():
    from oracle import reference_loader
    from oracle.reference_runner import run_reference_radfield

    run_reference_radfield(np.ones(1), np.full(1, 1e15), np.ones((1, 1)), 1.0e6, 1.0, np.full(1, 1e45), np.full(1, 1e15))  # tardis.util.base
    ref = os.path.join(reference_loader.REF, "tardis")
    m = types.ModuleType("tardis.plasma.properties")
    m.__path__ = [os.path.join(ref, "plasma", "properties")]
    sys.modules[m.__name__] = m

    class Placeholders(types.ModuleType):
        def __getattr__(self, k):
            if k.startswith("__"):
                raise AttributeError(k)
            return type(k, (), {})

    for n in ("tardis.plasma.electron_energy_distribution", "tardis.plasma.equilibrium", "tardis.plasma.equilibrium.level_populations",
              "tardis.plasma.equilibrium.rate_matrix", "tardis.plasma.equilibrium.rates"):
        sys.modules[n] = Placeholders(n)
    return reference_loader._Q


def run_reference(inp, opts, Q, chi_0_species=(20, 2)):
    import pandas as pd

    gen = importlib.import_module("tardis.plasma.properties.general")
    pf = importlib.import_module("tardis.plasma.properties.partition_function")
    ip = importlib.import_module("tardis.plasma.properties.ion_population")
    lp = importlib.import_module("tardis.plasma.properties.level_population")
    from tardis.plasma.radiation_field.planck_rad_field import DilutePlanckianRadiationField, PlanckianRadiationField

    zs, qs, lion = inp["ion_atomic_number"], inp["ion_charge"], inp["level_ion"]
    levels = pd.MultiIndex.from_arrays([zs[lion], qs[lion], np.arange(len(lion))], names=["atomic_number", "ion_number", "level_number"])
    g = pd.Series(inp["g"], index=levels)
    energy = pd.Series(inp["level_energy"], index=levels)
    meta = pd.Series(inp["metastable"].astype(bool), index=levels)
    ion_index = pd.MultiIndex.from_arrays([zs, qs], names=["atomic_number", "ion_number"])
    has_chi = qs > 0
    ionization_data = pd.Series(inp["ionization_energy"][has_chi], index=ion_index[has_chi])
    elements = pd.unique(zs)
    number_density = pd.DataFrame(inp["number_density"], index=pd.Index(elements, name="atomic_number"))
    t_rad, w = inp["t_rad"], inp["w"]

    beta_rad = gen.BetaRadiation(None).calculate(t_rad)
    if opts["excitation"] == "dilute-lte":
        lbf = pf.LevelBoltzmannFactorDiluteLTE(None).calculate(levels, g, energy, beta_rad, w, meta)
    else:
        lbf = pf.LevelBoltzmannFactorLTE.calculate(energy, g, beta_rad, levels)
    Z = pf.PartitionFunction(None).calculate(lbf)
    g_e = gen.GElectron(None).calculate(beta_rad)
    if opts["ionization"] == "nebular":
        t_e = gen.ElectronTemperature(None).calculate(t_rad, opts["link_t_rad_t_electron"])
        beta_e = gen.BetaElectron(None).calculate(t_e)
        rfc = ip.RadiationFieldCorrection(None, departure_coefficient=opts.get("departure_coefficient"), chi_0_species=chi_0_species,
                                          delta_treatment=opts.get("delta_treatment"))
        delta = rfc.calculate(w, ionization_data, beta_rad, t_e, t_rad, beta_e)
        zeta_data = pd.DataFrame(inp["zeta"], index=ion_index, columns=inp["zeta_temperatures"])
        import warnings

        with warnings.catch_warnings():
            warnings.simplefilter("ignore")  # "t_rads outside of zeta factor interpolation"
            phi = ip.PhiSahaNebular.calculate(t_rad, w, zeta_data, t_e, delta, g_e, beta_rad, Z, ionization_data)
    else:
        phi = ip.PhiSahaLTE.calculate(g_e, beta_rad, Z, ionization_data)
    fixed = opts.get("electron_densities")
    ind = ip.IonNumberDensity(None, ion_zero_threshold=opts["ion_zero_threshold"],
                              electron_densities=None if fixed is None else pd.Series(fixed))
    calls = []
    inner = ind.calculate_with_n_electron

    def counted(*a, **k):
        calls.append(1)
        return inner(*a, **k)

    ind.calculate_with_n_electron = counted
    ion_nd, n_e = ind.calculate(phi, Z, number_density)
    lnd_prop = lp.LevelNumberDensity.__new__(lp.LevelNumberDensity)
    lnd_prop.initialize_indices = True
    lnd = lnd_prop.calculate(lbf, ion_nd, levels, Z)
    nu = inp["line_nu"]
    if opts["radiative_rates_type"] == "dilute-blackbody":
        j_blues = DilutePlanckianRadiationField(Q(t_rad), w).calculate_mean_intensity(nu)
    else:
        j_blues = PlanckianRadiationField(Q(t_rad)).calculate_mean_intensity(nu)
    return dict(electron_densities=np.asarray(n_e, dtype=np.float64), ion_number_density=np.asarray(ion_nd.values, dtype=np.float64),
                level_number_density=np.asarray(lnd.values, dtype=np.float64), j_blues=np.asarray(j_blues, dtype=np.float64),
                iterations=np.int64(0 if fixed is not None else len(calls)), partition_function=np.asarray(Z.values, dtype=np.float64))


def write(name, arrays):
    # np.savez_compressed stamps the zip members with the current time; fixed stamps make the file reproducible
    path = os.path.join(HERE, name + ".npz")
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k, v in arrays.items():
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(v), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())
    return path


def main():
    Q = install_stand_ins()
    for name in CASES:
        inp, opts = case_inputs(name)
        out = run_reference(inp, opts, Q, CASES[name].get("chi_0_species", (20, 2)))
        stored = {**inp, **{"opt_" + k: np.asarray(v) for k, v in opts.items()}, **out}
        path = write(name, stored)
        pops = out["ion_number_density"]
        print(f"{name}: {os.path.getsize(path) / 1e3:.0f} kB; iterations {int(out['iterations'])}, zero ions {int((pops == 0).sum())} "
              f"of {pops.size}, n_e {out['electron_densities'].min():.3e} .. {out['electron_densities'].max():.3e}")


if __name__ == "__main__":
    main()
