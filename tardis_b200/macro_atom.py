"""Drop-ins for the continuum macro atom on the GPU: the absorbing-Markov-chain solve, create_absorbing_probs
(tardis/opacities/macro_atom/absorbing_markov_chain.py:19-134), and the whole per-iteration step that feeds it,
ContinuumMacroAtomSolver._solve_next_macroatom_iteration (opacities/macro_atom/macroatom_solver.py:1358-1668).

On the reference side either swap is one line:

    macroatom_solver.create_absorbing_probs = tardis_b200.macro_atom.create_absorbing_probs
    macroatom_solver.ContinuumMacroAtomSolver._solve_next_macroatom_iteration = tardis_b200.macro_atom.solve_next_macroatom_iteration

Same signature and return values: the [S, n, n] ndarray X and `deactivating_probs`, the input with its internal rows
multiplied by 0 (not normalised: the reference normalises it afterwards).  X is built by `tb200_build_absorbing_markov`.
The engine that later transports the iteration (the IIP mirror, `montecarlo.montecarlo_transport`) recognises this very
array when it comes back in OpacityStateNumbaIIP.absorbing_markov_probabilities and rebuilds the table in HBM from the
[T, S] input instead of uploading the [S, n, n] one."""
from __future__ import annotations

import numpy as np

_last = None  # (X returned by the last call, the inputs that rebuild it on any engine)


def _continuum_stub(S: int):
    """The smallest continuum model an engine accepts: the chain's build reads only the macro-atom tables of the model."""
    from types import SimpleNamespace

    return SimpleNamespace(
        bf_threshold_list_nu=np.array([3e15]), photo_ion_nu_threshold_mins=np.array([3e15]),
        photo_ion_nu_threshold_maxs=np.array([4e15]), photo_ion_block_references=np.array([0, 2]), chi_bf=np.zeros((2, S)),
        x_sect=np.zeros(2), phot_nus=np.array([3e15, 4e15]), ff_opacity_factor=np.zeros(S), emissivities=np.zeros((2, S)),
        photo_ion_activation_idx=np.zeros(1, dtype=np.int64), k_packet_idx=0, absorbing_markov_probabilities=None)


def create_absorbing_probs(transition_probabilities, metadata, max_workers: int = 1, engine=None):
    """`transition_probabilities`: DataFrame [T, S] of the normalised probabilities; `metadata`: DataFrame with
    source_level_idx, destination_level_idx, transition_type, rows grouped by source.  `max_workers` is accepted for the
    reference's signature (no host threads are used).  `engine`: the `Engine` to build on (default: this process's
    engine of device 0); its model is replaced by a stub and the option keep_opacity_tables is set, so that X can be read
    back."""
    global _last
    from .montecarlo import get_engine

    eng = engine if engine is not None else get_engine()
    tp = np.ascontiguousarray(transition_probabilities.to_numpy(dtype=np.float64))
    src = metadata.source_level_idx.to_numpy().astype(np.int64)
    tt = metadata.transition_type.to_numpy().astype(np.int64)
    dst = np.where(tt >= 0, metadata.destination_level_idx.fillna(-1).to_numpy(), -1).astype(np.int64)
    T, S = tp.shape
    n = int(src.max()) + 1
    edges = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(np.bincount(src, minlength=n), out=edges[1:])
    radii = np.arange(1, S + 2, dtype=np.float64) * 1e14
    eng.set_option("keep_opacity_tables", 1)
    eng.set_model(r_inner=radii[:-1], r_outer=radii[1:], time_explosion=1.0, electron_density=np.ones(S), line_list_nu=np.array([1e15]),
                  tau_sobolev=np.zeros((1, S)), line_interaction_type="macroatom", transition_probabilities=None,
                  line2macro_level_upper=np.zeros(1, dtype=np.int64), macro_block_edge_index=edges, transition_type=tt,
                  destination_level_id=dst, transition_line_id=np.zeros(T, dtype=np.int64), continuum=_continuum_stub(S),
                  t_electrons=np.full(S, 1e4), enable_full_relativity=True)
    inputs = dict(transition_probabilities=tp, source_level_idx=src, destination_level_idx=dst, transition_type=tt, n_states=n)
    eng.build_absorbing_markov(**inputs)
    X = eng.download_absorbing_markov(deactivating=False)["absorbing_markov_probabilities"]
    _last = (X, inputs)
    internal_mask = metadata.transition_type >= 0
    deactivating_probs = transition_probabilities.copy()
    deactivating_probs[internal_mask] *= 0  # as the reference returns them (absorbing_markov_chain.py:128-129)
    return X, deactivating_probs


def built_inputs(matrix, transition_type):
    """The inputs that rebuild `matrix` on an engine, when `matrix` is (a view of the whole of) the X the last
    `create_absorbing_probs` returned and the model's rows are its rows; else None."""
    if _last is None or matrix is None:
        return None
    X, inputs = _last
    m = np.asarray(matrix)
    same = m is X or (m.shape == X.shape and m.dtype == X.dtype and m.__array_interface__["data"][0] == X.__array_interface__["data"][0]
                      and m.strides == X.strides)
    if not same:
        return None
    tt = np.asarray(transition_type)
    if tt.shape != inputs["transition_type"].shape or not np.array_equal(tt, inputs["transition_type"]):
        return None
    return inputs


class WithoutMatrix:
    """The continuum fields of an OpacityStateNumbaIIP with absorbing_markov_probabilities hidden (the engine builds it)."""

    def __init__(self, state):
        self._state = state

    def __getattr__(self, name):
        if name == "absorbing_markov_probabilities":
            return None
        return getattr(self._state, name)


# ---- the continuum macro atom's rows (tb200_build_opacity in the continuum mode) -----------------------------------
RATE_TABLES = ("stim_recomb_corrected_photoionization_rate_coeff", "spontaneous_recombination_coeff", "coll_deexc_coeff",
               "coll_exc_coeff", "coll_ion_coeff", "coll_recomb_coeff")
COOLING_TABLES = ("fb_cool_probs_arr", "coll_exc_cool_arr", "coll_ion_cool_arr")


def continuum_row_map(solver, metadata, rates) -> dict:
    """The row map of tb200_continuum_rows for the rows of `metadata` (the reference's macro_atom_transition_metadata):
    which row of which rate / cooling table every row reads, and its energy factor -- by the lookups
    ContinuumMacroAtomSolver._solve_next_macroatom_iteration (opacities/macro_atom/macroatom_solver.py:1533-1631) makes,
    run on probe frames: the rate frames' own indexes carrying their row positions (or ones), so that pandas' label
    alignment, .loc and .iloc pick rows exactly as they do for the rates.  `solver` carries what the reference's first
    iteration left (photoionization_data_level_energies, _delta_E_yg, _delta_E_yg_ionization, _coll_energies_lower,
    _coll_ion_energies); `rates`: the rate frames / cooling arrays by their `solve` argument names (only their indexes and
    shapes are read).  Raises ValueError where the reference's lookup would not give one finite row per metadata row."""
    import pandas as pd

    tt = metadata.transition_type.to_numpy().astype(np.int64)
    T = len(tt)
    key, energy = np.full(T, -1, dtype=np.int64), np.zeros(T)

    def probe(name, how, energies):
        """`how(frame, energies)`: the reference's expression with `frame` in place of the rate frame"""
        idx = rates[name].index
        pos = pd.DataFrame({0: np.arange(len(idx), dtype=np.float64)}, index=idx)
        ones = pd.DataFrame({0: np.ones(len(idx))}, index=idx)
        unit = pd.Series(1.0, index=energies.index) if isinstance(energies, pd.Series) else np.ones(len(energies))
        return how(pos, unit)[0].to_numpy(), how(ones, energies)[0].to_numpy()

    def put(t, k, e):
        rows = np.flatnonzero(tt == t)
        if len(k) != len(rows) or not (np.isfinite(k).all() and np.isfinite(e).all()):
            raise ValueError(f"continuum rows of type {t}: the reference's lookup gives {len(k)} rows for {len(rows)}, or a missing label")
        key[rows], energy[rows] = k.astype(np.int64), e

    md = metadata
    pi_idx = md.photoionization_key_idx[tt == 2].to_numpy()
    sources = pd.MultiIndex.from_tuples(md.source[tt == 2])
    put(2, *probe(RATE_TABLES[0], lambda f, e: f.loc[sources].multiply(e, axis=0), solver.photoionization_data_level_energies.iloc[pi_idx]))
    put(-7, *probe(RATE_TABLES[1], lambda f, e: f.multiply(e, axis=0), solver._delta_E_yg_ionization.values))
    dests = pd.MultiIndex.from_tuples(md.destination[tt == 3])
    put(3, *probe(RATE_TABLES[1], lambda f, e: f.loc[dests].multiply(e, axis=0), solver.photoionization_data_level_energies.loc[dests]))
    ck = {t: md.collision_key_idx[tt == t].to_numpy() for t in (11, 5, 4, 6, 7, 14)}
    put(11, *probe(RATE_TABLES[2], lambda f, e: f.multiply(e, axis=0).iloc[ck[11]], solver._delta_E_yg))
    put(5, *probe(RATE_TABLES[2], lambda f, e: f.iloc[ck[5]].multiply(e, axis=0), solver._coll_energies_lower.iloc[ck[5]].values))
    put(4, *probe(RATE_TABLES[3], lambda f, e: f.iloc[ck[4]].multiply(e, axis=0), solver._coll_energies_lower.iloc[ck[4]].values))
    put(6, *probe(RATE_TABLES[4], lambda f, e: f.iloc[ck[6]].multiply(e, axis=0), solver._coll_ion_energies.iloc[ck[6]]))
    put(7, *probe(RATE_TABLES[5], lambda f, e: f.iloc[ck[7]].multiply(e, axis=0), solver._coll_ion_energies.iloc[ck[7]].values))
    put(14, *probe(RATE_TABLES[5], lambda f, e: f.iloc[ck[14]].multiply(e, axis=0), solver._delta_E_yg_ionization.iloc[ck[14]].values))
    for t, name in ((-20, COOLING_TABLES[0]), (21, COOLING_TABLES[1]), (22, COOLING_TABLES[2])):  # position inside the type
        n = int((tt == t).sum())
        if n != rates[name].shape[1]:
            raise ValueError(f"cooling rows of type {t}: {n} rows for {rates[name].shape[1]} columns of {name}")
        put(t, np.arange(n, dtype=np.float64), np.zeros(n))
    return dict(rate_key=key, energy=energy, n_rate_rows=[len(rates[n].index) for n in RATE_TABLES],
                n_cooling_rows=[rates[n].shape[1] for n in COOLING_TABLES])


def continuum_rates(rates) -> dict:
    """The per-iteration tables of tb200_continuum_rates from `solve`'s arguments (rate frames in their own row order,
    cooling arrays transposed to [key, S])."""
    n_e = rates["electron_densities"]
    for name in RATE_TABLES:
        if not rates[name].columns.equals(n_e.index):
            raise ValueError(f"{name}: its columns must be the shells of electron_densities")
    return dict(rate=[rates[n].to_numpy(dtype=np.float64) for n in RATE_TABLES],
                cooling=[np.asarray(rates[n], dtype=np.float64).T for n in COOLING_TABLES],
                electron_densities=n_e.to_numpy(dtype=np.float64),
                **{k: np.asarray(rates[k], dtype=np.float64) for k in ("ff_cool_rate", "fb_cool_rate", "coll_exc_cool_rate", "coll_ion_cool_rate")})


def solve_next_macroatom_iteration(self, mean_intensities_blue_wing, beta_sobolevs, stimulated_emission_factors,
                                   stim_recomb_corrected_photoionization_rate_coeff, spontaneous_recombination_coeff, coll_deexc_coeff,
                                   coll_exc_coeff, coll_ion_coeff, coll_recomb_coeff, electron_densities, coll_exc_cool_rate,
                                   coll_exc_cool_arr, coll_exc_cool_destinations, coll_ion_cool_rate, coll_ion_cool_arr, fb_cool_rate,
                                   fb_cool_probs_arr, ff_cool_rate, engine=None):
    """ContinuumMacroAtomSolver._solve_next_macroatom_iteration on the GPU: same arguments, same return values
    (normalised probabilities and normalised deactivating probabilities as DataFrames [T, S] on the metadata's index and
    beta_sobolevs' columns, and X [S, n, n]).  Reads what the reference's first iteration left on `self`
    (computed_metadata, _nus, _oscillator_strength_*, _energies_*, and what `continuum_row_map` reads).  The row map is
    derived once per metadata object.  Every row is built by `tb200_build_opacity` from the given beta / stim / J_blue
    and rates, normalised, and the chain solved from that table in HBM (`build_absorbing_markov(None)`).  `engine`: the
    `Engine` to build on (default: this process's engine of device 0); its model is replaced by a stub carrying the
    line list and the macro-atom rows, with the option keep_opacity_tables set.  The returned X is recognised by
    `montecarlo_transport` (`built_inputs`), which rebuilds it in HBM instead of uploading it."""
    global _last
    import pandas as pd

    from .montecarlo import get_engine

    metadata = self.computed_metadata[0]
    rates = dict(stim_recomb_corrected_photoionization_rate_coeff=stim_recomb_corrected_photoionization_rate_coeff,
                 spontaneous_recombination_coeff=spontaneous_recombination_coeff, coll_deexc_coeff=coll_deexc_coeff,
                 coll_exc_coeff=coll_exc_coeff, coll_ion_coeff=coll_ion_coeff, coll_recomb_coeff=coll_recomb_coeff,
                 electron_densities=electron_densities, coll_exc_cool_rate=coll_exc_cool_rate, coll_exc_cool_arr=coll_exc_cool_arr,
                 coll_ion_cool_rate=coll_ion_cool_rate, coll_ion_cool_arr=coll_ion_cool_arr, fb_cool_rate=fb_cool_rate,
                 fb_cool_probs_arr=fb_cool_probs_arr, ff_cool_rate=ff_cool_rate)
    cached = getattr(self, "_b200_row_map", None)
    if cached is None or cached[0] is not metadata:
        cached = (metadata, continuum_row_map(self, metadata, rates))
        self._b200_row_map = cached
    rows = cached[1]

    eng = engine if engine is not None else get_engine()
    beta = np.ascontiguousarray(beta_sobolevs.to_numpy(dtype=np.float64))
    L, S = beta.shape
    nus = np.asarray(self._nus, dtype=np.float64).ravel()
    tt = metadata.transition_type.to_numpy().astype(np.int64)
    src = metadata.source_level_idx.to_numpy().astype(np.int64)
    dst = np.where(tt >= 0, metadata.destination_level_idx.to_numpy(), -1).astype(np.int64)
    tline = np.where(np.isin(tt, (-1, 0, 1)), metadata.transition_line_idx.to_numpy(), 0).astype(np.int64)
    n = int(src.max()) + 1
    edges = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(np.bincount(src, minlength=n), out=edges[1:])
    radii = np.arange(1, S + 2, dtype=np.float64) * 1e14
    eng.set_option("keep_opacity_tables", 1)
    eng.set_model(r_inner=radii[:-1], r_outer=radii[1:], time_explosion=1.0, electron_density=np.ones(S), line_list_nu=nus,
                  tau_sobolev=np.zeros((L, S)), line_interaction_type="macroatom", transition_probabilities=None,
                  line2macro_level_upper=np.zeros(L, dtype=np.int64), macro_block_edge_index=edges, transition_type=tt,
                  destination_level_id=dst, transition_line_id=tline, continuum=_continuum_stub(S), t_electrons=np.full(S, 1e4),
                  enable_full_relativity=True)
    # The level arrays feed only tau and the stimulated-emission factor, which are given here (one dummy level).
    zeros = np.zeros(L, dtype=np.int64)
    eng.set_atomic_data(lines_lower_level_index=zeros, lines_upper_level_index=zeros, g=np.ones(1), metastability=np.zeros(1, dtype=np.uint8),
                        wavelength_cm=np.ones(L), f_lu=np.asarray(self._oscillator_strength_lu, dtype=np.float64).ravel(),
                        f_ul=np.asarray(self._oscillator_strength_ul, dtype=np.float64).ravel(),
                        energy_lower=np.asarray(self._energies_lower, dtype=np.float64).ravel(),
                        energy_upper=np.asarray(self._energies_upper, dtype=np.float64).ravel(), continuum_rows=rows)
    eng.build_opacity(None, 1.0, j_blues=mean_intensities_blue_wing.to_numpy(dtype=np.float64),
                      continuum=dict(continuum_rates(rates), beta_sobolev=beta,
                                     stimulated_emission_factor=np.asarray(stimulated_emission_factors, dtype=np.float64)))
    norm = eng.download_opacity(transition_probabilities=True)["transition_probabilities"]
    inputs = dict(transition_probabilities=norm, source_level_idx=src, destination_level_idx=dst, transition_type=tt, n_states=n)
    eng.build_absorbing_markov(None, src, dst, tt, n_states=n)
    got = eng.download_absorbing_markov()
    X = got["absorbing_markov_probabilities"]
    _last = (X, inputs)
    frame = lambda a: pd.DataFrame(a, index=metadata.index, columns=beta_sobolevs.columns)  # noqa: E731
    return frame(norm), frame(got["transition_probabilities"]), X
