"""Drop-in for the continuum macro atom's absorbing-Markov-chain solve, create_absorbing_probs
(tardis/opacities/macro_atom/absorbing_markov_chain.py:19-134), on the GPU.

On the reference side the swap is one line:

    macroatom_solver.create_absorbing_probs = tardis_b200.macro_atom.create_absorbing_probs

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
