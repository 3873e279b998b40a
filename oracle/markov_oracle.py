"""NumPy / SciPy restatement of the continuum macro atom's absorbing Markov chain (the checker of
tardis_b200/csrc/markov_build.cuh).  Paths relative to /root/reference/tardis/.

- `absorbing_probs`: create_absorbing_probs (opacities/macro_atom/absorbing_markov_chain.py:19-134).  Per shell, Q is the
  internal rows (transition_type >= 0) at (source_level_idx, destination_level_idx) with duplicate pairs summed
  (scipy.sparse.coo_matrix, :87-89), q = the row sums of Q (:101-103), and X solves (I - Q) X = diag(1 - q) (:104-108).
  `solver="splu"` factors I - Q as the reference does (splu, permc_spec="MMD_AT_PLUS_A"); `solver="lapack"` is the
  pivoted dense solve (scipy.linalg.solve); `solver="extended"` solves the same float64 system in numpy's long double (LU
  without pivoting, valid for an M-matrix): the accuracy yardstick on ill-conditioned shells.
- `deactivation_table`: the internal rows multiplied by 0 (:128-129), then normalize_transition_probabilities
  (opacities/macro_atom/macroatom_solver.py:709-739): p / (sum of p over the rows of the same source), NaN -> 0.  pandas
  sums a group with Kahan compensation in row order (pandas/_libs/groupby.pyx, group_sum), restated in `kahan_block_sums`.
"""
from __future__ import annotations

import numpy as np
import scipy.linalg
import scipy.sparse
import scipy.sparse.linalg


def kahan_block_sums(p: np.ndarray, edges: np.ndarray) -> np.ndarray:
    """[n_blocks, S]: per block of rows [edges[b], edges[b+1]) and per column, the compensated sum in row order."""
    n_blocks, S = len(edges) - 1, p.shape[1]
    sums = np.zeros((n_blocks, S))
    for b in range(n_blocks):
        s, c = np.zeros(S), np.zeros(S)
        for t in range(edges[b], edges[b + 1]):
            y = p[t] - c
            u = s + y
            c = (u - s) - y
            c[np.isnan(c)] = 0.0  # an infinite addend: pandas resets the compensation
            s = u
        sums[b] = s
    return sums


def deactivation_table(transition_probabilities: np.ndarray, transition_type: np.ndarray, edges: np.ndarray) -> np.ndarray:
    """The normalised deactivating probabilities [T, S] that the continuum transport reads."""
    p = np.array(transition_probabilities, dtype=np.float64)
    p[np.asarray(transition_type) >= 0] *= 0
    sums = kahan_block_sums(p, edges)
    rows = np.repeat(np.arange(len(edges) - 1), np.diff(edges))
    with np.errstate(invalid="ignore", divide="ignore"):
        out = p / sums[rows]
    out[np.isnan(out)] = 0.0
    return out


def _lu_solve_extended(A: np.ndarray, d: np.ndarray) -> np.ndarray:
    """(A^-1 diag(d)) computed in long double and rounded to float64 once."""
    a = A.astype(np.longdouble)
    n = len(a)
    y = np.diag(d.astype(np.longdouble))
    for k in range(n):
        a[k + 1:, k] /= a[k, k]
        a[k + 1:, k + 1:] -= np.outer(a[k + 1:, k], a[k, k + 1:])
        y[k + 1:] -= np.outer(a[k + 1:, k], y[k])
    for k in reversed(range(n)):
        y[k] /= a[k, k]
        y[:k] -= np.outer(a[:k, k], y[k])
    return y.astype(np.float64)


def absorbing_probs(transition_probabilities, source_level_idx, destination_level_idx, transition_type, n_states=None,
                    solver: str = "splu") -> np.ndarray:
    """X [S, n, n] with X[s] = (I - Q_s)^-1 diag(1 - q_s)."""
    p = np.asarray(transition_probabilities, dtype=np.float64)
    src, dst, tt = (np.asarray(a, dtype=np.int64) for a in (source_level_idx, destination_level_idx, transition_type))
    n = int(src.max()) + 1 if n_states is None else int(n_states)
    internal = tt >= 0
    rows, cols = src[internal], dst[internal]
    S = p.shape[1]
    out = np.zeros((S, n, n))
    eye = scipy.sparse.identity(n, format="csc")
    for s in range(S):
        vals = p[internal, s]
        Q = scipy.sparse.coo_matrix((vals, (rows, cols)), shape=(n, n))
        q = np.asarray(Q.sum(axis=1)).ravel()
        rhs = np.diag(1 - q)
        if solver == "splu":
            out[s] = scipy.sparse.linalg.splu((eye - Q).tocsc(), permc_spec="MMD_AT_PLUS_A").solve(rhs)
        elif solver == "lapack":
            out[s] = scipy.linalg.solve(np.eye(n) - Q.toarray(), rhs)
        elif solver == "extended":
            out[s] = _lu_solve_extended(np.eye(n) - Q.toarray(), 1 - q)
        else:
            raise ValueError(solver)
    return out
