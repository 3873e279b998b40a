"""CPU restatement of the reference's weighted black-body packet source.  TEST INFRASTRUCTURE ONLY.

`BasePacketSource.create_packets` (tardis/transport/montecarlo/packet_source/base.py:195-253) with the overrides of
`BlackBodyWeightedSource` (packet_source/black_body_weighted.py:55-108), written out operation by operation:

  seeds = rng.choice(2**32 - 1, N)                      the bounded draws of the plain source
  nus_bb = Carter-Cashwell from rng.random((5, N))      used only for min and max (black_body.py:166-179)
  nus = lo + (hi - lo) * rng.random(N)                  numpy's random_uniform, lo / hi the extremes of nus_bb
  mus = sqrt(rng.random(N))
  energies = I / pairwise_sum(I),  I = coefficient * nu**3 / (exp(h * nu * beta_rad) - 1)   (util/base.py:279-302)

The raw doubles are numpy's own `default_rng(seed)` (its stream is pinned independently by oracle/packet_source_oracle.c
and tests/test_packet_source.py); what is restated here is everything done with them, and above all `ndarray.sum()` as
numpy's pairwise summation over the whole array (`pairwise_sum` below), whose leaves are the tree the device follows.
"""
from __future__ import annotations

import numpy as np

K_B, H, C = 1.3806488e-16, 6.62606957e-27, 2.99792458e10  # CODATA-2010 cgs (tardis/constants.py)
PW_BLOCK = 128


def pairwise_leaves(n: int) -> list[tuple[int, int]]:
    """The runs where numpy's pairwise recursion stops, in order: (start, length)."""
    out, stack = [], [(0, n)]
    while stack:
        lo, m = stack.pop()
        if m <= PW_BLOCK:
            out.append((lo, m))
            continue
        n2 = m // 2
        n2 -= n2 % 8
        stack.append((lo + n2, m - n2))
        stack.append((lo, n2))
    return out


def leaf_sums(a: np.ndarray, leaves) -> dict[int, float]:
    """start -> the leaf's sum in numpy's order (eight interleaved accumulators, or in order below 8), vectorised over
    the leaves of one length: every operation is one IEEE add per leaf."""
    a = np.asarray(a, dtype=np.float64)
    out: dict[int, float] = {}
    by_len: dict[int, list[int]] = {}
    for s, m in leaves:
        by_len.setdefault(m, []).append(s)
    for m, starts in by_len.items():
        st = np.array(starts, dtype=np.int64)
        blk = a[st[:, None] + np.arange(m)[None, :]]
        if m < 8:
            res = np.full(len(st), -0.0)
            for i in range(m):
                res = res + blk[:, i]
        else:
            r = blk[:, :8].copy()
            i = 8
            while i < m - m % 8:
                r = r + blk[:, i:i + 8]
                i += 8
            res = ((r[:, 0] + r[:, 1]) + (r[:, 2] + r[:, 3])) + ((r[:, 4] + r[:, 5]) + (r[:, 6] + r[:, 7]))
            for j in range(i, m):
                res = res + blk[:, j]
        out.update(zip(starts, res.tolist()))
    return out


def combine(n: int, leaf_value) -> float:
    """The sum of an n-element tree from leaf_value(start), along numpy's recursion."""
    def rec(lo, m):
        if m <= PW_BLOCK:
            return leaf_value(lo)
        n2 = m // 2
        n2 -= n2 % 8
        return rec(lo, n2) + rec(lo + n2, m - n2)
    return 0.0 + rec(0, n)


def pairwise_sum(a: np.ndarray) -> float:
    """`a.sum()` for a contiguous float64 array, restated."""
    n = len(a)
    if n == 0:
        return 0.0
    sums = leaf_sums(a, pairwise_leaves(n))
    return combine(n, sums.__getitem__)


def intensity_black_body(nu: np.ndarray, temperature: float) -> np.ndarray:
    """util/base.py:279-302, the numexpr expression evaluated left to right by numpy"""
    beta_rad = 1 / (K_B * temperature)
    coefficient = 2 * H / C**2
    return coefficient * nu**3 / (np.exp(H * nu * beta_rad) - 1)


def create_packets(n_packets: int, seed: int, radius: float, temperature: float, l_samples: int = 1000,
                   max_seed_val: int = 2**32 - 1) -> dict:
    """The PacketCollection arrays of BlackBodyWeightedSource.create_packets for default_rng(seed), seed = base_seed +
    seed_offset, plus `nus_bb_min` / `nus_bb_max` and `energy_sum`."""
    n = int(n_packets)
    if n == 0:
        raise ValueError("zero-size array to reduction operation minimum which has no identity")
    rng = np.random.default_rng(seed)
    seeds = rng.choice(max_seed_val, n, replace=True).astype(np.int64)
    l_array = np.cumsum(np.arange(1, l_samples, dtype=np.float64) ** -4)
    xis = rng.random((5, n))
    l_ = l_array.searchsorted(xis[0] * (np.pi**4 / 90.0)) + 1.0
    nus_bb = (-np.log(((xis[1] * xis[2]) * xis[3]) * xis[4]) / l_) * (K_B * temperature) / H
    lo, hi = float(nus_bb.min()), float(nus_bb.max())
    nus = lo + (hi - lo) * rng.random(n)
    mus = np.sqrt(rng.random(n))
    intensity = intensity_black_body(nus, temperature)
    total = pairwise_sum(intensity)
    return dict(initial_radii=np.full(n, float(radius)), initial_nus=nus, initial_mus=mus, initial_energies=intensity / total,
                packet_seeds=seeds, nus_bb_min=lo, nus_bb_max=hi, energy_sum=total)
