"""Synthetic supernova-ejecta models and packet sources for tests and bench.

No atomic data file and no plasma solver can run in this environment
(SURVEY.md §8c), so the transport tables are generated directly with
Kurucz-like statistics following the recipe in SURVEY.md §8(d).  Everything is
seeded with ``numpy.random.default_rng`` so the same model can be rebuilt on
the GPU box, in the oracle and in the golden-vector generator.

The arrays mirror, field for field, what the reference hands to its Monte Carlo
loop: ``OpacityStateNumba`` (tardis/opacities/opacity_state_numba.py:13-72),
``NumbaHomologousRadial1DGeometry`` (tardis/model/geometry/radial1d_homologous.py:199-226),
``PacketCollection`` (tardis/transport/montecarlo/packets/packet_collections.py:14-76).
The packet source restates ``BlackBodySimpleSource``
(tardis/transport/montecarlo/packet_source/black_body.py:122-220,
packet_source/base.py:195-253).
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

# CODATA-2010 cgs (astropy.constants.astropyconst13 as used by tardis/constants.py:1)
C_SPEED_OF_LIGHT = 2.99792458e10
H_PLANCK = 6.62606957e-27
K_BOLTZMANN = 1.3806488e-16
SIGMA_THOMSON = 6.652458734e-25
SIGMA_SB = 5.670373e-5

MODEL_SEED = 20260924
BASE_SEED = 23111963  # tardis/io/configuration/schemas/montecarlo.yml:13-17
MAX_SEED_VAL = 2**32 - 1  # packet_source/base.py


@dataclass
class MacroAtomTables:
    """Flat macro-atom tables (tardis/opacities/opacity_state_numba.py:31-37)."""

    transition_probabilities: np.ndarray  # f64[T, S] C-order
    line2macro_level_upper: np.ndarray  # i64[L]
    macro_block_edge_index: np.ndarray  # i64[n_blocks + 1]
    transition_type: np.ndarray  # i64[T]
    destination_level_id: np.ndarray  # i64[T]
    transition_line_id: np.ndarray  # i64[T]


@dataclass
class ContinuumTables:
    """Continuum (IIP mode) fields of OpacityStateNumbaIIP (tardis/opacities/opacity_state_numba_iip.py:8-125)."""

    bf_threshold_list_nu: np.ndarray          # f64[n_cont], descending (estimators/radfield_estimator_calcs.py:91-92)
    p_fb_deactivation: np.ndarray             # f64[n_cont, S] (carried by the reference, unused by the IIP loop)
    photo_ion_nu_threshold_mins: np.ndarray   # f64[n_cont] first phot_nu of each block
    photo_ion_nu_threshold_maxs: np.ndarray   # f64[n_cont] last phot_nu of each block
    photo_ion_block_references: np.ndarray    # i64[n_cont + 1]
    chi_bf: np.ndarray                        # f64[n_phot, S]
    x_sect: np.ndarray                        # f64[n_phot]
    phot_nus: np.ndarray                      # f64[n_phot], ascending inside each block
    ff_opacity_factor: np.ndarray             # f64[S]
    emissivities: np.ndarray                  # f64[n_phot, S] per-block CDF in nu (0 ... 1)
    photo_ion_activation_idx: np.ndarray      # i64[30] (the reference hard-codes 30, opacities/opacity_state.py:259-264)
    k_packet_idx: int
    absorbing_markov_probabilities: np.ndarray  # f64[S, n_states, n_states]


@dataclass
class Model:
    """Everything the packet-propagation path reads for one MC iteration."""

    r_inner: np.ndarray
    r_outer: np.ndarray
    v_inner: np.ndarray
    v_outer: np.ndarray
    time_explosion: float
    electron_density: np.ndarray
    t_electrons: np.ndarray
    line_list_nu: np.ndarray  # f64[L], non-increasing
    tau_sobolev: np.ndarray  # f64[L, S] C-order (reference layout)
    macro: MacroAtomTables | None
    spectrum_frequency_grid: np.ndarray  # f64[B + 1]
    line_interaction_type: str = "scatter"
    meta: dict = field(default_factory=dict)
    continuum: ContinuumTables | None = None  # set => IIP mode (continuum processes, full relativity, no vpackets)

    @property
    def n_shells(self) -> int:
        return len(self.r_inner)

    @property
    def n_lines(self) -> int:
        return len(self.line_list_nu)


@dataclass
class Packets:
    """SoA packet inputs (PacketCollection, packet_collections.py:14-76)."""

    initial_radii: np.ndarray
    initial_nus: np.ndarray
    initial_mus: np.ndarray
    initial_energies: np.ndarray
    packet_seeds: np.ndarray  # i64, values < 2**32 - 1
    radiation_field_luminosity: float

    @property
    def time_of_simulation(self) -> float:
        return 1.0 / self.radiation_field_luminosity

    def __len__(self) -> int:
        return len(self.initial_nus)

    def slice(self, lo: int, hi: int) -> "Packets":
        return Packets(
            self.initial_radii[lo:hi],
            self.initial_nus[lo:hi],
            self.initial_mus[lo:hi],
            self.initial_energies[lo:hi],
            self.packet_seeds[lo:hi],
            self.radiation_field_luminosity,
        )


def scatter_dummy_macro() -> MacroAtomTables:
    """1-element dummies used for `scatter` (tardis/opacities/opacity_state.py:199-209)."""
    return MacroAtomTables(
        np.zeros((1, 1)),
        np.zeros(1, dtype=np.int64),
        np.zeros(1, dtype=np.int64),
        np.zeros(1, dtype=np.int64),
        np.zeros(1, dtype=np.int64),
        np.zeros(1, dtype=np.int64),
    )


def make_macro_atom(
    n_lines: int,
    n_shells: int,
    rng: np.random.Generator,
    mode: str,
    n_levels: int | None = None,
) -> MacroAtomTables:
    """Synthetic macro-atom tables with the reference's structure.

    Structure contract (SURVEY.md Appendix B; tardis/opacities/macro_atom/
    macroatom_solver.py:425-436,604-622,652-657,672-707): rows are transitions
    grouped by source level; inside a block the order is emission-down (-1),
    internal-down (0), internal-up (1); ``transition_line_id`` is the line index
    for all three types; ``destination_level_id`` indexes source levels;
    per-(block, shell) probabilities sum to one.  ``downbranch`` keeps only the
    emission rows (macroatom_solver.py:399-401) and sets destinations to -99.
    """
    if n_levels is None:
        n_levels = max(4, n_lines // 16)
    # heavy-tailed level popularity: a few levels own very many lines
    a = np.floor(n_levels * rng.random(n_lines) ** 2).astype(np.int64)
    b = np.floor(n_levels * rng.random(n_lines) ** 2).astype(np.int64)
    lower = np.minimum(a, b)
    upper = np.maximum(a, b)
    same = lower == upper
    upper[same] = np.minimum(upper[same] + 1, n_levels - 1)
    lower[same & (lower == upper)] -= 1  # only when both hit the top level
    line_id = np.arange(n_lines, dtype=np.int64)

    # candidate rows: (source, order-in-block, type, dest, line)
    src = np.concatenate([upper, upper, lower])
    order = np.concatenate([np.zeros(n_lines), np.ones(n_lines), 2 * np.ones(n_lines)]).astype(np.int64)
    ttype = np.concatenate([-np.ones(n_lines), np.zeros(n_lines), np.ones(n_lines)]).astype(np.int64)
    dest = np.concatenate([lower, lower, upper])
    tline = np.concatenate([line_id, line_id, line_id])
    weight_scale = np.concatenate([np.full(n_lines, 1.0), np.full(n_lines, 0.35), np.full(n_lines, 0.15)])

    if mode == "downbranch":
        keep = ttype == -1
        src, order, ttype, dest, tline, weight_scale = (
            x[keep] for x in (src, order, ttype, dest, tline, weight_scale)
        )
        dest = np.full_like(dest, -99)
    elif mode != "macroatom":
        raise ValueError(mode)

    perm = np.lexsort((tline, order, src))
    src, ttype, dest, tline, weight_scale = (x[perm] for x in (src, ttype, dest, tline, weight_scale))
    n_t = len(src)
    counts = np.bincount(src, minlength=n_levels)
    edges = np.zeros(n_levels + 1, dtype=np.int64)
    np.cumsum(counts, out=edges[1:])

    # raw rates: log-normal per transition with a mild shell dependence
    base = np.exp(rng.normal(0.0, 1.5, n_t)) * weight_scale
    shell_mod = np.exp(rng.normal(0.0, 0.3, (n_t, n_shells)))
    probs = base[:, None] * shell_mod
    nonempty = counts > 0
    starts = edges[:-1][nonempty]
    sums = np.add.reduceat(probs, starts, axis=0)  # [n_nonempty, S]
    block_of_row = np.repeat(np.arange(nonempty.sum()), counts[nonempty])
    probs /= sums[block_of_row]
    probs = np.ascontiguousarray(probs)

    return MacroAtomTables(
        transition_probabilities=probs,
        line2macro_level_upper=upper.astype(np.int64),
        macro_block_edge_index=edges,
        transition_type=ttype,
        destination_level_id=dest.astype(np.int64),
        transition_line_id=tline,
    )


def make_model(
    n_shells: int = 20,
    n_lines: int = 500_000,
    line_interaction_type: str = "scatter",
    mu_tau: float = -7.5,
    sigma_tau: float = 2.0,
    seed: int = MODEL_SEED,
    n_bins: int = 10_000,
    duplicate_fraction: float = 0.01,
    n_levels: int | None = None,
    lambda_min_A: float = 500.0,
    lambda_max_A: float = 20000.0,
) -> Model:
    """Build the synthetic model of SURVEY.md §8(d).

    Geometry: v = linspace(1.1e9, 2.0e9, S+1) cm/s, t_exp = 13 d
    (docs/tardis_example.yml:4-6,14-18).  Lines: log-uniform in wavelength on
    [500, 20000] A, sorted by descending nu, with ``duplicate_fraction`` of the
    lines made exact duplicates of their neighbour (real line lists have
    coincident lines; this exercises the close-line branch,
    transport/geometry/calculate_distances.py:98-101).  tau_Sobolev =
    10**N(mu_tau, sigma_tau) * (v/v0)**-7.  n_e = geomspace(2e9, 2e8, S).
    """
    rng = np.random.default_rng(seed)
    t_exp = 13.0 * 86400.0
    v = np.linspace(1.1e9, 2.0e9, n_shells + 1)
    r = v * t_exp
    lam = np.exp(rng.uniform(np.log(lambda_min_A), np.log(lambda_max_A), n_lines))
    lam.sort()
    nu = C_SPEED_OF_LIGHT / (lam * 1e-8)  # descending
    if duplicate_fraction > 0 and n_lines > 2:
        n_dup = int(duplicate_fraction * n_lines)
        idx = rng.choice(n_lines - 1, n_dup, replace=False) + 1
        nu[idx] = nu[idx - 1]
    assert np.all(np.diff(nu) <= 0)
    v_mid = 0.5 * (v[:-1] + v[1:])
    falloff = (v_mid / v_mid[0]) ** -7.0
    tau = 10.0 ** rng.normal(mu_tau, sigma_tau, (n_lines, n_shells)) * falloff[None, :]
    tau = np.ascontiguousarray(tau)
    n_e = np.geomspace(2e9, 2e8, n_shells)
    t_e = np.full(n_shells, 1.0e4)
    if line_interaction_type == "scatter":
        macro = scatter_dummy_macro()
    else:
        macro = make_macro_atom(n_lines, n_shells, rng, line_interaction_type, n_levels)
    grid = np.linspace(
        C_SPEED_OF_LIGHT / (lambda_max_A * 1e-8), C_SPEED_OF_LIGHT / (lambda_min_A * 1e-8), n_bins + 1
    )
    return Model(
        r_inner=np.ascontiguousarray(r[:-1]),
        r_outer=np.ascontiguousarray(r[1:]),
        v_inner=np.ascontiguousarray(v[:-1]),
        v_outer=np.ascontiguousarray(v[1:]),
        time_explosion=t_exp,
        electron_density=n_e,
        t_electrons=t_e,
        line_list_nu=np.ascontiguousarray(nu),
        tau_sobolev=tau,
        macro=macro,
        spectrum_frequency_grid=grid,
        line_interaction_type=line_interaction_type,
        meta=dict(seed=seed, mu_tau=mu_tau, sigma_tau=sigma_tau),
    )


def add_continuum(model: Model, seed: int = MODEL_SEED + 1, n_continua: int = 30, n_levels: int = 60,
                  points: tuple[int, int] = (12, 30), chi_bf_scale: float = 3e-3, adiabatic_fraction: float = 0.05) -> Model:
    """Turn `model` into an IIP-mode model (SURVEY.md §8d "Continuum (config 5)"): bound-free continua with hydrogenic
    cross-sections (x_sect ~ nu^-3) on ascending `phot_nus` blocks, `chi_bf = x_sect * n_level`, emissivity CDFs per
    (block, shell), free-free opacity factors, and the IIP macro atom: an absorbing-Markov-chain matrix
    [S, n_states, n_states] plus one block of normalised deactivation channels per state (line / bound-free /
    free-free emission, k-packet cooling channels incl. adiabatic cooling, photo-recombination emission).  The
    macro-atom tables of `model` are REPLACED by the IIP ones (opacities/opacity_state.py:212-292)."""
    rng = np.random.default_rng(seed)
    S, L = model.n_shells, model.n_lines
    thr = np.sort(np.exp(rng.uniform(np.log(3e14), np.log(4e15), n_continua)))[::-1].copy()
    counts = rng.integers(points[0], points[1], n_continua)
    refs = np.zeros(n_continua + 1, dtype=np.int64)
    refs[1:] = np.cumsum(counts)
    n_phot = int(refs[-1])
    phot_nus = np.empty(n_phot)
    x_sect = np.empty(n_phot)
    for k in range(n_continua):
        nus = thr[k] * np.exp(np.linspace(0, np.log(rng.uniform(3, 8)), counts[k]))
        phot_nus[refs[k]:refs[k + 1]] = nus
        x_sect[refs[k]:refs[k + 1]] = rng.uniform(1e-19, 6e-18) * (thr[k] / nus) ** 3
    n_level = 10 ** rng.uniform(2.0, 5.5, (n_continua, S)) * chi_bf_scale
    chi_bf = np.ascontiguousarray(x_sect[:, None] * np.repeat(n_level, counts, axis=0))
    em = np.empty((n_phot, S))
    for k in range(n_continua):
        w = rng.random((counts[k], S)) + 0.05
        w[0] = 0.0
        c = np.cumsum(w, axis=0)
        em[refs[k]:refs[k + 1]] = c / c[-1]
    ff_factor = 10 ** rng.uniform(19.5, 20.5, S)
    k_idx, pi_idx, n_states = n_levels, n_levels + 1, n_levels + 2
    types, tline, edges = [], [], [0]
    for lev in range(n_states):
        for _ in range(int(rng.integers(2, 7))):
            if lev == k_idx:
                t = int(rng.choice([-20, -21, -4], p=[0.65 - adiabatic_fraction, 0.35, adiabatic_fraction]))  # FB_COOLING, FF_COOLING, ADIABATIC
            elif lev == pi_idx:
                t = -7                                                   # PHOTO_RECOMB_EMISSION
            else:
                t = int(rng.choice([-1, -2, -3], p=[0.8, 0.15, 0.05]))  # BB, BF, FF emission
            types.append(t)
            tline.append(int(rng.integers(0, L - 1)) if t == -1 else (int(rng.integers(0, n_continua)) if t in (-2, -7, -20) else 0))
        edges.append(len(types))
    edges = np.array(edges, dtype=np.int64)
    n_t = len(types)
    tp = rng.random((n_t, S)) + 0.05
    for b in range(n_states):
        tp[edges[b]:edges[b + 1]] /= tp[edges[b]:edges[b + 1]].sum(axis=0)
    markov = rng.random((S, n_states, n_states)) ** 4
    markov /= markov.sum(axis=2, keepdims=True)
    model.macro = MacroAtomTables(
        transition_probabilities=np.ascontiguousarray(tp),
        line2macro_level_upper=rng.integers(0, n_levels, L).astype(np.int64),
        macro_block_edge_index=edges,
        transition_type=np.array(types, dtype=np.int64),
        destination_level_id=np.full(n_t, -99, dtype=np.int64),
        transition_line_id=np.array(tline, dtype=np.int64),
    )
    if model.line_interaction_type == "scatter":
        model.line_interaction_type = "macroatom"
    model.continuum = ContinuumTables(
        bf_threshold_list_nu=thr, p_fb_deactivation=np.full((n_continua, S), 1.0 / n_continua),
        photo_ion_nu_threshold_mins=phot_nus[refs[:-1]].copy(), photo_ion_nu_threshold_maxs=phot_nus[refs[1:] - 1].copy(),
        photo_ion_block_references=refs, chi_bf=chi_bf, x_sect=x_sect, phot_nus=phot_nus, ff_opacity_factor=ff_factor,
        emissivities=np.ascontiguousarray(em), photo_ion_activation_idx=np.full(30, pi_idx, dtype=np.int64),
        k_packet_idx=k_idx, absorbing_markov_probabilities=np.ascontiguousarray(markov))
    return model


@dataclass
class ContinuumMacroAtom:
    """What create_absorbing_probs takes (opacities/macro_atom/absorbing_markov_chain.py:19-56): the normalised probabilities
    and the rows' metadata.  Rows are grouped by source state; block b = state b."""

    transition_probabilities: np.ndarray  # f64[T, S], normalised per source block
    source_level_idx: np.ndarray          # i64[T]
    destination_level_idx: np.ndarray     # i64[T] (internal rows: a state; deactivation rows: -1)
    transition_type: np.ndarray           # i64[T]; >= 0 internal
    macro_block_edge_index: np.ndarray    # i64[n_states + 1]
    n_states: int


def add_continuum_macro_atom(model: Model, seed: int = MODEL_SEED + 2, n_levels: int = 60, internal_rows: tuple[int, int] = (1, 12),
                             deactivation_rows: tuple[int, int] = (1, 4), internal_share: tuple[float, float] = (0.3, 0.97),
                             n_groups: int = 1, duplicate_fraction: float = 0.0, self_loop_fraction: float = 0.0,
                             zero_blocks: int = 0, ill_conditioned_shell: int | None = None) -> ContinuumMacroAtom:
    """A continuum macro atom with real internal rows for `model` (made IIP by `add_continuum` first): `n_levels` levels plus a
    k-packet and an i-packet state.  Every state gets internal rows (internal down / up, type 0 / 1) to other states of its
    group (states g, g + n_groups, ...: with n_groups > 1 no path joins two groups, so X has a block zero pattern) and
    deactivation rows (line / bound-free / free-free emission for levels; k-packet: free-bound / free-free cooling and
    adiabatic cooling; i-packet: photo-recombination emission), in random order inside the block.  Per (state, shell) the
    internal rows carry a share drawn from `internal_share` (1 - 1e-6 everywhere in `ill_conditioned_shell`).
    `duplicate_fraction` repeats the previous destination, `self_loop_fraction` points a row at its own state, `zero_blocks`
    levels get all-zero probabilities.  The model's macro-atom tables become these rows, with the normalised probabilities
    as transition_probabilities and absorbing_markov_probabilities = None (to be built by the engine); `add_continuum` and
    the models it makes are unchanged."""
    rng = np.random.default_rng(seed)
    S, L = model.n_shells, model.n_lines
    n_cont = len(model.continuum.bf_threshold_list_nu)
    k_idx, i_idx, n_states = n_levels, n_levels + 1, n_levels + 2
    members = [np.arange(g, n_states, n_groups) for g in range(n_groups)]
    src, dst, ttype, tline, edges, share_rows = [], [], [], [], [0], []
    for b in range(n_states):
        group = members[b % n_groups]
        rows = []
        for _ in range(int(rng.integers(internal_rows[0], internal_rows[1] + 1))):
            if rows and rng.random() < duplicate_fraction:
                d = rows[-1][1]
            elif rng.random() < self_loop_fraction or len(group) == 1:
                d = b
            else:
                d = int(rng.choice(group[group != b]))
            rows.append((int(rng.integers(0, 2)), d, 0))
        for _ in range(int(rng.integers(deactivation_rows[0], deactivation_rows[1] + 1))):
            if b == k_idx:
                t = int(rng.choice([-20, -21, -4], p=[0.6, 0.35, 0.05]))
            elif b == i_idx:
                t = -7
            else:
                t = int(rng.choice([-1, -2, -3], p=[0.8, 0.15, 0.05]))
            rows.append((t, -1, int(rng.integers(0, L - 1)) if t == -1 else (int(rng.integers(0, n_cont)) if t in (-2, -7, -20) else 0)))
        for j in rng.permutation(len(rows)):
            t, d, tl = rows[j]
            src.append(b); ttype.append(t); dst.append(d); tline.append(tl)
        edges.append(len(src))
    src, dst, ttype, tline = (np.array(a, dtype=np.int64) for a in (src, dst, ttype, tline))
    edges = np.array(edges, dtype=np.int64)
    raw = rng.random((len(src), S)) + 0.05
    share = rng.uniform(internal_share[0], internal_share[1], (n_states, S))
    if ill_conditioned_shell is not None:
        share[:, ill_conditioned_shell] = 1.0 - 1e-6
    internal = ttype >= 0
    probs = np.zeros_like(raw)
    for b in range(n_states):
        blk = slice(edges[b], edges[b + 1])
        inn, out = internal[blk], ~internal[blk]
        r = raw[blk]
        part = np.zeros_like(r)
        if inn.any() and out.any():
            part[inn] = r[inn] / r[inn].sum(axis=0) * share[b]
            part[out] = r[out] / r[out].sum(axis=0) * (1.0 - share[b])
        else:
            part = r / r.sum(axis=0)
        probs[blk] = part
    for b in rng.choice(n_levels, zero_blocks, replace=False) if zero_blocks else ():
        probs[edges[b]:edges[b + 1]] = 0.0
    probs = np.ascontiguousarray(probs)
    model.macro = MacroAtomTables(
        transition_probabilities=probs,
        line2macro_level_upper=rng.integers(0, n_levels, L).astype(np.int64),
        macro_block_edge_index=edges,
        transition_type=ttype,
        destination_level_id=dst,
        transition_line_id=tline,
    )
    model.continuum.k_packet_idx = k_idx
    model.continuum.photo_ion_activation_idx = np.full(len(model.continuum.photo_ion_activation_idx), i_idx, dtype=np.int64)
    model.continuum.absorbing_markov_probabilities = None
    return ContinuumMacroAtom(probs, src, dst, ttype, edges, n_states)


def make_packets(
    n_packets: int,
    r_inner0: float,
    t_inner: float = 1.0e4,
    base_seed: int = BASE_SEED,
    iteration: int = 0,
    l_samples: int = 1000,
) -> Packets:
    """Restated ``BlackBodySimpleSource.create_packets``.

    Same draw order as the reference (packet_source/base.py:229-236): seeds by
    ``rng.choice(2**32 - 1, n)``, then nus via the Carter-Cashwell sampler
    (black_body.py:140-179), then mus = sqrt(xi) (black_body.py:198), energies
    1/n, all from one ``default_rng(base_seed + iteration)``.
    """
    rng = np.random.default_rng(base_seed + iteration)
    seeds = rng.choice(MAX_SEED_VAL, n_packets, replace=True).astype(np.int64)
    radii = np.ones(n_packets) * r_inner0
    l_array = np.cumsum(np.arange(1, l_samples, dtype=np.float64) ** -4)
    l_coef = np.pi**4 / 90.0
    xis = rng.random((5, n_packets))
    l = l_array.searchsorted(xis[0] * l_coef) + 1.0
    xis_prod = np.prod(xis[1:], 0)
    x = -np.log(xis_prod) / l
    nus = x * (K_BOLTZMANN * t_inner) / H_PLANCK
    mus = np.sqrt(rng.random(n_packets))
    energies = np.ones(n_packets) / n_packets
    lum = 4 * np.pi * SIGMA_SB * r_inner0**2 * t_inner**4
    return Packets(radii, nus, mus, energies, seeds, float(lum))


# ---------------------------------------------------------------------------------------------------------------------
# Inputs of the opacity build (SURVEY.md §8f rank 3): what the plasma hands to tau_sobolev / the macro-atom solver
# ---------------------------------------------------------------------------------------------------------------------
@dataclass
class AtomicData:
    """Static per-line / per-level data and the macro-atom row structure, in the reference's conventions:
    lines indexed (lower level, upper level) (atom_data.lines), levels with g / energy / metastable flag (atom_data.levels),
    macro-atom rows sorted by source level, inside a block emission-down (-1), internal-down (0), internal-up (1)
    (opacities/macro_atom/macroatom_solver.py:425-436,776-790); `transition_line_idx` = row of the line in the line list."""

    lower_level: np.ndarray       # i64[L]
    upper_level: np.ndarray       # i64[L]
    g: np.ndarray                 # f64[n_levels]
    energy: np.ndarray            # f64[n_levels] erg, increasing with the level index
    metastable: np.ndarray        # bool[n_levels]
    nu: np.ndarray                # f64[L] Hz (the line list, descending)
    wavelength_cm: np.ndarray     # f64[L]
    f_lu: np.ndarray              # f64[L]
    f_ul: np.ndarray              # f64[L]
    nlte_line: np.ndarray         # bool[L]
    transition_type: np.ndarray          # i64[T]
    transition_line_idx: np.ndarray      # i64[T]
    destination_level_id: np.ndarray     # i64[T] block index of the destination (-99: not a source)
    source_block: np.ndarray             # i64[T] block index of the row
    macro_block_edge_index: np.ndarray   # i64[n_blocks + 1]
    line2macro_level_upper: np.ndarray   # i64[L]

    @property
    def n_levels(self) -> int:
        return len(self.g)


@dataclass
class PlasmaState:
    """Per-iteration inputs of the opacity build."""

    level_number_density: np.ndarray   # f64[n_levels, S]
    j_blues: np.ndarray                # f64[L, S] (MCRadiationFieldPropertiesSolver output)
    time_explosion: float


def make_atomic_data(line_list_nu: np.ndarray, n_levels: int, mode: str = "macroatom", seed: int = MODEL_SEED + 7,
                     nlte_fraction: float = 0.1) -> AtomicData:
    rng = np.random.default_rng(seed)
    L = len(line_list_nu)
    a = np.floor(n_levels * rng.random(L) ** 2).astype(np.int64)
    b = np.floor(n_levels * rng.random(L) ** 2).astype(np.int64)
    lower, upper = np.minimum(a, b), np.maximum(a, b)
    same = lower == upper
    upper[same] = np.minimum(upper[same] + 1, n_levels - 1)
    lower[same & (lower == upper)] -= 1
    g = rng.integers(1, 9, n_levels).astype(np.float64) * 2 - 1
    energy = np.sort(rng.uniform(0.0, 4e-11, n_levels))
    energy[0] = 0.0
    metastable = rng.random(n_levels) < 0.15
    f_lu = 10 ** rng.uniform(-4, 0, L)
    f_ul = f_lu * g[lower] / g[upper]
    line_id = np.arange(L, dtype=np.int64)
    src = np.concatenate([upper, upper, lower])
    order = np.concatenate([np.zeros(L), np.ones(L), 2 * np.ones(L)]).astype(np.int64)
    ttype = np.concatenate([-np.ones(L), np.zeros(L), np.ones(L)]).astype(np.int64)
    dest = np.concatenate([lower, lower, upper])
    tline = np.concatenate([line_id, line_id, line_id])
    if mode == "downbranch":
        keep = ttype == -1
        src, order, ttype, dest, tline = (x[keep] for x in (src, order, ttype, dest, tline))
    perm = np.lexsort((tline, order, src))
    src, ttype, dest, tline = (x[perm] for x in (src, ttype, dest, tline))
    sources = np.unique(src)                                   # blocks = levels that are a source, ascending
    block_of_level = np.full(n_levels, -99, dtype=np.int64)
    block_of_level[sources] = np.arange(len(sources))
    source_block = block_of_level[src]
    edges = np.concatenate([np.searchsorted(source_block, np.arange(len(sources))), [len(src)]]).astype(np.int64)
    dest_block = np.where(mode == "downbranch", -99, block_of_level[dest]).astype(np.int64)
    return AtomicData(lower, upper, g, energy, metastable, np.ascontiguousarray(line_list_nu), C_SPEED_OF_LIGHT / np.asarray(line_list_nu),
                      f_lu, f_ul, rng.random(L) < nlte_fraction, ttype, tline, dest_block, source_block, edges, block_of_level[upper])


def make_plasma_state(atomic: AtomicData, n_shells: int, time_explosion: float, seed: int = MODEL_SEED + 8,
                      zero_fraction: float = 0.02, inversion_fraction: float = 0.02, noise: float = 0.3) -> PlasmaState:
    """Boltzmann-like level populations with a density fall-off, a few empty levels (n_lower == 0) and a few inverted
    pairs (negative stimulated-emission factors, zeroed for metastable / NLTE lines by the reference)."""
    rng = np.random.default_rng(seed)
    n = atomic.n_levels
    t = rng.uniform(8e3, 1.4e4, n_shells)
    dens = np.geomspace(1e9, 1e7, n_shells)
    lnd = atomic.g[:, None] * np.exp(-atomic.energy[:, None] / (K_BOLTZMANN * t[None, :])) * dens[None, :]
    lnd *= np.exp(rng.normal(0.0, 0.3, lnd.shape) * (noise / 0.3))
    lnd[rng.random(n) < zero_fraction] = 0.0
    boost = rng.random(n) < inversion_fraction
    lnd[boost] *= 1e3
    L = len(atomic.nu)
    j_blues = 10 ** rng.uniform(-9, -5, (L, n_shells))
    return PlasmaState(np.ascontiguousarray(lnd), np.ascontiguousarray(j_blues), float(time_explosion))


def make_nonhomologous_velocities(model: Model, amplitude: float = 0.08, seed: int = MODEL_SEED + 9) -> Model:
    """A copy of `model` for the nonhomologous mode: radii kept, the interior shell-edge velocities multiplied by
    1 + amplitude * U(-1, 1) (deterministic in `seed`).  The innermost and outermost edges are kept.  If no shell ends up
    decelerating (v_outer < v_inner), the middle interior edge is raised above its outer neighbour, so at least one
    shell scans its lines backwards."""
    import dataclasses

    v = np.concatenate([model.v_inner, model.v_outer[-1:]]).astype(np.float64)
    rng = np.random.default_rng(seed)
    if len(v) > 2:
        v[1:-1] *= 1.0 + amplitude * rng.uniform(-1.0, 1.0, len(v) - 2)
        if not np.any(v[1:] < v[:-1]):
            k = (len(v) - 1) // 2
            v[k] = v[k + 1] * (1.0 + 0.5 * amplitude)
    return dataclasses.replace(model, v_inner=np.ascontiguousarray(v[:-1]), v_outer=np.ascontiguousarray(v[1:]))


# ---------------------------------------------------------------------------------------------------------------------
# Inputs of the continuum (IIP) macro atom's per-iteration rows (ContinuumMacroAtomSolver.solve,
# opacities/macro_atom/macroatom_solver.py:861-1020), in the reference's index layout
# ---------------------------------------------------------------------------------------------------------------------
@dataclass
class ContinuumRateInputs:
    """Static atomic data as the reference's ContinuumMacroAtomSolver takes it (levels, lines, photoionization_data,
    ionization_energies: pandas objects indexed by (atomic_number, ion_number, level_number[_lower, _upper])), the same
    data as arrays for the engine's opacity build (`atomic`, rows of `levels`), and per iteration the level populations,
    J_blue and the continuum rates / cooling arrays of `solve` (`rates[i]`: keyword arguments of `solve` without
    mean_intensities_blue_wing / beta_sobolevs / stimulated_emission_factors, which follow from the populations)."""

    levels: object                 # DataFrame [n_levels] energy, g, metastable
    lines: object                  # DataFrame [L] nu, f_lu, f_ul, wavelength_cm, line_id (descending nu)
    photoionization_data: object   # DataFrame, two cross-section points per level with a bound-free continuum
    ionization_energies: object    # Series indexed by the next ion's ground state
    atomic: AtomicData             # the line / level arrays (macro-row fields empty: the reference's metadata fills them)
    plasma: list                   # [PlasmaState] per iteration
    rates: list                    # [dict] per iteration


def make_continuum_rate_inputs(n_shells: int, n_h_levels: int = 8, n_he_levels: int = 6, seed: int = MODEL_SEED + 10,
                               n_lines: int | None = None, n_iterations: int = 2, shuffle_rates: bool = False,
                               zero_levels: int = 0, infinite_rate: bool = False) -> ContinuumRateInputs:
    """Hydrogen (H I levels + the H II ground state) and helium (He I levels + the He II ground state).  Every H I level and
    the lower half of He I have a bound-free continuum; collisional (de-)excitation joins every pair of levels of an ion,
    collisional ionization / recombination every level with a continuum; collisional-excitation cooling points at the
    pair's upper level (so destinations repeat).  Rates are log-uniform per (key, shell) and differ per iteration.
    `shuffle_rates`: the photoionization / recombination / collisional-ionization frames are stored in a permuted row order
    (their labels still name the level), so a lookup by position instead of by label reads another level's rate.
    `zero_levels`: that many H I levels get all-zero rates, populations and lines removed -- empty source blocks.
    `infinite_rate`: one photoionization rate is +inf in shell 0 of the second iteration (its level's block normalises to
    0 / inf and inf / inf -> NaN -> 0; a ground-state rate times energy 0 is NaN, which pandas' group sum skips)."""
    import pandas as pd

    rng = np.random.default_rng(seed)
    S = n_shells
    species = [(1, 0, n_h_levels), (1, 1, 1), (2, 0, n_he_levels), (2, 1, 1)]
    tuples, energy = [], []
    for a, ion, n in species:
        e = np.sort(rng.uniform(1e-12, 3e-11, n))
        e[0] = 0.0
        for lev in range(n):
            tuples.append((a, ion, lev))
            energy.append(e[lev])
    level_index = pd.MultiIndex.from_tuples(tuples, names=["atomic_number", "ion_number", "level_number"])
    n_levels = len(tuples)
    g = (rng.integers(1, 9, n_levels) * 2 - 1).astype(np.float64)
    metastable = rng.random(n_levels) < 0.1
    levels = pd.DataFrame({"energy": np.array(energy), "g": g, "metastable": metastable}, index=level_index)
    row_of = {t: i for i, t in enumerate(tuples)}
    zero = set()
    if zero_levels:
        zero = {(1, 0, int(lev)) for lev in rng.choice(np.arange(1, n_h_levels), zero_levels, replace=False)}

    # lines: every pair of an ion's levels (a random subset when n_lines is given), sorted by descending frequency
    pairs = [(a, ion, lo, up) for a, ion, n in species for lo in range(n) for up in range(lo + 1, n)
             if (a, ion, lo) not in zero and (a, ion, up) not in zero]
    if n_lines is not None and n_lines < len(pairs):
        pairs = [pairs[i] for i in np.sort(rng.choice(len(pairs), n_lines, replace=False))]
    e_lo = np.array([levels.energy.iloc[row_of[(a, i, lo)]] for a, i, lo, up in pairs])
    e_up = np.array([levels.energy.iloc[row_of[(a, i, up)]] for a, i, lo, up in pairs])
    nu = (e_up - e_lo) / H_PLANCK
    order = np.argsort(-nu, kind="stable")
    pairs = [pairs[i] for i in order]
    nu = nu[order]
    L = len(pairs)
    lo_row = np.array([row_of[(a, i, lo)] for a, i, lo, up in pairs], dtype=np.int64)
    up_row = np.array([row_of[(a, i, up)] for a, i, lo, up in pairs], dtype=np.int64)
    f_lu = 10 ** rng.uniform(-3, 0, L)
    f_ul = f_lu * g[lo_row] / g[up_row]
    line_index = pd.MultiIndex.from_tuples(pairs, names=["atomic_number", "ion_number", "level_number_lower", "level_number_upper"])
    lines = pd.DataFrame({"nu": nu, "f_lu": f_lu, "f_ul": f_ul, "wavelength_cm": C_SPEED_OF_LIGHT / nu,
                          "line_id": np.arange(L, dtype=np.int64)}, index=line_index)
    atomic = AtomicData(lo_row, up_row, g, levels.energy.to_numpy().copy(), metastable, nu.copy(), C_SPEED_OF_LIGHT / nu, f_lu, f_ul,
                        np.zeros(L, dtype=bool), *(np.zeros(0, dtype=np.int64) for _ in range(6)))

    # continua and collisions
    bf = [(1, 0, lev) for lev in range(n_h_levels)] + [(2, 0, lev) for lev in range((n_he_levels + 1) // 2)]
    bf_index = pd.MultiIndex.from_tuples(bf, names=["atomic_number", "ion_number", "level_number"])
    pi_rows = pd.MultiIndex.from_tuples([t for t in bf for _ in range(2)], names=bf_index.names)
    photoionization_data = pd.DataFrame({"nu": rng.uniform(1e15, 4e15, len(pi_rows)), "x_sect": rng.uniform(1e-19, 6e-18, len(pi_rows))},
                                        index=pi_rows)
    ion_e = {(1, 1, 0): 2.18e-11, (2, 1, 0): 3.94e-11}
    ionization_energies = pd.Series(ion_e).rename_axis(["atomic_number", "ion_number", "level_number"])
    coll = [(a, ion, lo, up) for a, ion, n in species if ion == 0 for lo in range(n) for up in range(lo + 1, n)]
    coll_index = pd.MultiIndex.from_tuples(coll, names=["atomic_number", "ion_number", "level_number_lower", "level_number_upper"])
    delta_E_yg = pd.Series([levels.energy.iloc[row_of[(a, i, up)]] - levels.energy.iloc[row_of[(a, i, lo)]] for a, i, lo, up in coll],
                           index=coll_index)
    exc_dest = pd.MultiIndex.from_tuples([(a, i, up) for a, i, lo, up in coll], names=bf_index.names)
    perm = rng.permutation(len(bf)) if shuffle_rates else np.arange(len(bf))
    columns = pd.RangeIndex(S)

    def frame(keys, index, lo=-14.0, hi=-8.0):
        v = 10 ** rng.uniform(lo, hi, (len(index), S))
        for k, key in enumerate(keys):
            if zero.intersection(key):
                v[k] = 0.0
        return pd.DataFrame(v, index=index, columns=columns)

    def by_level(lo=-14.0, hi=-8.0):
        f = frame([(t,) for t in bf], bf_index, lo, hi)
        return f.iloc[perm]

    plasma, rates = [], []
    for it in range(n_iterations):
        t = rng.uniform(6e3, 1.4e4, S)
        lnd = g[:, None] * np.exp(-levels.energy.to_numpy()[:, None] / (K_BOLTZMANN * t[None, :])) * np.geomspace(1e9, 1e7, S)[None, :]
        lnd *= np.exp(rng.normal(0.0, 0.3, S))[None, :]   # per shell: no inverted pairs, so every probability is >= 0
        for key in zero:
            lnd[row_of[key]] = 0.0
        plasma.append(PlasmaState(np.ascontiguousarray(lnd), np.ascontiguousarray(10 ** rng.uniform(-9, -5, (L, S))), 1.0e6 * (1 + it)))
        coll_keys = [((a, i, lo), (a, i, up)) for a, i, lo, up in coll]
        pi = by_level()
        if infinite_rate and it == n_iterations - 1:
            pi.iloc[int(np.flatnonzero(perm == 0)[0]), 0] = np.inf      # the H ground state (energy 0): inf * 0 = NaN
            pi.iloc[int(np.flatnonzero(perm == 1)[0]), 0] = np.inf      # the first excited H level: its block -> 0 / inf
        r = dict(
            stim_recomb_corrected_photoionization_rate_coeff=pi,
            spontaneous_recombination_coeff=by_level(-13.0, -11.0),
            coll_deexc_coeff=frame(coll_keys, coll_index, -9.0, -6.0),
            coll_exc_coeff=frame(coll_keys, coll_index, -12.0, -7.0),
            coll_ion_coeff=by_level(-16.0, -10.0),
            coll_recomb_coeff=by_level(-22.0, -18.0),
            electron_densities=pd.Series(np.geomspace(1e9, 1e8, S) * rng.uniform(0.8, 1.2, S), index=columns),
            delta_E_yg=delta_E_yg,
            coll_exc_cool_rate=10 ** rng.uniform(-12, -9, S),
            coll_exc_cool_arr=rng.dirichlet(np.ones(len(coll)), S),
            coll_exc_cool_destinations=exc_dest,
            coll_ion_cool_rate=10 ** rng.uniform(-12, -9, S),
            coll_ion_cool_arr=rng.dirichlet(np.ones(len(bf)), S),
            fb_cool_rate=10 ** rng.uniform(-12, -9, S),
            fb_cool_probs_arr=rng.dirichlet(np.ones(len(bf)), S),
            ff_cool_rate=10 ** rng.uniform(-12, -9, S),
        )
        for k in ("coll_exc_cool_arr", "coll_ion_cool_arr", "fb_cool_probs_arr"):
            r[k][:, 0] = 0.0 if it == 0 else r[k][:, 0]   # a zero cooling channel in the first iteration
        rates.append(r)
    return ContinuumRateInputs(levels, lines, photoionization_data, ionization_energies, atomic, plasma, rates)


# ---------------------------------------------------------------------------------------------------------------------
# Inputs of the classic plasma (tb200_solve_plasma): an ion structure over make_atomic_data's levels
# ---------------------------------------------------------------------------------------------------------------------
EV_ERG = 1.602176565e-12  # CODATA-2010 (tardis/constants.py:1)


@dataclass
class PlasmaStructure:
    """Ions over the levels of an AtomicData, in the reference's frame order: elements in ascending atomic number, each with
    its ions of charge 0 ... Z (the bare ion included, as atomic data carry it), each ion a contiguous block of levels.
    `ionization_energy` is ionization_data of (Z, charge): the energy into the ion (NaN for charge 0)."""

    level_energy: np.ndarray       # f64[n_levels] erg: excitation energy (0 for the first level of every ion)
    level_ion: np.ndarray          # i64[n_levels] row of the level's ion
    ion_atomic_number: np.ndarray  # i64[n_ions]
    ion_charge: np.ndarray         # i64[n_ions]
    ionization_energy: np.ndarray  # f64[n_ions] erg
    number_density: np.ndarray     # f64[n_elements, S] cm^-3
    zeta_temperatures: np.ndarray  # f64[n_T] K
    zeta: np.ndarray               # f64[n_ions, n_T]


def make_plasma_structure(atomic: AtomicData, n_shells: int, atomic_numbers=tuple(range(1, 31)), seed: int = MODEL_SEED + 11,
                          log_density: tuple[float, float] = (3.0, 9.0)) -> PlasmaStructure:
    """Every ion gets at least one level and the rest of the levels are dealt out at random, in order.  A level's excitation
    energy is its `atomic.energy` above the first level of its ion.  Ionisation energies grow with the charge (5-15 eV times
    charge ** 1.3), so highly charged ions have Phi = 0 and populations below the zero threshold; zeta is U(0.05, 0.95) on a
    2000-40000 K grid."""
    rng = np.random.default_rng(seed)
    zs = np.asarray(atomic_numbers, dtype=np.int64)
    ion_z = np.concatenate([np.full(z + 1, z) for z in zs]).astype(np.int64)
    ion_q = np.concatenate([np.arange(z + 1) for z in zs]).astype(np.int64)
    n_ions, n = len(ion_z), atomic.n_levels
    if n < n_ions:
        raise ValueError(f"{n} levels cannot give {n_ions} ions one level each")
    per_ion = 1 + rng.multinomial(n - n_ions, np.full(n_ions, 1.0 / n_ions))
    level_ion = np.repeat(np.arange(n_ions, dtype=np.int64), per_ion)
    first = np.concatenate([[0], np.cumsum(per_ion)[:-1]])
    level_energy = atomic.energy - atomic.energy[first][level_ion]
    chi = rng.uniform(5.0, 15.0, n_ions) * np.maximum(ion_q, 1) ** 1.3 * EV_ERG
    chi[ion_q == 0] = np.nan
    nd = 10 ** rng.uniform(*log_density, (len(zs), n_shells))
    grid = np.arange(2000.0, 40001.0, 2000.0)
    zeta = rng.uniform(0.05, 0.95, (n_ions, len(grid)))
    return PlasmaStructure(np.ascontiguousarray(level_energy), level_ion, ion_z, ion_q, chi, np.ascontiguousarray(nd), grid, zeta)
