"""Transport decisions placed exactly at their thresholds, kernel against oracle.

Random packets on a log-uniform line list bring a boundary-versus-line decision within a few ulps of its threshold
about once in 1e15 traces, so the code the kernels keep for those cases (the full-relativity frequency window, the
virtual-packet windows, the continuum breakpoint ties, the close-distance recomputation in partial relativity) is never
run by the rest of the suite.  Here the workloads place lines or breakpoints at a packet's FIRST trace, at the
threshold computed with the oracle's own exported arithmetic (IEEE C, -ffp-contract=off), and a few ulps around it.

Each workload has two halves:
  * a CPU test (no gpu mark) that runs the oracle and proves the placements are sharp: moving them by the smallest
    step changes the oracle's integer outcome for a stated number of packets;
  * a GPU test that runs every kernel that makes the decision on the same inputs and requires the oracle's integers
    exactly (counters, fates, last-interaction columns, event logs), per-packet floats to 1e-11, estimators to 1e-10
    with the exact zero pattern of J_blue / Edotlu, and vhist to 1e-11.
"""
from __future__ import annotations

import copy
import functools
import math

import numpy as np
import pytest

from golden_util import assert_close

C_LIGHT = 2.99792458e10  # the oracle's and the kernels' C_SPEED_OF_LIGHT
TAU_LINE = 1e3           # a placed line always stops a trace that reaches it (tau_event = -log(u) < 40)
N_E_SCALE = 1e-6         # electron scattering so thin that no continuum distance can tie with anything
NU_KEY_SHIFT = 36        # the kernels' frequency-bucket key: the top 28 bits of the binary64 pattern
N_TRACKED = 1000         # packets whose event logs are compared (all of them in workloads 1-3)
MAX_EVENTS = 64


def _bits(x: float) -> int:
    return int(np.float64(x).view(np.int64))


def _from_bits(b: int) -> float:
    return float(np.int64(b).view(np.float64))


def _step(x: float, k: int) -> float:
    """x moved by k ulps (positive doubles: the bit pattern is monotone)."""
    return _from_bits(_bits(x) + k)


def _last_true(pred, lo: float, hi: float) -> float:
    """Largest double in [lo, hi) with pred true, for pred monotone (true below, false above)."""
    a, b = _bits(lo), _bits(hi)
    assert pred(lo) and not pred(hi)
    while b - a > 1:
        m = (a + b) // 2
        if pred(_from_bits(m)):
            a = m
        else:
            b = m
    return _from_bits(a)


@functools.lru_cache(maxsize=None)
def _oracle():
    from oracle import cpu_oracle

    cpu_oracle.build()
    return cpu_oracle


# ---------------------------------------------------------------------------------------------------------------------
# First-trace state of a packet injected at r with the source's (comoving) nu0, mu0, restated from the oracle's
# single_packet_loop / packet_propagation_iip: nu0 to the lab frame, with full relativity mu0 aberrated.
# ---------------------------------------------------------------------------------------------------------------------
def first_trace_state(r, nu0, mu0, t_exp, r_inner, r_outer, full_rel):
    o = _oracle()
    velocity = r / t_exp
    nu = nu0 * o.inverse_doppler_factor(velocity, mu0, full_rel)
    mu = mu0
    if full_rel:
        beta = (r / t_exp) / C_LIGHT
        mu = (mu0 + beta) / (1 + beta * mu0)
    comov_nu = nu * o.doppler_factor(velocity, mu, full_rel)
    d_b, delta = o.distance_boundary(r, mu, r_inner, r_outer)
    return nu, mu, comov_nu, d_b, delta


def kernel_nu_b(r, mu, nu, comov_nu, d_b, t_exp, full_rel):
    """The comoving frequency at the boundary point as the jump kernels compute it (trace_phase_a)."""
    inv_ct = 1.0 / (C_LIGHT * t_exp)
    if full_rel:
        r2 = r * r + d_b * d_b + 2.0 * r * d_b * mu
        beta2 = r2 * inv_ct * inv_ct
        return nu * (1.0 - (mu * r + d_b) * inv_ct) / math.sqrt(1.0 - beta2)
    return comov_nu - d_b * nu * inv_ct


def line_tie(r, mu, nu, comov_nu, d_b, t_exp, full_rel, nu_guess):
    """nu*: the largest line frequency that a trace from (r, mu, nu) does not reach before its boundary
    (d_boundary <= d_line, the test of trace_packet and trace_vpacket_within_shell); one ulp above it, it does."""
    o = _oracle()

    def boundary_first(nu_l):
        d, err = o.distance_line(r, mu, nu, comov_nu, False, nu_l, t_exp, full_rel)
        assert err == 0
        return d_b <= d

    return _last_true(boundary_first, nu_guess * (1 - 1e-9), comov_nu)


def with_lines(model, placed):
    """`model` with one line per packet at `placed` (tau TAU_LINE in shell 0, 0 elsewhere) and a last line far below
    the first traces (no trace interacts with the last line of the list)."""
    m = copy.copy(model)
    nu = np.sort(np.asarray(placed, dtype=np.float64))[::-1]
    nu = np.concatenate([nu, [nu[-1] * 0.5]])
    tau = np.zeros((len(nu), model.n_shells))
    tau[:-1, 0] = TAU_LINE
    m.line_list_nu, m.tau_sobolev = np.ascontiguousarray(nu), tau
    return m


def assert_sweeps_disjoint(lo, hi, placed):
    """Packet i's first traces sweep the comoving frequencies [lo_i, hi_i]; its own line must lie in there and no other
    packet's line may."""
    lines = np.sort(placed)
    inside = np.searchsorted(lines, hi, "right") - np.searchsorted(lines, lo, "left")
    assert (inside == 1).all() and (lo <= placed).all() and (placed <= hi).all()


def spaced_frequencies(sweep_frac, start=1e14, gap=1e-3):
    """Source frequencies nu0_i, ascending, such that the sweeps [nu0_i (1 - sweep_frac_i), nu0_i] are apart by `gap`."""
    nu0 = np.empty(len(sweep_frac))
    top = start
    for i, f in enumerate(sweep_frac):
        nu0[i] = top * (1 + gap) / (1 - f)
        top = nu0[i] * (1 + gap)
    return nu0


def shell0_model(v_shells, seed):
    """A 4-shell scatter model with velocity edges `v_shells` (units of c) and thin electron scattering."""
    from tardis_b200 import synthetic as syn

    model = syn.make_model(len(v_shells) - 1, 8, "scatter", seed=seed, duplicate_fraction=0.0)
    v = np.asarray(v_shells) * C_LIGHT
    t = model.time_explosion
    model.v_inner, model.v_outer = v[:-1].copy(), v[1:].copy()
    model.r_inner, model.r_outer = v[:-1] * t, v[1:] * t
    model.electron_density = model.electron_density * N_E_SCALE
    return model


# ---------------------------------------------------------------------------------------------------------------------
# Comparison against the oracle
# ---------------------------------------------------------------------------------------------------------------------
INT_COLUMNS = ("last_interaction_type", "last_event_id", "last_shell_id", "last_line_absorb_id", "last_line_emit_id")
FLOAT_COLUMNS = ("last_radius", "last_before_nu", "last_before_mu", "last_before_energy", "last_after_nu", "last_after_mu",
                 "last_after_energy")
CONT_ESTIMATORS = ("photo_ion_estimator", "stim_recomb_estimator", "bf_heating_estimator", "stim_recomb_cooling_estimator",
                   "ff_heating_estimator")


def run_oracle(model, packets, n_tracked=N_TRACKED, max_events=MAX_EVENTS, **kw):
    ref = _oracle().run_oracle(model, packets, n_tracked_packets=min(n_tracked, len(packets)), max_events_per_packet=max_events,
                               **kw)
    assert (ref["event_counts"] < max_events).all()  # whole logs: the oracle stops counting at the capacity, the engine does not
    return ref


def run_engine(eng, model, packets, n_tracked=N_TRACKED, max_events=MAX_EVENTS, **cfg):
    eng.set_model_from(model, **cfg)
    return eng.run_packets(packets, track_last_interaction=True, n_tracked_packets=min(n_tracked, len(packets)),
                           max_events_per_packet=max_events)


def assert_matches_oracle(res, ref, what):
    for k, v in ref["counters"].items():
        assert res["counters"][k] == v, (what, k, res["counters"][k], v)
    assert np.array_equal(np.sign(res["output_energies"]), np.sign(ref["output_energies"])), what
    assert np.array_equal(res["output_energies"] == -99.0, ref["output_energies"] == -99.0), what
    for k in INT_COLUMNS:
        assert np.array_equal(res[k], ref[k]), (what, k)
    assert np.array_equal(res["event_counts"], ref["event_counts"]), what
    a, b = np.concatenate(res["events"]), np.concatenate(ref["events"])
    for k in ("packet_id", "interaction_type", "status", "before_shell_id", "after_shell_id", "line_absorb_id", "line_emit_id"):
        assert np.array_equal(a[k], b[k]), (what, "event " + k)
    for k in ("radius", "before_nu", "before_mu", "before_energy", "after_nu", "after_mu", "after_energy"):
        assert_close(a[k], b[k], 1e-11, f"{what}: event_{k}")
    for k in ("output_nus", "output_energies") + FLOAT_COLUMNS:
        assert_close(res[k], ref[k], 1e-11, f"{what}: {k}")
    for k in ("j", "nu_bar", "j_blue", "edotlu"):
        assert_close(res[k], ref[k], 1e-10, f"{what}: {k}")
    for k in ("j_blue", "edotlu"):
        assert np.array_equal(res[k] == 0, ref[k] == 0), (what, k + " zero pattern")
    assert_close(res["vhist"], ref["vhist"], 1e-11, f"{what}: vhist")
    if "photo_ion_estimator" in ref:
        for k in CONT_ESTIMATORS:
            assert_close(res[k], ref[k], 1e-10, f"{what}: {k}")
        assert np.array_equal(res["photo_ion_estimator_statistics"], ref["photo_ion_estimator_statistics"]), what


# kernel choices (engine options); none of them may change a result
SCAN = {"algorithm": 0}
POOLED = {"algorithm": 1, "pooled": 1}
LANE = {"algorithm": 1, "pooled": 0}
VOLLEY_1 = {"algorithm": 1, "vol_min": 1}
VOLLEY_32 = {"algorithm": 1, "vol_min": 32}


def check_kernel(options, cases):
    """Run every (name, model, packets, engine config, event tracking, oracle result) case on an engine with `options`.
    The engine configs use the oracle's keyword names."""
    from tardis_b200.engine import Engine

    eng = Engine(0)
    try:
        for k, v in options.items():
            eng.set_option(k, v)
        for name, model, packets, cfg, track, ref in cases:
            assert_matches_oracle(run_engine(eng, model, packets, **track, **cfg), ref, name)
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# Workload 1: boundary / line ties at the first trace, partial and full relativity
# ---------------------------------------------------------------------------------------------------------------------
ULP_STEPS = tuple(range(-6, 7))
WINDOW_EDGES = tuple(s * w for w in (1e-12 * (1 - 1e-6), 1e-12 * (1 + 1e-6), 1e-13, 1e-11) for s in (-1.0, 1.0))


@functools.lru_cache(maxsize=None)
def boundary_ties(full_rel: bool, n_groups: int = 4, group: int = 250, seed: int = 4101):
    """`n_groups` x `group` packets at r_inner[0] with mu > 0.  Shell 0 is thick (0.05 c to 0.08 c), so that one ulp of a
    line frequency is a few tens of ulps of distance and the partial-relativity product can round across the threshold.
    Inside a group the frequencies are spaced so that no packet's first trace can meet another packet's line; each group
    is its own run and spans ~1e4 in frequency (the jump kernels' fixed-point line estimators hold one scale per run).
    -> (model, [(packets, state [group, 5] = (nu, mu, comov_nu, d_boundary, kernel nu_b), nu* [group])] per group)."""
    from tardis_b200 import synthetic as syn

    model = shell0_model([0.05, 0.08, 0.10, 0.12, 0.14], seed)
    rng = np.random.default_rng(seed)
    t, r0, ro = model.time_explosion, float(model.r_inner[0]), float(model.r_outer[0])
    groups = []
    for _ in range(n_groups):
        mus0 = rng.uniform(0.6, 1.0, group)
        frac = np.array([first_trace_state(r0, 1.0, m, t, r0, ro, full_rel)[3] / (C_LIGHT * t) * 1.05 for m in mus0])
        nus0 = spaced_frequencies(frac)
        st = np.empty((group, 5))
        ties = np.empty(group)
        for i in range(group):
            nu, mu, comov, d_b, delta = first_trace_state(r0, nus0[i], mus0[i], t, r0, ro, full_rel)
            assert delta == 1
            nu_b = kernel_nu_b(r0, mu, nu, comov, d_b, t, full_rel)
            st[i] = (nu, mu, comov, d_b, nu_b)
            ties[i] = line_tie(r0, mu, nu, comov, d_b, t, full_rel, nu_b)
        packets = syn.Packets(np.full(group, r0), nus0, mus0, np.full(group, 1.0 / group),
                              rng.integers(1, 2**32 - 1, group).astype(np.int64), 1.0)
        groups.append((packets, st, ties))
    return model, groups


def boundary_tie_placements(st, ties, full_rel):
    """(name, line frequency per packet) of the workload-1 runs of one group: nu* + k ulps, and with full relativity the
    edges of the phase-A window nu_b (1 +- 1e-12) and points well inside and outside it."""
    out = [(f"nu*{k:+d}ulp", np.array([_step(x, k) for x in ties])) for k in ULP_STEPS]
    if full_rel:
        out += [(f"nu_b*(1{w:+.7g})", st[:, 4] * (1.0 + w)) for w in WINDOW_EDGES]
    return out


def first_outcome(res):
    """(interaction type, absorbing line) of each tracked packet's first event after injection."""
    return np.array([(e[1]["interaction_type"], e[1]["line_absorb_id"]) for e in res["events"]])


@pytest.mark.parametrize("full_rel", [False, True], ids=["partial_rel", "full_rel"])
def test_boundary_line_ties_are_sharp(full_rel):
    """At nu* every packet crosses the boundary, one ulp above it every packet meets its own line (1000 packets); no
    packet's first trace can reach another packet's line; and in partial relativity the kernels' product
    nu_diff * (c t (1/nu)) decides at least 5 placements the other way from the reference's (nu_diff / nu) * c * t."""
    o = _oracle()
    model, groups = boundary_ties(full_rel)
    t, r0, ct = model.time_explosion, float(model.r_inner[0]), C_LIGHT * model.time_explosion
    forks = sharp = 0
    for packets, st, ties in groups:
        n = len(packets)
        at = run_oracle(with_lines(model, ties), packets, enable_full_relativity=full_rel)
        above = run_oracle(with_lines(model, [_step(x, 1) for x in ties]), packets, enable_full_relativity=full_rel)
        a, b = first_outcome(at), first_outcome(above)
        assert (a[:, 1] == -1).all()                           # boundary crossing
        assert np.array_equal(b[:, 1], n - 1 - np.arange(n))   # the packet's own line (lines are sorted by descending nu)
        sharp += (a != b).any(axis=1).sum()
        for name, placed in boundary_tie_placements(st, ties, full_rel):
            assert_sweeps_disjoint(st[:, 4] * (1 - 1e-9), st[:, 2], placed)
        if not full_rel:
            for k in ULP_STEPS:
                for i in range(n):
                    nu, mu, comov, d_b = st[i, :4]
                    nu_l = _step(ties[i], k)
                    literal, _ = o.distance_line(r0, mu, nu, comov, False, nu_l, t, False)
                    product = (comov - nu_l) * (ct * (1.0 / nu))
                    forks += (d_b <= literal) != (d_b <= product)
    assert sharp == 1000
    assert full_rel or forks >= 5


@functools.lru_cache(maxsize=None)
def boundary_tie_cases(full_rel):
    model, groups = boundary_ties(full_rel)
    cfg = dict(enable_full_relativity=full_rel)
    out = []
    for g, (packets, st, ties) in enumerate(groups):
        for name, placed in boundary_tie_placements(st, ties, full_rel):
            m = with_lines(model, placed)
            out.append((f"group {g} {name}", m, packets, cfg, {}, run_oracle(m, packets, **cfg)))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", [SCAN, POOLED, LANE], ids=["scan", "pooled", "lane"])
@pytest.mark.parametrize("full_rel", [False, True], ids=["partial_rel", "full_rel"])
def test_boundary_line_ties_match_the_oracle(kernel, full_rel):
    check_kernel(kernel, boundary_tie_cases(full_rel))


# ---------------------------------------------------------------------------------------------------------------------
# Workload 2: virtual-packet window ties.  Every packet owes a volley of two virtual packets at injection; the first one
# draws its direction first (trace_vpacket_volley: mu = mu_min + (0 + u) * mu_bin, mu_min = 0 on the inner boundary), and
# its line is placed where that virtual packet reaches the outer boundary of shell 0.
# ---------------------------------------------------------------------------------------------------------------------
N_VPACKETS = 2


def first_vpacket(r, nu0, mu0, seed, t_exp, r_inner, r_outer, full_rel):
    """-> (v_nu, v_mu, comov_nu, d_boundary) of the packet's first virtual packet, and the packet's own first trace."""
    o = _oracle()
    nu, mu, comov, d_b, _ = first_trace_state(r, nu0, mu0, t_exp, r_inner, r_outer, full_rel)
    velocity = r / t_exp
    v_mu = 0.0 + 0 * (1.0 / N_VPACKETS) + o.rng_double(int(seed), 0) * ((1.0 - 0.0) / N_VPACKETS)
    if full_rel:
        beta = r / (C_LIGHT * t_exp)
        v_mu = (v_mu + beta) / (1.0 + beta * v_mu)
    v_nu = nu * (o.doppler_factor(velocity, mu, full_rel) / o.doppler_factor(velocity, v_mu, full_rel))
    v_comov = v_nu * o.doppler_factor(velocity, v_mu, full_rel)
    v_db, delta = o.distance_boundary(r, v_mu, r_inner, r_outer)
    assert delta == 1
    return (v_nu, v_mu, v_comov, v_db), (nu, mu, comov, d_b)


def volley_nu_stop(r, v_mu, v_nu, r_outer, t_exp, full_rel):
    """The comoving frequency at which the warp volley's closed form puts the virtual packet at r_outer[0]."""
    inv_ct = 1.0 / (C_LIGHT * t_exp)
    s_x = math.sqrt(r_outer * r_outer - r * r * (1.0 - v_mu * v_mu))
    if full_rel:
        bx = r_outer * inv_ct
        return v_nu * (1.0 - s_x * inv_ct) / math.sqrt(1.0 - bx * bx)
    return v_nu * (1.0 - s_x * inv_ct)


@functools.lru_cache(maxsize=None)
def vpacket_ties(full_rel: bool, n: int = 1000, seed: int = 4202):
    """`n` packets at r_inner[0] with mu0 in [0.6, 1): their own first trace and their second virtual packet (mu >= 0.5)
    end above the first virtual packet's boundary frequency, so its line is met by that virtual packet alone.
    -> (model, packets, nu_stop of the warp volley [n], nu* [n], sweep bottoms [n], sweep tops [n])."""
    from tardis_b200 import synthetic as syn

    model = shell0_model([0.05, 0.052, 0.06, 0.07, 0.08], seed)
    rng = np.random.default_rng(seed)
    t, r0, ro = model.time_explosion, float(model.r_inner[0]), float(model.r_outer[0])
    mus0 = rng.uniform(0.6, 1.0, n)
    seeds = rng.integers(1, 2**32 - 1, n).astype(np.int64)
    vp = [first_vpacket(r0, 1.0, mus0[i], seeds[i], t, r0, ro, full_rel) for i in range(n)]
    frac = np.array([(v[3] / (C_LIGHT * t)) * 1.05 for v, _ in vp])
    nus0 = spaced_frequencies(frac)
    stop, ties, lo, hi = (np.empty(n) for _ in range(4))
    for i in range(n):
        (v_nu, v_mu, v_comov, v_db), (nu, mu, comov, d_b) = first_vpacket(r0, nus0[i], mus0[i], seeds[i], t, r0, ro, full_rel)
        assert d_b < v_db
        stop[i] = volley_nu_stop(r0, v_mu, v_nu, ro, t, full_rel)
        ties[i] = line_tie(r0, v_mu, v_nu, v_comov, v_db, t, full_rel, stop[i])
        lo[i] = stop[i] * (1 - 1e-9)
        hi[i] = max(comov, v_comov) * (1 + 1e-9)
        # the packet's own first trace ends above the line
        assert kernel_nu_b(r0, mu, nu, comov, d_b, t, full_rel) > stop[i] * (1 + 1e-9)
    packets = syn.Packets(np.full(n, r0), nus0, mus0, np.full(n, 1.0 / n), seeds, 1.0)
    grid_lo, grid_hi = 0.5 * lo.min(), 2.0 * hi.max()
    model.spectrum_frequency_grid = np.linspace(grid_lo, grid_hi, 4001)
    return model, packets, stop, ties, lo, hi


def vpacket_tie_placements(full_rel):
    model, packets, stop, ties, lo, hi = vpacket_ties(full_rel)
    out = [(f"vp nu*{k:+d}ulp", np.array([_step(x, k) for x in ties])) for k in ULP_STEPS]
    out += [(f"nu_stop*(1{w:+.7g})", stop * (1.0 + w)) for w in WINDOW_EDGES[:4]]
    return out


def first_vpacket_energy(res, n):
    """Energy the first virtual packet of every packet's first volley leaves in the log."""
    m = res["vlog_count"]
    idx = res["vlog_packet_index"][:m]
    first = np.searchsorted(idx, np.arange(n))  # the log is in packet order (one thread), each volley in draw order
    assert np.array_equal(idx[first], np.arange(n))
    return res["vlog_energies"][:m][first]


@pytest.mark.parametrize("full_rel", [False, True], ids=["partial_rel", "full_rel"])
def test_vpacket_window_ties_are_sharp(full_rel):
    """At nu* the first virtual packet stops before its line and escapes with energy; one ulp above it crosses the line
    (tau 1e3), so Russian roulette (survival probability 0) kills it: for every packet.  No first trace meets another
    packet's line."""
    model, packets, stop, ties, lo, hi = vpacket_ties(full_rel)
    n = len(packets)
    kw = dict(enable_full_relativity=full_rel, number_of_vpackets=N_VPACKETS, vlog_capacity=40 * n)
    at = _oracle().run_oracle(with_lines(model, ties), packets, **kw)
    above = _oracle().run_oracle(with_lines(model, [_step(x, 1) for x in ties]), packets, **kw)
    ea, eb = first_vpacket_energy(at, n), first_vpacket_energy(above, n)
    assert (ea > 0).all() and (eb == 0).all()
    assert above["counters"]["n_rng_draws"] == at["counters"]["n_rng_draws"] + n
    for name, placed in vpacket_tie_placements(full_rel):
        assert_sweeps_disjoint(lo, hi, placed)


@functools.lru_cache(maxsize=None)
def vpacket_tie_cases(full_rel):
    model, packets, _, _, _, _ = vpacket_ties(full_rel)
    cfg = dict(enable_full_relativity=full_rel, number_of_vpackets=N_VPACKETS)
    out = []
    for name, placed in vpacket_tie_placements(full_rel):
        m = with_lines(model, placed)
        out.append((name, m, packets, cfg, {}, run_oracle(m, packets, **cfg)))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", [VOLLEY_1, VOLLEY_32, SCAN], ids=["volley_min1", "volley_min32", "scan"])
@pytest.mark.parametrize("full_rel", [False, True], ids=["partial_rel", "full_rel"])
def test_vpacket_window_ties_match_the_oracle(kernel, full_rel):
    check_kernel(kernel, vpacket_tie_cases(full_rel))


# ---------------------------------------------------------------------------------------------------------------------
# Workload 3: continuum breakpoint ties.  One packet per phot_nus breakpoint; the breakpoint is moved onto the packet's
# first comoving frequency (a shift of ~1e-16 relative, the table stays ascending).  The first point of a block is where
# the reference's index arithmetic wraps (searchsorted gives 0, the lower neighbour becomes the block's last point).
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def breakpoint_ties(seed: int = 4303):
    """-> (model with breakpoints at the packets' first comoving frequencies, the same with them 1 ulp higher, packets)."""
    from tardis_b200 import synthetic as syn

    model = syn.make_model(6, 2000, "macroatom", mu_tau=-4.0, seed=seed)
    syn.add_continuum(model, seed=seed + 1, n_continua=30, points=(4, 9))  # (at most 30: photo_ion_activation_idx)
    cont = model.continuum
    n = len(cont.phot_nus)
    rng = np.random.default_rng(seed)
    t, r0, ro = model.time_explosion, float(model.r_inner[0]), float(model.r_outer[0])
    mus0 = np.sqrt(rng.uniform(0.0, 1.0, n))
    nus0 = cont.phot_nus.copy()
    comov = np.array([first_trace_state(r0, nus0[i], mus0[i], t, r0, ro, True)[2] for i in range(n)])
    assert np.all(np.abs(comov / nus0 - 1) < 1e-14)
    base = syn.make_packets(n, r0, base_seed=seed)
    packets = syn.Packets(np.full(n, r0), nus0, mus0, base.initial_energies, base.packet_seeds, base.radiation_field_luminosity)

    def tabled(points):
        m = copy.copy(model)
        c = copy.copy(cont)
        refs = c.photo_ion_block_references
        c.phot_nus = np.ascontiguousarray(points)
        c.photo_ion_nu_threshold_mins = c.phot_nus[refs[:-1]].copy()
        c.photo_ion_nu_threshold_maxs = c.phot_nus[refs[1:] - 1].copy()
        m.continuum = c
        return m

    return tabled(comov), tabled(np.array([_step(x, 1) for x in comov])), packets


def test_breakpoint_ties_are_sharp():
    """Tied and 1-ulp-moved breakpoints give different continuum estimators, and different photo-ionisation counts
    (a frequency tied with a block's first point lies inside the block; with that point one ulp higher, outside)."""
    at_model, moved_model, packets = breakpoint_ties()
    cont = at_model.continuum
    assert len(packets) == len(cont.phot_nus) and np.all(np.diff(cont.phot_nus[cont.photo_ion_block_references[0]:]) != 0)
    at = _oracle().run_oracle(at_model, packets)
    moved = _oracle().run_oracle(moved_model, packets)
    for k in ("photo_ion_estimator", "bf_heating_estimator"):
        assert not np.array_equal(at[k], moved[k]), k
    stats = at["photo_ion_estimator_statistics"].sum() - moved["photo_ion_estimator_statistics"].sum()
    assert stats >= len(cont.bf_threshold_list_nu) // 2


@functools.lru_cache(maxsize=None)
def breakpoint_tie_cases():
    at_model, moved_model, packets = breakpoint_ties()
    track = dict(max_events=256)
    return [(name, m, packets, {}, track, run_oracle(m, packets, **track)) for name, m in (("tied", at_model), ("moved", moved_model))]


@pytest.mark.gpu
@pytest.mark.parametrize("ctas", [2, 3])
@pytest.mark.parametrize("pooled", [1, 0], ids=["pooled", "lane"])
def test_breakpoint_ties_match_the_oracle(pooled, ctas):
    check_kernel({"algorithm": 1, "pooled": pooled, "ctas_per_sm": ctas}, breakpoint_tie_cases())


# ---------------------------------------------------------------------------------------------------------------------
# Workload 4: a clustered line list.  Most lines sit in frequency buckets (NU_KEY_SHIFT) of 12 lines, which sends the
# boundary guess to its bisection branch and the virtual packets to vp_first_break_search; some lines sit exactly on
# bucket edges; the list covers only the middle of the packets' spectrum, so boundary frequencies fall above the highest
# and below the lowest bucket.
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def clustered_model(seed: int = 4404):
    from tardis_b200 import synthetic as syn

    model = syn.make_model(8, 6000, "macroatom", mu_tau=-2.5, seed=seed, duplicate_fraction=0.0)
    rng = np.random.default_rng(seed)
    L = model.n_lines
    lo_key, hi_key = _bits(4e14) >> NU_KEY_SHIFT, _bits(1.2e15) >> NU_KEY_SHIFT
    keys = rng.choice(np.arange(lo_key, hi_key), (L * 3) // 4 // 12, replace=False)
    nu = [_from_bits(int((k << NU_KEY_SHIFT) + b)) for k in keys for b in rng.integers(1, 1 << NU_KEY_SHIFT, 12)]
    edges = rng.choice(np.arange(lo_key + 1, hi_key), L // 20, replace=False)
    nu += [_from_bits(int(k << NU_KEY_SHIFT)) for k in edges]
    nu += list(np.exp(rng.uniform(np.log(4e14), np.log(1.2e15), L - len(nu))))
    model.line_list_nu = np.ascontiguousarray(np.sort(np.array(nu))[::-1])
    assert len(model.line_list_nu) == L
    packets = syn.make_packets(20000, model.r_inner[0], base_seed=seed)
    return model, packets


def test_clustered_line_list_is_clustered():
    model, packets = clustered_model()
    nu = model.line_list_nu
    keys = np.array([_bits(x) >> NU_KEY_SHIFT for x in nu])
    _, inverse, counts = np.unique(keys, return_inverse=True, return_counts=True)
    assert (counts[inverse] >= 9).mean() > 0.5                       # most lines share a bucket with >= 8 others
    on_edge = np.array([(_bits(x) & ((1 << NU_KEY_SHIFT) - 1)) == 0 for x in nu])
    assert on_edge.sum() >= len(nu) // 25
    # boundary frequencies of first traces (partial relativity) beyond both ends of the list
    t, r0 = model.time_explosion, model.r_inner[0]
    mu = packets.initial_mus
    nu_lab = packets.initial_nus / (1.0 - mu * (r0 / t) / C_LIGHT)
    d_b = np.sqrt(model.r_outer[0] ** 2 + (mu * mu - 1.0) * r0 * r0) - r0 * mu
    nu_b = nu_lab * (1.0 - mu * (r0 / t) / C_LIGHT) - d_b * nu_lab / (C_LIGHT * t)
    assert (nu_b > nu[0]).sum() > 1000 and (nu_b < nu[-1]).sum() > 1000


@functools.lru_cache(maxsize=None)
def clustered_cases(vpackets: int):
    model, packets = clustered_model()
    out = []
    for full_rel in (False, True):
        cfg = dict(enable_full_relativity=full_rel, number_of_vpackets=vpackets)
        track = dict(n_tracked=200, max_events=4096)
        out.append((f"clustered fr={full_rel} vp={vpackets}", model, packets, cfg, track,
                    run_oracle(model, packets, nthreads=8, **track, **cfg)))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,vpackets", [(SCAN, 0), (POOLED, 0), (LANE, 0), (VOLLEY_1, 3), (SCAN, 3)],
                         ids=["scan", "pooled", "lane", "volley", "scan_vpackets"])
def test_clustered_line_list_matches_the_oracle(kernel, vpackets):
    check_kernel(kernel, clustered_cases(vpackets))
