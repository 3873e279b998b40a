"""Phase B of the jump kernels against the oracle: the search for a parked trace's stopping line and the classic macro atom.

Phase B finds the first line at which a parked trace stops by a search over the tau prefix table, and draws macro-atom
jumps by a search inside a guide-table bracket of running sums.  Random workloads rarely force the cases these searches
have to get exactly right:
  * a stopping line at the first, the last and every split position of the searched interval, in partial and full
    relativity: one placed line per run, at every position of a 64-line interval;
  * macro-atom blocks whose probabilities are so skewed that guide brackets are wide, blocks of one transition, and a
    block whose probabilities sum to less than one (MacroAtomError).
The GPU tests require the oracle's integers exactly (counters, fates, last-interaction columns, event logs).
"""
from __future__ import annotations

import copy
import functools

import numpy as np
import pytest

from golden_util import assert_close

C_LIGHT = 2.99792458e10
N_INNER = 64        # lines inside the first trace's sweep; the placed line takes each of their positions in turn
N_PACKETS = 64
MAX_EVENTS = 64
TAU_STOP = 1e3      # the placed line always stops a trace that reaches it (tau_event = -log(u) < 40)

POOLED = {"algorithm": 1, "pooled": 1}
LANE = {"algorithm": 1, "pooled": 0}


@functools.lru_cache(maxsize=None)
def _oracle():
    from oracle import cpu_oracle

    cpu_oracle.build()
    return cpu_oracle


def run_oracle(model, packets, **kw):
    ref = _oracle().run_oracle(model, packets, n_tracked_packets=len(packets), max_events_per_packet=MAX_EVENTS, **kw)
    assert (ref["event_counts"] < MAX_EVENTS).all()
    return ref


def assert_matches_oracle(res, ref, what):
    for k, v in ref["counters"].items():
        assert res["counters"][k] == v, (what, k, res["counters"][k], v)
    assert np.array_equal(np.sign(res["output_energies"]), np.sign(ref["output_energies"])), what
    for k in ("last_interaction_type", "last_event_id", "last_shell_id", "last_line_absorb_id", "last_line_emit_id"):
        assert np.array_equal(res[k], ref[k]), (what, k)
    assert np.array_equal(res["event_counts"], ref["event_counts"]), what
    a, b = np.concatenate(res["events"]), np.concatenate(ref["events"])
    for k in ("packet_id", "interaction_type", "status", "before_shell_id", "after_shell_id", "line_absorb_id", "line_emit_id"):
        assert np.array_equal(a[k], b[k]), (what, "event " + k)
    for k in ("radius", "before_nu", "before_mu", "after_nu", "after_mu"):
        assert_close(a[k], b[k], 1e-11, f"{what}: event_{k}")
    for k in ("output_nus", "output_energies"):
        assert_close(res[k], ref[k], 1e-11, f"{what}: {k}")
    for k in ("j", "nu_bar", "j_blue", "edotlu"):
        assert_close(res[k], ref[k], 1e-10, f"{what}: {k}")


def check_kernel(options, cases):
    from tardis_b200.engine import Engine

    eng = Engine(0)
    try:
        for k, v in options.items():
            eng.set_option(k, v)
        for name, model, packets, cfg, ref in cases:
            eng.set_model_from(model, **cfg)
            res = eng.run_packets(packets, track_last_interaction=True, n_tracked_packets=len(packets),
                                  max_events_per_packet=MAX_EVENTS)
            assert_matches_oracle(res, ref, name)
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# Workload 1: the stopping line of a parked trace at every position of the searched interval
# ---------------------------------------------------------------------------------------------------------------------
def sweep_model(seed: int = 5101):
    """Four scatter shells (0.05 c to 0.14 c), thin electron scattering, and N_PACKETS packets at r_inner[0] with one
    frequency and direction: every first trace sweeps the same comoving frequencies [nu_b, nu_cmf].  N_INNER lines lie
    evenly in the middle half of that sweep (tau 0), one more far below it.  -> (model, packets, inner line frequencies)."""
    from tardis_b200 import synthetic as syn

    model = syn.make_model(4, 8, "scatter", seed=seed, duplicate_fraction=0.0)
    v = np.array([0.05, 0.08, 0.10, 0.12, 0.14]) * C_LIGHT
    t = model.time_explosion
    model.v_inner, model.v_outer = v[:-1].copy(), v[1:].copy()
    model.r_inner, model.r_outer = v[:-1] * t, v[1:] * t
    model.electron_density = model.electron_density * 1e-6
    r0, ro, mu0, nu0 = float(model.r_inner[0]), float(model.r_outer[0]), 0.9, 1.0e15
    d_b = np.sqrt(ro * ro - r0 * r0 * (1 - mu0 * mu0)) - r0 * mu0
    nu_b = nu0 * (1 - d_b / (C_LIGHT * t) / (1 - r0 * mu0 / (C_LIGHT * t)))  # about; the middle half is far from its edges
    inner = np.linspace(nu0 - 0.25 * (nu0 - nu_b), nu_b + 0.25 * (nu0 - nu_b), N_INNER)
    rng = np.random.default_rng(seed)
    packets = syn.Packets(np.full(N_PACKETS, r0), np.full(N_PACKETS, nu0), np.full(N_PACKETS, mu0),
                          np.full(N_PACKETS, 1.0 / N_PACKETS), rng.integers(1, 2**32 - 1, N_PACKETS).astype(np.int64), 1.0)
    return model, packets, inner


def with_stop(model, inner, j):
    """`model` with the inner lines and a last line far below; inner line j has tau TAU_STOP in shell 0."""
    m = copy.copy(model)
    nu = np.concatenate([inner, [inner[-1] * 0.5]])
    tau = np.zeros((len(nu), model.n_shells))
    tau[j, 0] = TAU_STOP
    m.line_list_nu, m.tau_sobolev = np.ascontiguousarray(nu), tau
    return m


def first_outcome(res):
    """(interaction type, absorbing line) of each packet's first event after injection."""
    return np.array([(e[1]["interaction_type"], e[1]["line_absorb_id"]) for e in res["events"]])


@functools.lru_cache(maxsize=None)
def stop_cases(full_rel: bool):
    model, packets, inner = sweep_model()
    cfg = dict(enable_full_relativity=full_rel)
    out = []
    for j in range(N_INNER):
        m = with_stop(model, inner, j)
        out.append((f"stop at inner line {j}", m, packets, cfg, run_oracle(m, packets, **cfg)))
    return out


@pytest.mark.parametrize("full_rel", [False, True], ids=["partial_rel", "full_rel"])
def test_every_packet_stops_at_the_placed_line(full_rel):
    """The placement is what it claims: in the oracle, every packet's first trace ends in a line interaction at the placed
    line, whichever of the N_INNER positions it takes."""
    for j, (name, m, packets, cfg, ref) in enumerate(stop_cases(full_rel)):
        first = first_outcome(ref)
        assert (first[:, 0] == 2).all(), name  # InteractionType.LINE
        assert (first[:, 1] == j).all(), name


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", [POOLED, LANE], ids=["pooled", "lane"])
@pytest.mark.parametrize("full_rel", [False, True], ids=["partial_rel", "full_rel"])
def test_stopping_line_at_every_position_matches_the_oracle(kernel, full_rel):
    check_kernel(kernel, stop_cases(full_rel))


# ---------------------------------------------------------------------------------------------------------------------
# Workload 2: skewed macro-atom blocks
# ---------------------------------------------------------------------------------------------------------------------
def block_of_rows(edges):
    return np.repeat(np.arange(len(edges) - 1), np.diff(edges))


@functools.lru_cache(maxsize=None)
def skewed_model(seed: int = 5202):
    """A macroatom model whose transition probabilities are log-normal with sigma 6 per (transition, shell), normalised
    per block: most of a block's weight sits in one or two transitions, so guide buckets pile up on them.  Half as many
    levels as lines: besides the large blocks of the popular levels there are blocks of a single transition."""
    from tardis_b200 import synthetic as syn

    model = syn.make_model(6, 3000, "macroatom", mu_tau=-3.0, seed=seed, n_levels=1500)
    mac = model.macro
    rng = np.random.default_rng(seed)
    edges = np.asarray(mac.macro_block_edge_index)
    raw = np.exp(rng.normal(0.0, 6.0, mac.transition_probabilities.shape))
    block = block_of_rows(edges)
    sums = np.zeros((len(edges) - 1, raw.shape[1]))
    np.add.at(sums, block, raw)
    mac.transition_probabilities = np.ascontiguousarray(raw / sums[block])
    return model


def guide_brackets(tp_col, edges):
    """Widest guide bracket of each block (macro_guide_kernel and macro_atom_event restated) for one shell's probabilities."""
    widths = np.zeros(len(edges) - 1, dtype=np.int64)
    for b in range(len(edges) - 1):
        b0, b1 = int(edges[b]), int(edges[b + 1])
        n = b1 - b0
        if n == 0:
            continue
        cum = np.cumsum(tp_col[b0:b1])
        g = np.array([min(int(np.searchsorted(cum, k / n, side="right")), n - 1) for k in range(n)])
        widths[b] = max((g[min(k + 2, n - 1)] if k + 2 < n else n - 1) - g[max(k - 1, 0)] for k in range(n))
    return widths


def test_skewed_blocks_have_wide_brackets_and_single_transitions():
    """The skewed model has blocks whose guide brackets span more than eight transitions and blocks of a single
    transition."""
    model = skewed_model()
    edges = np.asarray(model.macro.macro_block_edge_index)
    widths = guide_brackets(model.macro.transition_probabilities[:, 0], edges)
    assert (widths > 8).sum() >= 20
    assert (np.diff(edges) == 1).sum() >= 5


def skewed_packets(model, n=2000, seed=5203):
    from tardis_b200 import synthetic as syn

    return syn.make_packets(n, model.r_inner[0], base_seed=seed)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", [POOLED, LANE], ids=["pooled", "lane"])
@pytest.mark.parametrize("full_rel", [False, True], ids=["partial_rel", "full_rel"])
def test_skewed_macro_atom_matches_the_oracle(kernel, full_rel):
    model = skewed_model()
    packets = skewed_packets(model)
    cfg = dict(enable_full_relativity=full_rel)
    ref = run_oracle(model, packets, **cfg)
    assert ref["counters"]["n_macro_jumps"] > len(packets)
    check_kernel(kernel, [("skewed macro atom", model, packets, cfg, ref)])


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", [POOLED, LANE], ids=["pooled", "lane"])
def test_block_total_below_one_raises(kernel):
    """The block of the level that most lines activate sums to 0.5 in every shell: the oracle and the engine both stop
    with MacroAtomError ("MacroAtom ran out of the block")."""
    from tardis_b200.engine import Engine, MacroAtomError

    model = copy.deepcopy(skewed_model())
    mac = model.macro
    edges = np.asarray(mac.macro_block_edge_index)
    level = int(np.bincount(np.asarray(mac.line2macro_level_upper)).argmax())
    mac.transition_probabilities[edges[level]:edges[level + 1]] *= 0.5
    packets = skewed_packets(model, n=500)
    with pytest.raises(Exception, match="MacroAtom"):
        run_oracle(model, packets)
    eng = Engine(0)
    try:
        for k, v in kernel.items():
            eng.set_option(k, v)
        eng.set_model_from(model)
        with pytest.raises(MacroAtomError):
            eng.run_packets(packets)
    finally:
        eng.close()
