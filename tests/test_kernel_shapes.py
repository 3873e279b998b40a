"""Transport kernels at the shell counts where their dispatch changes, and with random streams long enough to reach every
tier of the generator, kernel against oracle.

The engine picks its transport kernel and its shared-memory layout from the shell count S, and refuses some shell counts
on the host.  These are the switches, each stated below as a formula over the constants the kernels are built with:
  * the pooled jump kernel runs while 4 S doubles of shell table plus the warps' packet pools fit in 110 KiB; above that
    the lane-resident jump kernel runs (classic mode: S <= 1344, continuum mode: S <= 576 at 256 threads per CTA);
  * the warp volleys pack virtual packets into sub-batches of cap = VOL_ITEMS - 2 S items, and from S = 160 (cap < 1) or
    S = 256 (a shell no longer fits the 8-bit meta field) every virtual packet takes the literal path;
  * more than 200 KiB of shell table (jump: S > 6400, scan: S > 12800), and jump layouts that exceed the CTA's shared
    memory (warp volleys: S > 5408 on an H100), are refused before a launch.
The generator of a packet has three tiers (transport_kernel.cuh): outputs 0..226 from the seed recurrence, 227..623 read
back from the packet's ring, then the in-place recurrence.  A double takes two outputs, so packets that end at 113 / 114,
311 / 312 and 623 / 624 doubles end on both sides of a tier change, and packets past 1248 doubles wrap the ring twice.

Every workload has a CPU half (no gpu mark) that proves it reaches what it is meant to reach, and a GPU half that runs
every kernel that can run it and requires the oracle's integers exactly (counters, fates, last-interaction columns, event
logs), per-packet floats to 1e-11, estimators to 1e-10 with the exact J_blue / Edotlu zero patterns, vhist to 1e-11, the
continuum estimators to 1e-10 with exact statistics, and the virtual-packet log per packet to 1e-11.
"""
from __future__ import annotations

import copy
import functools
import os
import re
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from golden_util import assert_close
from test_decision_ties import CONT_ESTIMATORS, LANE, POOLED, SCAN, VOLLEY_1, VOLLEY_32, _oracle, assert_matches_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "tardis_b200", "csrc")
N_TRACKED = 50
H100_SMEM_OPTIN = 227 * 1024  # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100 (sm_90)


# ---------------------------------------------------------------------------------------------------------------------
# Thresholds, from the constants in the source
# ---------------------------------------------------------------------------------------------------------------------
def _grab(name, pattern):
    """The groups of `pattern` in csrc/`name`; a layout change that moves them fails here, and the workloads below must
    then be moved to the new thresholds."""
    with open(os.path.join(CSRC, name)) as f:
        m = re.search(pattern, f.read())
    assert m, f"{name} no longer contains /{pattern}/: restate the threshold and move the shell-count workloads"
    return [int(g) for g in m.groups()]


@functools.lru_cache(maxsize=None)
def layout():
    k = "transport_kernel.cuh"
    (vol_items,) = _grab(k, r"constexpr int VOL_ITEMS = (\d+);")
    nd_c, nd = _grab(k, r"constexpr int trace_nd\(bool cont\) \{ return cont \? (\d+) : (\d+); \}")
    ni_c, ni = _grab(k, r"constexpr int trace_ni\(bool cont\) \{ return cont \? (\d+) : (\d+); \}")
    (pool_nd_extra,) = _grab(k, r"constexpr int pool_nd\(bool cont\) \{ return (\d+) \+ trace_nd\(cont\); \}")
    pool_ni_extra = sum(_grab(k, r"constexpr int pool_ni\(bool cont\) \{ return (\d+) \+ trace_ni\(cont\) \+ (\d+); \}"))
    (slot_list,) = _grab(k, r"constexpr int pool_bytes_per_slot\(bool cont\) \{ return pool_nd\(cont\) \* 8 \+ pool_ni\(cont\) \* 4 \+ (\d+); \}")
    vd = _grab(k, r"constexpr int vol_doubles_per_warp\(bool\) \{ return VOL_ITEMS \+ VOL_ITEMS / (\d+) \+ VOL_ITEMS / (\d+) \+ (\d+) \* (\d+) \+ (\d+); \}")
    e = "engine.cu"
    (pool_fit_kib,) = _grab(e, r"pool_bytes_per_slot\(en->continuum != 0\) <= (\d+) \* 1024;")
    (bulk_kib,) = _grab(e, r"if \(smem > (\d+) \* 1024\) return fail\(TB200_ERR_INVALID, \"too many shells")
    jump_words, scan_words = _grab(e, r"size_t smem = \(size_t\)\(en->algorithm == 1 \? (\d+) : (\d+)\) \* S \* sizeof\(double\);")
    park_default, _ = _grab(e, r"park_min = en->park_min < 1 \? \(want_pool \? (\d+) : (\d+)\)")
    slots_base, slots_add = _grab(e, r"const int pool_slots = \((\d+) \+ park_min \+ (\d+)\) & ~1;")
    trace = {c: (nd_c if c else nd) * 8 + (ni_c if c else ni) * 4 for c in (False, True)}
    slot = {c: (pool_nd_extra + (nd_c if c else nd)) * 8 + (pool_ni_extra + (ni_c if c else ni)) * 4 + slot_list for c in (False, True)}
    return dict(vol_items=vol_items, trace_bytes=trace, slot_bytes=slot,
                vol_bytes_per_warp=8 * (vol_items + vol_items // vd[0] + vol_items // vd[1] + vd[2] * vd[3] + vd[4]),
                pool_fit=pool_fit_kib * 1024, bulk_cap=bulk_kib * 1024, jump_words=jump_words, scan_words=scan_words,
                pool_slots=(slots_base + park_default + slots_add) & ~1)


def pool_limit(cont: bool, threads: int = 256) -> int:
    """Largest S at which launch_transport runs the pooled jump kernel (default park_min)."""
    t = layout()
    return (t["pool_fit"] - (threads // 32) * t["pool_slots"] * t["slot_bytes"][cont]) // (t["jump_words"] * 8)


def bulk_limit(algorithm: int) -> int:
    """Largest S whose shell table / estimator rows (4 S or 2 S doubles) the engine accepts."""
    t = layout()
    return t["bulk_cap"] // ((t["jump_words"] if algorithm == 1 else t["scan_words"]) * 8)


def volley_limit(threads: int = 256, optin: int = H100_SMEM_OPTIN) -> int:
    """Largest S whose warp-volley kernel layout (shell table, parked-lane columns, item slots) fits one CTA."""
    t = layout()
    rest = threads * t["trace_bytes"][False] + (threads // 32) * t["vol_bytes_per_warp"]
    return (optin - rest) // (t["jump_words"] * 8)


def volley_cap(S: int) -> int:
    return layout()["vol_items"] - 2 * S


CLASSIC_POOL_SHELLS = (1343, 1344, 1345)
CLASSIC_POOL_SHELLS_128 = (2431, 2432, 2433)
CONT_POOL_SHELLS = (575, 576, 577)
VP_SHELLS = (20, 100, 150, 158, 159, 160, 255, 256)
JUMP_LIMIT, SCAN_LIMIT = 6400, 12800
VP_RUNS, VP_REFUSED = 5000, 6000
TIER_ENDS = (113, 114, 311, 312, 623, 624)  # doubles; outputs 226 / 228, 622 / 624, 1246 / 1248
TIER_WRAP = 1248


def test_thresholds_sit_where_the_workloads_are():
    t = layout()
    assert t["slot_bytes"] == {False: 136, True: 184} and t["pool_slots"] == 64
    assert pool_limit(False) == CLASSIC_POOL_SHELLS[1] == 1344
    assert pool_limit(True) == CONT_POOL_SHELLS[1] == 576
    assert pool_limit(False, 128) == CLASSIC_POOL_SHELLS_128[1] == 2432
    assert pool_limit(True, 128) == 2048 and CONT_POOL_SHELLS[-1] < 2048  # the continuum tier runs of the pool at 128 threads
    assert bulk_limit(1) == JUMP_LIMIT and bulk_limit(0) == SCAN_LIMIT
    assert VP_RUNS <= volley_limit() < VP_REFUSED and volley_limit() == 5408
    assert volley_cap(150) > 1 and volley_cap(158) == 4 and volley_cap(159) == 2 and volley_cap(160) == 0
    assert 255 in VP_SHELLS and 256 in VP_SHELLS and max(volley_cap(s) for s in VP_SHELLS) >= 280
    assert [2 * d for d in TIER_ENDS] == [226, 228, 622, 624, 1246, 1248] and 2 * TIER_WRAP // 624 == 4


# ---------------------------------------------------------------------------------------------------------------------
# Running oracle and engine
# ---------------------------------------------------------------------------------------------------------------------
def whole_logs(model, packets, n_tracked=N_TRACKED, cap=None, **cfg):
    """Oracle run whose event logs of the first `n_tracked` packets are whole -> (result, log capacity)."""
    cap = cap or 2 * model.n_shells + 512
    while True:
        ref = _oracle().run_oracle(model, packets, n_tracked_packets=min(n_tracked, len(packets)), max_events_per_packet=cap,
                                   nthreads=8, **cfg)
        if (ref["event_counts"] < cap).all():
            return ref, cap
        cap *= 4


def run_engine(eng, model, packets, cap, n_tracked=N_TRACKED, vlog=0, **cfg):
    eng.set_model_from(model, **cfg)
    return eng.run_packets(packets, track_last_interaction=True, n_tracked_packets=min(n_tracked, len(packets)),
                           max_events_per_packet=cap, vlog_capacity=vlog)


def vlog_rows(res):
    """The virtual-packet log in (packet, nu, mu) order: the kernels append volleys as they finish."""
    m = res["vlog_count"]
    cols = {k: res[k][:m] for k in ("vlog_packet_index", "vlog_nus", "vlog_energies", "vlog_initial_mus", "vlog_initial_rs")}
    order = np.lexsort((cols["vlog_initial_mus"], cols["vlog_nus"], cols["vlog_packet_index"]))
    return {k: v[order] for k, v in cols.items()}


def assert_vlog_matches(res, ref, what):
    assert res["vlog_count"] == ref["vlog_count"], (what, res["vlog_count"], ref["vlog_count"])
    a, b = vlog_rows(res), vlog_rows(ref)
    assert np.array_equal(a["vlog_packet_index"], b["vlog_packet_index"]), what
    for k in ("vlog_nus", "vlog_energies", "vlog_initial_mus", "vlog_initial_rs"):
        assert_close(a[k], b[k], 1e-11, f"{what}: {k}")


def check_cases(options, cases):
    """Run every case (name, model, packets, engine config, oracle result, log capacity, vlog capacity) on one engine."""
    from tardis_b200.engine import Engine

    eng = Engine(0)
    try:
        for k, v in options.items():
            eng.set_option(k, v)
        for name, model, packets, cfg, ref, cap, vlog in cases:
            res = run_engine(eng, model, packets, cap, n_tracked=len(ref["event_counts"]), vlog=vlog, **cfg)
            assert_matches_oracle(res, ref, name)
            if vlog:
                assert_vlog_matches(res, ref, name)
    finally:
        eng.close()


def thin_model(S, mode, seed, n_lines=400, continuum=False, n_e_scale=1.0, mu_tau=-7.5):
    """S thin shells of the synthetic model: a trace rarely ends before its boundary, so every packet draws about one
    double per boundary it crosses."""
    from tardis_b200 import synthetic as syn

    m = syn.make_model(S, n_lines, mode, mu_tau=mu_tau, seed=seed, n_bins=2000)
    if continuum:
        syn.add_continuum(m, seed=seed + 1, n_continua=12, points=(4, 9))
    m.electron_density = m.electron_density * n_e_scale
    return m


def packets_for(model, n, seed):
    from tardis_b200 import synthetic as syn

    return syn.make_packets(n, model.r_inner[0], base_seed=seed)


# ---------------------------------------------------------------------------------------------------------------------
# Workload 1: both sides of the pool fallback, classic and continuum mode
# ---------------------------------------------------------------------------------------------------------------------
POOL_GROUPS = {
    "classic_256": (CLASSIC_POOL_SHELLS, ("macroatom", "scatter"), False, 256),
    "classic_128": (CLASSIC_POOL_SHELLS_128, ("macroatom", "scatter"), False, 128),
    "continuum_256": (CONT_POOL_SHELLS, ("macroatom",), True, 256),
}


@functools.lru_cache(maxsize=None)
def pool_cases(group):
    shells, modes, cont, _ = POOL_GROUPS[group]
    out = []
    for mode in modes:
        for S in shells:
            m = thin_model(S, mode, seed=S, n_lines=300 if S < 2000 else 150, continuum=cont)
            p = packets_for(m, 3000, seed=S + 7)
            ref, cap = whole_logs(m, p)
            out.append((f"{group} {mode} S={S}", m, p, {}, ref, cap, 0))
    return out


def test_pool_workloads_cross_every_shell():
    """The packets of the pool-threshold workloads cross about as many boundaries as there are shells, so every shell
    table entry and, in the pooled kernel, a full pool's worth of parked packets is used."""
    for group in POOL_GROUPS:
        for name, m, p, _, ref, _, _ in pool_cases(group):
            draws = ref["counters"]["n_rng_draws"] / len(p)
            assert draws > 0.8 * m.n_shells, (name, draws)
            assert ref["counters"]["n_boundary_events"] > 0.8 * m.n_shells * len(p), name


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", [SCAN, POOLED, LANE], ids=["scan", "pooled", "lane"])
@pytest.mark.parametrize("group", list(POOL_GROUPS))
def test_pool_threshold_matches_the_oracle(group, kernel):
    check_cases({**kernel, "threads_per_cta": POOL_GROUPS[group][3]}, pool_cases(group))


# ---------------------------------------------------------------------------------------------------------------------
# Workload 2: virtual packets around the volley's sub-batch cap and meta limit, with Russian roulette inside the volleys
# ---------------------------------------------------------------------------------------------------------------------
VP_CFG = dict(number_of_vpackets=2, survival_probability=0.5)


def vp_model(S):
    return thin_model(S, "macroatom", seed=1000 + S, n_lines=300, n_e_scale=8.0, mu_tau=-5.0)


@functools.lru_cache(maxsize=None)
def vp_cases(full_rel):
    out = []
    for S in VP_SHELLS:
        m = vp_model(S)
        p = packets_for(m, 1000, seed=2000 + S)
        cfg = dict(VP_CFG, enable_full_relativity=full_rel)
        vlog = 4_000_000
        ref, cap = whole_logs(m, p, vlog_capacity=vlog, **cfg)
        assert ref["vlog_count"] < vlog
        out.append((f"vpackets fr={full_rel} S={S}", m, p, cfg, ref, cap, vlog))
    return out


@pytest.mark.parametrize("full_rel", [False, True], ids=["partial_rel", "full_rel"])
def test_vpacket_workloads_play_roulette(full_rel):
    """In every vpacket workload virtual packets reach tau_russian inside the volleys: at least 50 more of them leave no
    energy than in the same run with survival probability 1, where the roulette kills none."""
    for name, m, p, cfg, ref, _, vlog in vp_cases(full_rel):
        sure = _oracle().run_oracle(m, p, nthreads=8, track_last_interaction=False, vlog_capacity=vlog,
                                    **dict(cfg, survival_probability=1.0))
        died = (ref["vlog_energies"][:ref["vlog_count"]] == 0).sum() - (sure["vlog_energies"][:sure["vlog_count"]] == 0).sum()
        assert died >= 50, (name, died)
        assert ref["counters"]["n_vpackets"] >= 2 * len(p), name


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", [VOLLEY_1, VOLLEY_32, SCAN], ids=["volley_min1", "volley_min32", "scan"])
@pytest.mark.parametrize("full_rel", [False, True], ids=["partial_rel", "full_rel"])
def test_vpacket_shell_counts_match_the_oracle(full_rel, kernel):
    check_cases(kernel, vp_cases(full_rel))


# ---------------------------------------------------------------------------------------------------------------------
# Workload 3: the host-side shell limits, each on both sides; after a refusal the same engine runs a small model
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def limit_case(S, mode, n, vpackets=False):
    m = thin_model(S, mode, seed=S, n_lines=60, n_e_scale=0.5)
    p = packets_for(m, n, seed=S + 3)
    cfg = dict(number_of_vpackets=2) if vpackets else {}
    ref, cap = whole_logs(m, p, n_tracked=20, **cfg)
    return (f"{mode} S={S} vp={vpackets}", m, p, cfg, ref, cap, 0)


@functools.lru_cache(maxsize=None)
def small_case():
    m = thin_model(12, "macroatom", seed=12, n_lines=2000, mu_tau=-4.0)
    p = packets_for(m, 4000, seed=13)
    ref, cap = whole_logs(m, p)
    return ("small model after a refusal", m, p, {}, ref, cap, 0)


def assert_refused_then_usable(eng, S, mode, cfg):
    from tardis_b200.engine import EngineError

    m = thin_model(S, mode, seed=S, n_lines=60)
    eng.set_model_from(m, **cfg)
    with pytest.raises(EngineError, match="too many shells"):
        eng.run_packets(packets_for(m, 64, seed=S))
    name, m, p, cfg, ref, cap, _ = small_case()
    assert_matches_oracle(run_engine(eng, m, p, cap, **cfg), ref, f"{name} (S={S} refused)")


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", [POOLED, LANE], ids=["pooled", "lane"])
def test_jump_shell_limit(kernel):
    """S = 6400 runs (the pools do not fit: the lane-resident kernel) and matches the oracle; 6401 is refused."""
    from tardis_b200.engine import Engine

    eng = Engine(0)
    try:
        for k, v in kernel.items():
            eng.set_option(k, v)
        name, m, p, cfg, ref, cap, _ = limit_case(JUMP_LIMIT, "macroatom", 1000)
        assert_matches_oracle(run_engine(eng, m, p, cap, n_tracked=20, **cfg), ref, name)
        assert_refused_then_usable(eng, JUMP_LIMIT + 1, "macroatom", {})
    finally:
        eng.close()


@pytest.mark.gpu
def test_scan_shell_limit():
    """The scan kernel keeps 2 S doubles per CTA: S = 12800 runs and matches the oracle, 12801 is refused; S = 6401,
    refused by the jump kernels, runs."""
    from tardis_b200.engine import Engine

    eng = Engine(0)
    try:
        eng.set_option("algorithm", 0)
        for S in (JUMP_LIMIT + 1, SCAN_LIMIT):
            name, m, p, cfg, ref, cap, _ = limit_case(S, "scatter", 400)
            assert_matches_oracle(run_engine(eng, m, p, cap, n_tracked=20, **cfg), ref, name)
        assert_refused_then_usable(eng, SCAN_LIMIT + 1, "scatter", {})
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", [VOLLEY_1, VOLLEY_32], ids=["volley_min1", "volley_min32"])
def test_vpacket_shell_limit(kernel):
    """The warp volleys' item slots come on top of the shell table: 5000 shells run and match the oracle, 6000 (within
    the 200 KiB of shell table) do not fit the CTA and are refused on the host."""
    from tardis_b200.engine import Engine

    eng = Engine(0)
    try:
        for k, v in kernel.items():
            eng.set_option(k, v)
        name, m, p, cfg, ref, cap, _ = limit_case(VP_RUNS, "macroatom", 400, vpackets=True)
        assert_matches_oracle(run_engine(eng, m, p, cap, n_tracked=20, **cfg), ref, name)
        assert VP_REFUSED <= bulk_limit(1)
        assert_refused_then_usable(eng, VP_REFUSED, "macroatom", dict(number_of_vpackets=2))
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# Workload 4: every generator tier.  Thick models: packets drawn from a pool of candidates for the many that wrap the
# ring (> 1248 doubles), plus random ones.  Thin models of T shells with thin opacities: almost every packet crosses the T
# shells without an interaction and ends at exactly T doubles, one for each trace.
# ---------------------------------------------------------------------------------------------------------------------
TIER_MODES = ("continuum", "scatter", "downbranch", "macroatom")
TIER_N = 2500
TIER_POOL = 20000


def draw_counts(model, packets, **cfg):
    """Doubles each packet draws in the oracle, one packet per call (the calls run in threads: the oracle keeps no state
    between runs and ctypes releases the GIL)."""
    def one(i):
        return _oracle().run_oracle(model, packets.slice(i, i + 1), track_last_interaction=False,
                                    **cfg)["counters"]["n_rng_draws"]

    with ThreadPoolExecutor(8) as ex:
        return np.fromiter(ex.map(one, range(len(packets))), dtype=np.int64, count=len(packets))


def thick_model(mode):
    from tardis_b200 import synthetic as syn

    if mode == "continuum":
        m = syn.make_model(6, 2000, "macroatom", mu_tau=-4.0, seed=5151)
        syn.add_continuum(m, seed=5152, n_continua=12, points=(4, 9))
        m.electron_density = m.electron_density * 100.0
    else:
        m = syn.make_model(4, 3000, mode, mu_tau=-2.0, seed=31)
        m.electron_density = m.electron_density * 100.0
    return m


def tier_cfgs(mode):
    return [dict(enable_full_relativity=False)] if mode == "continuum" else [dict(enable_full_relativity=fr) for fr in (False, True)]


@functools.lru_cache(maxsize=None)
def thick_selection(mode, full_rel):
    """-> (model, selected packets, their draw counts): every candidate past TIER_WRAP doubles (at most 1500) and every
    one ending at a tier edge, filled with random ones to TIER_N."""
    m = thick_model(mode)
    cand = packets_for(m, TIER_POOL, seed=6000 + len(mode))
    cfg = dict(enable_full_relativity=full_rel)
    c = draw_counts(m, cand, **cfg)
    rng = np.random.default_rng(61)
    keep = np.flatnonzero(c > TIER_WRAP)[:1500]
    keep = np.union1d(keep, np.flatnonzero(np.isin(c, TIER_ENDS)))
    rest = np.setdiff1d(np.arange(TIER_POOL), keep)
    keep = np.union1d(keep, rng.choice(rest, TIER_N - len(keep), replace=False))
    rng.shuffle(keep)
    return m, take(cand, keep), c[keep]


def take(packets, idx):
    from tardis_b200 import synthetic as syn

    return syn.Packets(packets.initial_radii[idx], packets.initial_nus[idx], packets.initial_mus[idx],
                       packets.initial_energies[idx], packets.packet_seeds[idx], packets.radiation_field_luminosity)


@functools.lru_cache(maxsize=None)
def tier_end_selection(mode, full_rel, T):
    """-> (model of T thin shells, 64 packets that draw exactly T doubles)."""
    m = thin_model(T, "macroatom" if mode == "continuum" else mode, seed=7000 + T, n_lines=200,
                   continuum=mode == "continuum", n_e_scale=1e-3)
    if mode == "continuum":
        cont = copy.copy(m.continuum)
        cont.chi_bf = cont.chi_bf * 1e-6
        cont.ff_opacity_factor = cont.ff_opacity_factor * 1e-6
        m.continuum = cont
    cand = packets_for(m, 256, seed=7100 + T)
    c = draw_counts(m, cand, enable_full_relativity=full_rel)
    idx = np.flatnonzero(c == T)[:64]
    return m, take(cand, idx), c[idx]


@pytest.mark.parametrize("mode", TIER_MODES)
def test_tier_workloads_reach_every_tier(mode):
    """Per run of the mode: >= 500 packets past 1248 doubles and >= 32 ending at each tier edge; per workload the draws
    the oracle reports for the selected packets together equal the sum of the one-packet counts."""
    for cfg in tier_cfgs(mode):
        fr = cfg["enable_full_relativity"]
        m, p, c = thick_selection(mode, fr)
        assert len(p) == TIER_N and (c > TIER_WRAP).sum() >= 500, (mode, fr, (c > TIER_WRAP).sum())
        ends = {T: int((c == T).sum()) for T in TIER_ENDS}
        for T in TIER_ENDS:
            tm, tp, tc = tier_end_selection(mode, fr, T)
            ends[T] += len(tp)
            assert (tc == T).all()
        assert min(ends.values()) >= 32, (mode, fr, ends)
        tot = _oracle().run_oracle(m, p, nthreads=8, track_last_interaction=False, **cfg)["counters"]["n_rng_draws"]
        assert tot == c.sum(), (mode, fr)


@functools.lru_cache(maxsize=None)
def tier_cases(mode):
    out = []
    for cfg in tier_cfgs(mode):
        fr = cfg["enable_full_relativity"]
        m, p, _ = thick_selection(mode, fr)
        ref, cap = whole_logs(m, p, cap=8192, **cfg)
        out.append((f"{mode} fr={fr} thick", m, p, cfg, ref, cap, 0))
        for T in TIER_ENDS:
            tm, tp, _ = tier_end_selection(mode, fr, T)
            ref, cap = whole_logs(tm, tp, **cfg)
            out.append((f"{mode} fr={fr} ends at {T}", tm, tp, cfg, ref, cap, 0))
    return out


TIER_KERNELS = {
    "continuum": [("pooled_128", {**POOLED, "threads_per_cta": 128}), ("lane", LANE), ("scan", SCAN)],
    "classic": [("pooled", POOLED), ("lane", LANE), ("scan", SCAN)],
}


@pytest.mark.gpu
@pytest.mark.parametrize("mode,kernel", [(m, k) for m in TIER_MODES for k in TIER_KERNELS["continuum" if m == "continuum" else "classic"]],
                         ids=lambda v: v if isinstance(v, str) else v[0])
def test_generator_tiers_match_the_oracle(mode, kernel):
    check_cases(kernel[1], tier_cases(mode))


@pytest.mark.gpu
def test_generator_tiers_in_the_default_continuum_pool():
    """The continuum pool at its default 256 threads per CTA on the thick workload (the exact-end runs of 623 / 624
    shells are above its pool limit there)."""
    check_cases(POOLED, tier_cases("continuum")[:1])


# ---------------------------------------------------------------------------------------------------------------------
# Workload 5: scheduling.  How often the pooled and lane kernels park, swap and refill must not change a trajectory.
# ---------------------------------------------------------------------------------------------------------------------
SCHEDULES = [(1, 1, 1, 128), (32, 32, 2, 128), (7, 3, 4, 256), (16, 8, 3, 256), (2, 32, 2, 256)]


@functools.lru_cache(maxsize=None)
def continuum_schedule_case():
    m = thick_model("continuum")
    p = packets_for(m, 20000, seed=8101)
    ref, cap = whole_logs(m, p, n_tracked=100, cap=8192)
    assert ref["counters"]["n_rng_draws"] / len(p) > 100
    return ("thick continuum", m, p, {}, ref, cap, 0)


@pytest.mark.gpu
@pytest.mark.parametrize("park_min,refill_min,ctas,threads", SCHEDULES)
@pytest.mark.parametrize("pooled", [1, 0], ids=["pooled", "lane"])
def test_continuum_scheduling_is_invisible(pooled, park_min, refill_min, ctas, threads):
    check_cases({"algorithm": 1, "pooled": pooled, "park_min": park_min, "refill_min": refill_min, "ctas_per_sm": ctas,
                 "threads_per_cta": threads}, [continuum_schedule_case()])


@functools.lru_cache(maxsize=None)
def classic_schedule_case(vpackets):
    from tardis_b200 import synthetic as syn

    if vpackets:
        m = syn.make_model(12, 6000, "macroatom", mu_tau=-3.5, seed=71)
        p = packets_for(m, 6000, seed=72)
        cfg = dict(number_of_vpackets=5, vpacket_spawn_start_frequency=2e14, vpacket_spawn_end_frequency=3e15)
        ref, cap = whole_logs(m, p, spawn_start=2e14, spawn_end=3e15, number_of_vpackets=5, vlog_capacity=2_000_000)
        return ("classic vpackets", m, p, cfg, ref, cap, 2_000_000)
    m = thick_model("macroatom")
    p = packets_for(m, 20000, seed=8202)
    ref, cap = whole_logs(m, p, n_tracked=100, cap=8192)
    return ("thick classic", m, p, {}, ref, cap, 0)


@pytest.mark.gpu
@pytest.mark.parametrize("ctas", [1, 4])
@pytest.mark.parametrize("kernel,vpackets", [(LANE, False), (VOLLEY_1, True)], ids=["lane", "volley"])
def test_classic_lane_and_volley_at_128_threads(kernel, vpackets, ctas):
    check_cases({**kernel, "threads_per_cta": 128, "ctas_per_sm": ctas}, [classic_schedule_case(vpackets)])


# ---------------------------------------------------------------------------------------------------------------------
# Workload 6: processing order and the pipelined run; each against a default-option run of the same engine
# ---------------------------------------------------------------------------------------------------------------------
def assert_same_run(a, b, what, cont=False, fixed_point=True):
    """Per-packet outputs and counters identical; J_blue / Edotlu identical where the jump kernels sum them in fixed point
    (the scan kernel adds them in f64 atomics, whose last bits follow the order: there 1e-12 and the same zero pattern)."""
    lines = ("j_blue", "edotlu")
    for k in ("output_nus", "output_energies") + (lines if fixed_point else ()) + (
            ("last_interaction_type", "last_line_absorb_id") if "last_interaction_type" in a else ()):
        assert np.array_equal(a[k], b[k]), (what, k)
    if not fixed_point:
        for k in lines:
            assert np.array_equal(a[k] == 0, b[k] == 0), (what, k + " zero pattern")
            assert_close(a[k], b[k], 1e-12, f"{what}: {k}")
    assert all(a["counters"][k] == v for k, v in b["counters"].items() if k != "n_search_probes"), what
    for k in ("j", "nu_bar") + (CONT_ESTIMATORS if cont else ()):
        assert_close(a[k], b[k], 1e-12, f"{what}: {k}")
    if cont:
        assert np.array_equal(a["photo_ion_estimator_statistics"], b["photo_ion_estimator_statistics"]), what


def wide_packets(model, n, seed):
    """Packets whose frequencies run from 1/30 of the lowest line to 30 times the highest: the order keys of many are
    clamped to the first or the last key."""
    from tardis_b200 import synthetic as syn

    p = packets_for(model, n, seed)
    rng = np.random.default_rng(seed)
    lo, hi = model.line_list_nu[-1] / 30.0, model.line_list_nu[0] * 30.0
    nus = np.exp(rng.uniform(np.log(lo), np.log(hi), n))
    return syn.Packets(p.initial_radii, nus, p.initial_mus, p.initial_energies, p.packet_seeds, p.radiation_field_luminosity)


def test_wide_packets_lie_beyond_both_ends_of_the_line_list():
    from tardis_b200 import synthetic as syn

    m = syn.make_model(20, 20000, "macroatom", mu_tau=-4.0, seed=91)
    p = wide_packets(m, 50000, 92)
    assert (p.initial_nus > m.line_list_nu[0]).sum() > 5000 and (p.initial_nus < m.line_list_nu[-1]).sum() > 5000


@pytest.mark.gpu
@pytest.mark.parametrize("options", [{"sort_packets": 0}, {"sort_bits": 0}, {"sort_bits": 16}],
                         ids=["unsorted", "sort_bits_0", "sort_bits_16"])
@pytest.mark.parametrize("kernel", [POOLED, LANE, SCAN], ids=["pooled", "lane", "scan"])
def test_processing_order_is_invisible(kernel, options):
    """sort_bits = 16 gives one order key per line-list bucket (far more than 2048: the ordering kernels' global-atomic
    branch); the wide packets clamp their keys at both ends of the list."""
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import Engine

    m = syn.make_model(20, 20000, "macroatom", mu_tau=-4.0, seed=91)
    runs = {}
    for name, p in (("bench-like", packets_for(m, 50000, 93)), ("wide", wide_packets(m, 50000, 92))):
        for which, opts in (("default", {}), ("option", options)):
            eng = Engine(0)
            try:
                for k, v in {**kernel, **opts}.items():
                    eng.set_option(k, v)
                eng.set_model_from(m)
                runs[which] = eng.run_packets(p, track_last_interaction=True)
            finally:
                eng.close()
        assert_same_run(runs["option"], runs["default"], f"{name} {options}", fixed_point=kernel["algorithm"] == 1)


@pytest.mark.gpu
@pytest.mark.parametrize("pooled", [1, 0], ids=["pooled", "lane"])
def test_pipelined_continuum_run_matches_resident(pooled):
    """tb200_run splits >= 4e6 packets into ranges whose copies and kernels overlap; in continuum mode too the result equals
    the single-launch device-resident run."""
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import Engine

    m = syn.make_model(8, 2500, "macroatom", mu_tau=-4.0, seed=131)
    syn.add_continuum(m, seed=9131, adiabatic_fraction=0.3)
    p = packets_for(m, 4_200_000, 132)
    eng = Engine(0)
    try:
        eng.set_option("pooled", pooled)
        eng.set_model_from(m)
        piped = eng.run_packets(p)
        eng.upload_packets(p.initial_radii, p.initial_nus, p.initial_mus, p.initial_energies, p.packet_seeds)
        eng.transport(True)
        eng.sync()
        resident = eng.download()
    finally:
        eng.close()
    assert_same_run(piped, resident, "pipelined continuum", cont=True)
