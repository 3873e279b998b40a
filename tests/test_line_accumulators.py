"""The jump kernels' fixed-point line estimators against exact integer and rational arithmetic.

With the jump algorithm J_blue and Edotlu are not floating-point sums.  Every trace adds +w at its first line and -w
behind its last to 64-bit integer words (fixed_term / fixed_add in transport_kernel.cuh: w * scale split at 2^29 into a
high and a low word), and finalize_line_estimators_kernel turns the words into the two tables with 128-bit prefix sums.
This file checks that path on its own, with Python `int` and `fractions.Fraction` as the reference:

  A. a model of the words and of the epilogue in Python, tested on the CPU against the constants in the source;
  B. finalize_line_estimators_kernel on crafted words: every cell of both tables against the model (tile loop and carry,
     mixed-sign recombination, the inclusive read of cell n_lines, pad cells, the int128 -> double conversion), and what
     it must refuse: a row that does not sum to zero, and a wrap that the closing cell mirrors (a negative prefix), by
     one engine and after the word sum of an engine group;
  C. the transport kernels on packets that never interact.  A packet's frequency and energy are taken to the lab frame
     once, where it enters the grid, and then never change: the run returns them as output_nus / output_energies.  With
     these E_p and nu_p, Edotlu[s][i] = nu_i sum E_p / nu_p and J_blue[s][i] = nu_i sum E_p / nu_p^2 over the packets
     whose trace in shell s covers line i (full relativity: sum E_p and sum E_p / nu_p).  WHICH cells a packet covers is
     the C oracle's decision (run on that packet alone); the VALUE is a Fraction of those doubles.  Packet sets: equal energies,
     energies 2^-30 .. 2^30 apart, one packet of ~2^32 typical terms (just inside the range of a word), a line list
     spanning a factor 1e4 in frequency; and the packet of 2^35 typical terms that fixed_term must refuse.

That a launch stopped by a macro-atom error still reports the macro-atom error (the ranges its packets left open make
the row totals meaningless, and must not mask it) is asserted by test_phase_b_search.py::test_block_total_below_one_raises:
six shells, both jump kernels, the exception type.
"""
from __future__ import annotations

import functools
import math
import os
import re
from fractions import Fraction

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNELS = os.path.join(ROOT, "tardis_b200", "csrc", "transport_kernel.cuh")

POOLED = {"algorithm": 1, "pooled": 1}
LANE = {"algorithm": 1, "pooled": 0}
SCAN = {"algorithm": 0}


# ---------------------------------------------------------------------------------------------------------------------
# A. The word model
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def constants():
    """FIXED_SPLIT, FIXED_TYPICAL_LOG2 and the refusal limit of fixed_term, read from the source."""
    with open(KERNELS) as f:
        src = f.read()
    out = {}
    for key, pattern, conv in (("split", r"constexpr double FIXED_SPLIT = ([0-9.]+);", float),
                               ("typical_log2", r"constexpr int FIXED_TYPICAL_LOG2 = (\d+);", int),
                               ("limit", r"!\(th < ([0-9.e+]+)\) \|\| !\(t >= 0\.0\)", float),
                               ("recombine", r"\(__int128\)hi \* \(__int128\)(\d+)ll \+ \(__int128\)lo", int)):
        m = re.search(pattern, src)
        assert m, f"transport_kernel.cuh no longer contains /{pattern}/: restate the word model of this file"
        out[key] = conv(m.group(1))
    out["headroom_comment"] = re.search(
        r"low word holds 2\^(\d+) same-sign terms, its high word 2\^(\d+) typical ones \(2\^(\d+) of the heaviest that equal\s*"
        r"// energies and a line list spanning a factor (\d+) in frequency", src)
    return out


class FixedPointRange(ValueError):
    """Where fixed_term raises ERR_FIXED_POINT and adds nothing."""


def fixed_words(w: float, scale: float) -> tuple[int, int]:
    """(hi, lo) of fixed_term: t = w * scale as the double the kernel forms, hi = floor(t / 2^29) (__double2ll_rd),
    lo = rint(t - hi * 2^29) (__double2ll_rn; the difference is exact).  Raises where the kernel refuses."""
    c = constants()
    t = w * scale
    th = t * (1.0 / c["split"])
    if not th < c["limit"] or not t >= 0.0:
        raise FixedPointRange(f"w * scale = {t!r}")
    hi = math.floor(th)
    lo = round(t - float(hi) * c["split"])  # round() of a float is round-half-even, as cvt.rni
    return hi, lo


def signed64(v: int) -> int:
    """The signed reading of a 64-bit word that holds v mod 2^64."""
    return (v + 2**63) % 2**64 - 2**63


def row_prefixes(words, n_lines: int):
    """words [S][>= n_lines + 1][4] (any integers; read mod 2^64, signed) -> prefix [S][2][n_lines] of hi * 2^29 + lo as
    Python ints (quantity 0: the w1 words, 1: the w2 words) and the row totals [S][2], which include cell n_lines."""
    split = int(constants()["split"])
    prefixes, totals = [], []
    for shell in words:
        p_shell, t_shell = [], []
        for q in (0, 1):
            run, pre = 0, []
            for i in range(n_lines + 1):
                run += signed64(int(shell[i][2 * q])) * split + signed64(int(shell[i][2 * q + 1]))
                if i < n_lines:
                    pre.append(run)
            p_shell.append(pre)
            t_shell.append(run)
        prefixes.append(p_shell)
        totals.append(t_shell)
    return prefixes, totals


def finalize_rows(words, nu_line, scales, full_rel: bool):
    """finalize_line_estimators_kernel in exact arithmetic.  scales = (scale_j_blue, scale_edotlu), the order of
    Engine.line_accumulators: the w1 words (columns 0, 1) are Edotlu at scale_edotlu, the w2 words (columns 2, 3) J_blue at
    scale_j_blue.  -> (edotlu [S][L], j_blue [S][L]) as Fractions, row totals [S][2] (w1, w2) as ints."""
    n_lines = len(nu_line)
    prefixes, totals = row_prefixes(words, n_lines)
    scale_j_blue, scale_edotlu = (Fraction(s) for s in scales)
    nu = [Fraction(1) if full_rel else Fraction(float(x)) for x in nu_line]
    edotlu = [[Fraction(p) / scale_edotlu * nu[i] for i, p in enumerate(row[0])] for row in prefixes]
    j_blue = [[Fraction(p) / scale_j_blue * nu[i] for i, p in enumerate(row[1])] for row in prefixes]
    return edotlu, j_blue, totals


def typical_energy(energies) -> float:
    """The engine's typical packet energy: the mean |E| over a strided sample of at most 65536 packets, summed in order."""
    n = len(energies)
    m = min(n, 65536)
    acc = 0.0
    for e in np.abs(np.asarray(energies, dtype=np.float64)[:: n // m][:m]).tolist():
        acc += e
    return acc / m


def model_scales(line_list_nu, e_typ: float, full_rel: bool) -> tuple[float, float]:
    """(scale_j_blue, scale_edotlu) as the engine derives them: the typical term, e_typ / nu_typ (full relativity: e_typ)
    for Edotlu and that over nu_typ for J_blue, nu_typ = sqrt(nu_first nu_last), lands in [2^58, 2^59)."""
    nu_typ = math.sqrt(abs(float(line_list_nu[0]) * float(line_list_nu[-1])))
    w1 = e_typ if full_rel else e_typ / nu_typ
    w2 = w1 / nu_typ
    k = constants()["typical_log2"]
    return math.ldexp(1.0, k - (math.frexp(w2)[1] - 1)), math.ldexp(1.0, k - (math.frexp(w1)[1] - 1))


def symmetric_wrap_row(n_cells: int, first: int, behind_last: int, k: int = 3):
    """Words [1][n_cells][4] of a w1 row whose true high-word sum at `first` is 2^63 + k and at `behind_last`
    -(2^63 + k): the 64-bit words read -2^63 + k and 2^63 - k."""
    row = [[0, 0, 0, 0] for _ in range(n_cells)]
    row[first][0] = signed64(2**63 + k)
    row[behind_last][0] = signed64(-(2**63) - k)
    return [row]


def test_words_recombine_to_the_rounded_term():
    """hi * 2^29 + lo == rint(t) for t across 2^0 .. 2^90.7 and next to multiples of 2^29, with 0 <= lo <= 2^29."""
    c = constants()
    assert c["split"] == 2.0**29 and c["recombine"] == 2**29
    rng = np.random.default_rng(8101)
    top = math.log2(c["limit"] * c["split"])
    ts = list(np.exp2(rng.uniform(0.0, top - 1e-9, 4000)))
    for m in (1, 2, 3, 12345, 2**20 + 1, 2**33 - 1):
        base = m * c["split"]
        for d in (-1.0, -0.75, -0.5, -0.25, 0.0, 0.25, 0.5, 0.75, 1.0):
            ts.append(base + d)
        ts += [math.nextafter(base, 0.0), math.nextafter(base, math.inf)]
    ts += [0.0, 0.5, 1.5, 2.5, 2.0**29 - 0.5, 2.0**53 + 2.0, 2.0**82, 2.0**82 * 1.5]
    for t in ts:
        hi, lo = fixed_words(float(t), 1.0)
        want = int(Fraction(float(t)).__round__())  # Fraction rounds half to even, exactly
        assert hi * 2**29 + lo == want, (t, hi, lo)
        assert 0 <= lo <= 2**29 and 0 <= hi < 2**63, (t, hi, lo)
    # a scale moves the binary point and nothing else
    assert fixed_words(3.0 * 2.0**-70, 2.0**100) == fixed_words(3.0 * 2.0**30, 1.0) == (6, 0)


def test_refusal_threshold_sits_where_the_constants_say():
    c = constants()
    limit, split, k = c["limit"], c["split"], c["typical_log2"]
    assert limit == 4.0e18 and k == 58
    assert limit < 2.0**63, "an accepted high word must fit a signed 64-bit word"
    inside = math.nextafter(limit, 0.0) * split
    assert fixed_words(inside, 1.0) == (int(math.nextafter(limit, 0.0)), 0)
    for bad in (limit * split, limit * split * 2, math.inf, math.nan, -1.0, -math.ldexp(1.0, -1074)):
        with pytest.raises(FixedPointRange):
            fixed_words(bad, 1.0)
    # the typical term lands in [2^58, 2^59): every term up to 2^31 typical ones is accepted whatever the mantissas,
    # 2^32 only below 4e18 / 2^61 = 1.73 of its binade, and 2^33 never
    scale = math.ldexp(1.0, k)
    assert fixed_words(math.nextafter(2.0, 0.0) * 2.0**31, scale)[0] < limit
    assert fixed_words(1.7 * 2.0**32, scale)[0] < limit
    for w in (1.75 * 2.0**32, 2.0**33, 2.0**35):
        with pytest.raises(FixedPointRange):
            fixed_words(w, scale)


def test_headroom_stated_beside_fixed_term_follows_from_the_constants():
    """The comment above fixed_term: same-sign terms a low word holds, typical terms a high word holds, and terms of the
    heaviest kind that equal energies and a line list spanning the stated factor in frequency produce (a packet at the
    red end has w2 = (nu_typ / nu_last)^2 = that factor of typical ones)."""
    c = constants()
    m = c["headroom_comment"]
    assert m, "the headroom comment above fixed_term changed: restate this test"
    low, high_typical, high_heaviest, factor = (int(g) for g in m.groups())
    split_log2 = int(math.log2(c["split"]))
    assert low == 63 - split_log2                                        # lo < 2^29 per term
    typical_hi_log2 = c["typical_log2"] + 1 - split_log2                 # t < 2^59  ->  hi < 2^30
    assert high_typical == 63 - typical_hi_log2
    assert high_heaviest == math.floor(63 - typical_hi_log2 - math.log2(factor))


def test_finalize_rows_on_a_hand_made_row():
    nu = [4.0, 2.0, 1.0]
    words = [[[1, -3, 0, 5], [0, 0, 2, 0], [-1, 1, 0, -5], [0, 2, -2, 0], [9, 9, 9, 9]]]  # the cell behind n_lines + 1 is not read
    edotlu, j_blue, totals = finalize_rows(words, nu, (8.0, 2.0), False)
    s = 2**29
    assert totals == [[0, 0]]
    assert edotlu == [[Fraction(s - 3, 2) * 4, Fraction(s - 3, 2) * 2, Fraction(-2, 2) * 1]]
    assert j_blue == [[Fraction(5, 8) * 4, Fraction(2 * s + 5, 8) * 2, Fraction(2 * s, 8) * 1]]
    edotlu_fr, _, _ = finalize_rows(words, nu, (8.0, 2.0), True)
    assert edotlu_fr == [[Fraction(s - 3, 2), Fraction(s - 3, 2), Fraction(-1)]]
    assert finalize_rows([[[2**64 - 1, 0, 0, 0], [1, 0, 0, 0]]], [1.0], (1.0, 1.0), True)[0] == [[Fraction(-s)]]  # mod 2^64, signed


def test_symmetric_wrap_sums_to_zero_and_shows_as_a_negative_prefix():
    """A wrap that the closing cell mirrors passes the row-total check; every cell between the two is 2^64 * 2^29 / scale
    too low, hence negative, which a sum of non-negative weights never is."""
    words = symmetric_wrap_row(12, 2, 9, k=3)
    prefixes, totals = row_prefixes(words, 11)
    assert totals == [[0, 0]]
    assert prefixes[0][0][:2] == [0, 0] and prefixes[0][0][9:] == [0, 0]
    assert all(p == (3 - 2**63) * 2**29 for p in prefixes[0][0][2:9])
    assert all(p - (3 + 2**63) * 2**29 == -(2**64) * 2**29 for p in prefixes[0][0][2:9])


# ---------------------------------------------------------------------------------------------------------------------
# Shared pieces of the GPU tests
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def engine():
    from tardis_b200.engine import Engine

    eng = Engine(0)
    yield eng
    eng.close()


def configure(eng, options):
    for k, v in {"algorithm": 1, "pooled": 1, **options}.items():
        eng.set_option(k, v)


def device_words(eng):
    """(int64 CUDA tensor [S][line_pitch + 1][4] aliasing the accumulators, (scale_j_blue, scale_edotlu))"""
    from tardis_b200.parallel import line_accumulator_tensor

    words, scales = line_accumulator_tensor(eng)
    lay = eng.estimator_layout()
    return words.view(lay["n_shells"], lay["line_pitch"] + 1, 4), scales


def write_words(eng, cells):
    """Replace the accumulators by `cells` [S][n][4] (Python ints that fit a signed word; further cells zero)."""
    import torch

    eng.sync()
    words, _ = device_words(eng)
    host = np.zeros(tuple(words.shape), dtype=np.int64)
    for s, row in enumerate(cells):
        host[s, : len(row)] = np.array(row, dtype=np.int64)
    words.copy_(torch.from_numpy(host).to(words.device))
    torch.cuda.synchronize()


def device_tables(eng):
    """(edotlu, j_blue) [S][line_pitch] as they lie in the estimator buffer, pad cells included."""
    from tardis_b200.parallel import estimator_tensor

    lay = eng.estimator_layout()
    S, pitch = lay["n_shells"], lay["line_pitch"]
    est = estimator_tensor(eng)
    jb = est[lay["off_j_blue"]: lay["off_j_blue"] + S * pitch].view(S, pitch).cpu().numpy().copy()
    ed = est[lay["off_edotlu"]: lay["off_edotlu"] + S * pitch].view(S, pitch).cpu().numpy().copy()
    return ed, jb


def fill_tables(eng, value: float):
    import torch
    from tardis_b200.parallel import estimator_tensor

    lay = eng.estimator_layout()
    est = estimator_tensor(eng)
    est[lay["off_j_blue"]: lay["off_j_blue"] + 2 * lay["n_shells"] * lay["line_pitch"]] = value
    torch.cuda.synchronize()


def ulp_distance(got: np.ndarray, prefixes, nu_line, scale: float, full_rel: bool, max_ulps: float, what: str) -> float:
    """Every got[i] against prefix[i] / scale * nu_i in exact arithmetic: exactly 0.0 where the prefix is 0, within
    max_ulps ulp(exact) elsewhere.  -> the largest distance seen beyond a correct rounding, in ulps."""
    sc = Fraction(scale)
    nus = [Fraction(1) if full_rel else Fraction(float(x)) for x in nu_line]
    num = [p * sc.denominator * nu.numerator for p, nu in zip(prefixes, nus)]
    den = [sc.numerator * nu.denominator for nu in nus]
    rounded = np.array([n / d for n, d in zip(num, den)])  # int / int is correctly rounded
    zero = np.array([p == 0 for p in prefixes])
    assert np.array_equal(got[zero], np.zeros(int(zero.sum()))) and not np.signbit(got[zero]).any(), f"{what}: cells without a term must be 0.0"
    worst = 0.0
    for i in np.nonzero(got != rounded)[0]:  # equal to the correctly rounded value: within half an ulp
        ulp = math.ulp(rounded[i])
        d = abs(Fraction(float(got[i])) - Fraction(num[i], den[i])) / Fraction(ulp)
        assert d <= max_ulps, f"{what}: cell {i}: {got[i]!r} is {float(d):.3f} ulp from the exact {rounded[i]!r}"
        worst = max(worst, float(d))
    return worst


# ---------------------------------------------------------------------------------------------------------------------
# B. finalize_line_estimators_kernel on crafted words
# ---------------------------------------------------------------------------------------------------------------------
FINALIZE_LINES = (1, 31, 32, 33, 1023, 1024, 1025, 2047, 2048, 2049, 5000)
FINALIZE_SHELLS = (1, 3, 20)
TILE = 1024  # FIN_THREADS: cells per tile of the epilogue


def crafted_rows(n_lines: int, n_shells: int, seed: int):
    """[S][n_lines + 1][4]: every (shell, quantity) row gets its own +v / -v pairs (v > 0, first cell < closing cell), so
    every prefix is >= 0 and every row sums to zero:
      * 40 random pairs whose high and low words have opposite signs (either way round);
      * a low word holding a sum far beyond 2^29: +-(2^62 - r - 1), and on odd rows a pair (+2^34, -2^62 + r);
      * even rows: +big at cell 0 and -big at cell n_lines, big ~ 2^62 in the high word (a prefix of 2^91 in every cell:
        more than 64 bits, and every tile needs the running carry);
      * pairs on the cells around every tile edge (1022 .. 1025, 2046 .. 2049, ...);
      * with three shells or more, every fifth row stays all zero.
    Odd rows have cells before their first pair: exact zeros."""
    rng = np.random.default_rng(seed)
    cells = [[[0, 0, 0, 0] for _ in range(n_lines + 1)] for _ in range(n_shells)]

    def pair(s, q, a, b, hi, lo):
        assert 0 <= a < b <= n_lines and hi * 2**29 + lo > 0
        cells[s][a][2 * q] += hi; cells[s][a][2 * q + 1] += lo
        cells[s][b][2 * q] -= hi; cells[s][b][2 * q + 1] -= lo

    def mixed(flip):
        if flip:
            return -int(rng.integers(1, 2**10)), int(rng.integers(2**45, 2**50))
        return int(rng.integers(2**20, 2**40)), -int(rng.integers(1, 2**45))

    for s in range(n_shells):
        for q in (0, 1):
            r = 2 * s + q
            if n_shells >= 3 and r % 5 == 3:
                continue
            first = 0 if r % 2 == 0 else min(n_lines - 1, 1 + int(rng.integers(0, 7)))
            for j in range(40):
                a = int(rng.integers(first, n_lines))
                pair(s, q, a, int(rng.integers(a + 1, n_lines + 1)), *mixed(j % 2))
            a = int(rng.integers(first, n_lines))
            b = int(rng.integers(a + 1, n_lines + 1))
            pair(s, q, a, b, 0, 2**62 - r - 1)
            if r % 2 == 1:
                pair(s, q, a, b, 2**34, -(2**62) + r)
            else:
                pair(s, q, 0, n_lines, 2**62 - 12345 * r, int(rng.integers(0, 2**29)))
            for edge in range(TILE, n_lines + 1, TILE):
                for a in (edge - 2, edge - 1, edge):
                    if first <= a and a + 1 <= n_lines:
                        pair(s, q, a, a + 1, *mixed(a % 2))
    assert all(abs(w) < 2**63 for shell in cells for cell in shell for w in cell)
    return cells


def finalize_model(n_shells: int, n_lines: int):
    from tardis_b200 import synthetic as syn

    model = syn.make_model(n_shells, n_lines, "scatter", mu_tau=-4.0, seed=8200 + n_lines)
    packets = syn.make_packets(64, model.r_inner[0], base_seed=8201)  # energies 2^-6: the typical energy is exact
    return model, packets


def start_engine(eng, model, packets, **config):
    """One small run, so that the accumulators exist and have their scales; -> its result."""
    configure(eng, POOLED)
    eng.set_model_from(model, **config)
    return eng.run_packets(packets)


@pytest.mark.gpu
@pytest.mark.parametrize("full_rel", [False, True], ids=["partial_rel", "full_rel"])
@pytest.mark.parametrize("n_shells", FINALIZE_SHELLS)
@pytest.mark.parametrize("n_lines", FINALIZE_LINES)
def test_finalize_kernel_matches_exact_prefix_sums(engine, n_lines, n_shells, full_rel):
    """Every cell of both tables from crafted words.  Bars: a cell whose exact prefix is 0 is exactly 0.0, as are the pad
    cells; any other within 1 ulp of the exact value in full relativity, 2 ulps otherwise.  Where the ulps come from:
    i128_to_double rounds twice (the low 64 bits to a double, then the sum with the exact high part: at most 3/4 ulp
    together, and a single rounding when the value fits 64 bits); `* inv_scale` is exact (a power of two); `* nu_i` rounds
    once more (1/2 ulp), and the 3/4 ulp before it can weigh up to 3/2 ulp of the product."""
    model, packets = finalize_model(n_shells, n_lines)
    start_engine(engine, model, packets, enable_full_relativity=full_rel)
    scale_j_blue, scale_edotlu = model_scales(model.line_list_nu, typical_energy(packets.initial_energies), full_rel)
    _, api_scales = device_words(engine)
    assert sorted(api_scales) == sorted((scale_j_blue, scale_edotlu))
    cells = crafted_rows(n_lines, n_shells, seed=n_lines * 100 + n_shells * 2 + full_rel)
    write_words(engine, cells)
    fill_tables(engine, 7.0)  # the kernel must write every cell of both tables, pads included
    engine.finalize_line_estimators()
    engine.sync()
    edotlu, j_blue = device_tables(engine)
    assert np.array_equal(edotlu[:, n_lines:], np.zeros_like(edotlu[:, n_lines:])), "Edotlu pad cells"
    assert np.array_equal(j_blue[:, n_lines:], np.zeros_like(j_blue[:, n_lines:])), "J_blue pad cells"
    prefixes, totals = row_prefixes(cells, n_lines)
    assert all(t == [0, 0] for t in totals)
    bar = 1 if full_rel else 2
    for s in range(n_shells):
        ulp_distance(edotlu[s, :n_lines], prefixes[s][0], model.line_list_nu, scale_edotlu, full_rel, bar, f"Edotlu shell {s}")
        ulp_distance(j_blue[s, :n_lines], prefixes[s][1], model.line_list_nu, scale_j_blue, full_rel, bar, f"J_blue shell {s}")
    down = engine.download()
    assert np.array_equal(down["j_blue"], j_blue[:, :n_lines].T) and np.array_equal(down["edotlu"], edotlu[:, :n_lines].T)


DETECT_LINES, DETECT_SHELLS = 2500, 3


def expect_fixed_point_error(eng):
    from tardis_b200.engine import EngineError

    eng.finalize_line_estimators()
    with pytest.raises(EngineError, match="fixed-point line-estimator accumulator"):
        eng.sync()


@pytest.mark.gpu
def test_finalize_kernel_detects_rows_that_cannot_be_sums(engine):
    """What the epilogue refuses and what it must not: each case on the words of one engine, each followed by an ordinary
    run on the same engine that gives the first run's tables again."""
    model, packets = finalize_model(DETECT_SHELLS, DETECT_LINES)
    first = start_engine(engine, model, packets)
    L = DETECT_LINES

    def runs_again():
        again = engine.run_packets(packets)
        assert np.array_equal(again["j_blue"], first["j_blue"]) and np.array_equal(again["edotlu"], first["edotlu"])

    def rows(s, q, entries, n_cells=L + 2):
        cells = [[[0, 0, 0, 0] for _ in range(n_cells)] for _ in range(DETECT_SHELLS)]
        for i, hi, lo in entries:
            cells[s][i][2 * q], cells[s][i][2 * q + 1] = hi, lo
        return cells

    # a row that does not sum to zero, in either word
    for s, q, entries in ((1, 1, [(10, 5, 0)]), (2, 0, [(3, 7, 1), (2000, -7, 0)])):
        write_words(engine, rows(s, q, entries))
        expect_fixed_point_error(engine)
        runs_again()
    # the closing word at cell n_lines is counted: a range over every line raises nothing ...
    write_words(engine, rows(0, 1, [(0, 2**40, 17), (L, -(2**40), -17)]))
    engine.finalize_line_estimators()
    engine.sync()
    _, j_blue = device_tables(engine)
    assert (j_blue[0, :L] > 0).all() and not j_blue[1:].any()
    # ... and without it the row is refused, whatever lies one cell further (the last cell of the row: never a range's end)
    write_words(engine, rows(0, 1, [(0, 2**40, 17), (L + 1, -(2**40), -17)]))
    expect_fixed_point_error(engine)
    runs_again()
    write_words(engine, rows(2, 0, [(L + 1, 7, 7)]))
    engine.finalize_line_estimators()
    engine.sync()
    edotlu, j_blue = device_tables(engine)
    assert not edotlu.any() and not j_blue.any()
    runs_again()


@pytest.mark.gpu
@pytest.mark.parametrize("quantity", [0, 1], ids=["edotlu_words", "j_blue_words"])
def test_finalize_kernel_detects_a_wrap_that_the_closing_cell_mirrors(engine, quantity):
    """True high-word sums of 2^63 + k and -(2^63 + k) read as -2^63 + k and 2^63 - k: the row sums to zero, and every
    prefix between them is negative.  The tables it would give are wrong by 2^93 / scale; it must be an error."""
    model, packets = finalize_model(DETECT_SHELLS, DETECT_LINES)
    first = start_engine(engine, model, packets)
    wrap = symmetric_wrap_row(DETECT_LINES + 1, 1500, 2200, k=5)[0]  # inside the second and the third tile
    cells = [[[0, 0, 0, 0]] for _ in range(DETECT_SHELLS)]
    cells[1] = [[c[0], 0, 0, 0] if quantity == 0 else [0, 0, c[0], 0] for c in wrap]
    assert row_prefixes([cells[1]], DETECT_LINES)[1] == [[0, 0]]
    write_words(engine, cells)
    expect_fixed_point_error(engine)
    again = engine.run_packets(packets)
    assert np.array_equal(again["j_blue"], first["j_blue"]) and np.array_equal(again["edotlu"], first["edotlu"])


@pytest.mark.gpu
def test_group_collective_detects_a_wrap_of_the_summed_words():
    """The same wrap the way it arises: each of two members holds a valid row (zero total, positive prefixes, high words of
    2^62 + k and 2^62), and the collective sums the words before it finalises.  The group call must report it, naming a
    member, and the group must run again."""
    from tardis_b200.engine import EngineError, EngineGroup

    model, packets = finalize_model(DETECT_SHELLS, DETECT_LINES)
    arrays = (packets.initial_radii, packets.initial_nus, packets.initial_mus, packets.initial_energies, packets.packet_seeds)
    g = EngineGroup([0, 0])
    try:
        g.set_model_from(model)
        first = g.run(*arrays)
        g.upload_packets(*arrays)
        g.transport()
        g.sync()
        for member, hi in zip(g.members, (2**62 + 5, 2**62)):
            cells = [[[0, 0, 0, 0]] for _ in range(DETECT_SHELLS)]
            cells[2] = [[0, 0, 0, 0] for _ in range(DETECT_LINES + 1)]
            cells[2][700][2], cells[2][1800][2] = hi, -hi
            write_words(member, cells)
            member.finalize_line_estimators()  # on its own each half is a valid row
            member.sync()
            assert (device_tables(member)[1][2, 700:1800] > 0).all()
        with pytest.raises(EngineError, match=r"group member \d \(device 0\): .*fixed-point line-estimator accumulator"):
            g.allreduce()
        again = g.run(*arrays)
        assert np.array_equal(again["j_blue"], first["j_blue"]) and np.array_equal(again["edotlu"], first["edotlu"])
    finally:
        g.close()


@pytest.mark.gpu
def test_line_accumulator_scales_are_the_ones_their_names_say(engine):
    """Engine.line_accumulators returns (.., J_blue scale, Edotlu scale).  Rebuilding Edotlu from the w1 words and J_blue from
    the w2 words of an ordinary run with the scales as named gives the downloaded tables (to the epilogue's 2 ulps); with
    the two exchanged they would be off by the power of two next to nu_typ."""
    from tardis_b200 import synthetic as syn

    model = syn.make_model(5, 2000, "macroatom", mu_tau=-3.0, seed=8301)
    packets = syn.make_packets(20_000, model.r_inner[0], base_seed=8302)
    configure(engine, POOLED)
    engine.set_model_from(model)
    res = engine.run_packets(packets)
    words, scales = device_words(engine)
    assert scales == model_scales(model.line_list_nu, typical_energy(packets.initial_energies), False) and scales[0] != scales[1]
    host = words.cpu().numpy()
    edotlu, j_blue, totals = finalize_rows(host, model.line_list_nu, scales, False)
    assert all(t == [0, 0] for t in totals)
    assert np.count_nonzero(res["j_blue"]) > 1000
    for name, exact in (("edotlu", edotlu), ("j_blue", j_blue)):
        for s in range(model.n_shells):
            for i, x in enumerate(exact[s]):
                got = float(res[name][i, s])
                if x == 0:
                    assert got == 0.0, (name, s, i)
                else:
                    assert abs(Fraction(got) - x) <= 2 * Fraction(math.ulp(float(x))), (name, s, i, got, float(x))


# ---------------------------------------------------------------------------------------------------------------------
# C. Term conversion and range placement through the transport kernels
# ---------------------------------------------------------------------------------------------------------------------
SIGMA_OFF = 1e-200      # Thomson cross-section: no electron scattering
FREE_LINES = 3000
FREE_SHELLS = (1, 2, 7)
SETS = ("equal", "powers_of_two", "heavy", "wide")
N_TRAJECTORIES = 256    # distinct (nu, mu) of a packet set
HEAVY_PACKETS = 2 * 65536  # the typical energy is sampled at every second packet: the odd ones do not count
REFUSED_LOG2 = 35


@functools.lru_cache(maxsize=None)
def _oracle():
    from oracle import cpu_oracle

    cpu_oracle.build()
    return cpu_oracle


@functools.lru_cache(maxsize=None)
def free_model(n_shells: int, wide: bool):
    """Scatter model whose lines have tau ~ 1e-40: with SIGMA_OFF no packet ever interacts.  wide: the line list spans a
    factor 1e4 in frequency (w2 of packets at its two ends then spans 1e8) instead of 40."""
    from tardis_b200 import synthetic as syn

    kw = dict(lambda_min_A=100.0, lambda_max_A=1.0e6) if wide else {}
    return syn.make_model(n_shells, FREE_LINES, "scatter", mu_tau=-40.0, seed=8400 + n_shells, **kw)


def trajectories(model, seed: int):
    """N_TRAJECTORIES (nu, mu) at r_inner[0]: log-uniform over the line list, and at fixed slots packets that start above
    it and sweep into it, above it for good, on its last lines (they run off its end) and below it.  (nu is the comoving
    frequency at injection; on its way out a packet sweeps about 3 % down from it.)"""
    rng = np.random.default_rng(seed)
    first, last = float(model.line_list_nu[0]), float(model.line_list_nu[-1])
    nus = np.exp(rng.uniform(np.log(last), np.log(first), N_TRAJECTORIES))
    mus = np.sqrt(rng.random(N_TRAJECTORIES))
    nus[1] = math.sqrt(first * last) * 1.003       # the heavy packet's slot: a typical frequency
    nus[2:10] = [first * 1.01, first * 1.005, first * 1.05, first * 1.5, last * 1.01, last * 1.005, last * 0.9, last * 0.5]
    mus[2:10] = [0.95, 0.99, 0.9, 0.3, 0.9, 0.5, 0.9, 0.3]
    return nus, mus


def lab_frame(model, nu: float, mu: float, energy: float, full_rel: bool):
    """(nu, E) of one packet in the lab frame, from the oracle."""
    from tardis_b200 import synthetic as syn

    one = syn.Packets(np.array([float(model.r_inner[0])]), np.array([nu]), np.array([mu]), np.array([energy]), np.array([1], dtype=np.int64), 1.0)
    ref = _oracle().run_oracle(model, one, sigma_thomson=SIGMA_OFF, enable_full_relativity=full_rel, track_last_interaction=False)
    return float(ref["output_nus"][0]), float(ref["output_energies"][0])


def heaviest_log2(model, nu: float, e_lab: float, e_typ: float, full_rel: bool) -> int:
    """Largest k for which a packet of lab-frame energy 2^k e_lab and frequency nu passes fixed_term in both words."""
    scale_j_blue, scale_edotlu = model_scales(model.line_list_nu, e_typ, full_rel)
    k = 0
    while True:
        try:
            w1 = math.ldexp(e_lab, k + 1) if full_rel else math.ldexp(e_lab, k + 1) * (1.0 / nu)
            fixed_words(w1, scale_edotlu), fixed_words(w1 * (1.0 / nu), scale_j_blue)
        except FixedPointRange:
            return k
        k += 1


@functools.lru_cache(maxsize=None)
def packet_set(name: str, n_shells: int, heavy_log2: int | None = None):
    """(model, packets).  Energies:
      equal          1 / 256 each, as every other test of the suite has them;
      powers_of_two  2^k / 512, k uniform in -30 .. 30.  The typical energy is the mean over all 256 (the sample stride is 1
                     below 65536 packets), which the few largest dominate: 2^25.7 / 512.  The smallest Edotlu term is then
                     2^1.6 units of the low word, the largest 2^65 units (2^7 typical ones);
      heavy          131072 packets of 2^-17 on the 256 trajectories in turn, and one of 2^k 2^-17 at index 1, k the largest
                     that fixed_term accepts in partial and in full relativity (31 or 32): the sample takes the even indices,
                     so the typical energy stays 2^-17 and the heavy term is 2^k typical ones;
      wide           equal energies on the model whose line list spans 1e4 in frequency."""
    from tardis_b200 import synthetic as syn

    model = free_model(n_shells, name == "wide")
    nus, mus = trajectories(model, 8500 + SETS.index(name))
    rng = np.random.default_rng(8600 + SETS.index(name))
    n = HEAVY_PACKETS if name == "heavy" else N_TRAJECTORIES
    idx = np.arange(n) % N_TRAJECTORIES
    if name == "powers_of_two":
        energies = np.ldexp(1.0 / 512, rng.integers(-30, 31, n))
    elif name == "heavy":
        energies = np.full(n, 2.0**-17)
        k = heavy_log2 if heavy_log2 is not None else min(
            heaviest_log2(model, *lab_frame(model, nus[1], mus[1], 2.0**-17, fr), 2.0**-17, fr) for fr in (False, True))
        energies[1] = math.ldexp(2.0**-17, k)
    else:
        energies = np.full(n, 1.0 / n)
    seeds = rng.integers(1, 2**32 - 1, n).astype(np.int64)
    return model, syn.Packets(np.full(n, float(model.r_inner[0])), nus[idx].copy(), mus[idx].copy(), energies, seeds, 1.0)


@functools.lru_cache(maxsize=None)
def coverage(name: str, n_shells: int, full_rel: bool):
    """[trajectory][shell] -> (first, behind last) of the lines the packet's trace in that shell covers: the non-zero pattern
    of the oracle's J_blue for that packet alone.  Also asserts that the oracle saw no interaction."""
    from tardis_b200 import synthetic as syn

    model, packets = packet_set(name, n_shells)
    out = []
    for t in range(N_TRAJECTORIES):
        one = syn.Packets(*(np.array(a[t: t + 1]) for a in (packets.initial_radii, packets.initial_nus, packets.initial_mus)),
                          np.array([1.0]), np.array(packets.packet_seeds[t: t + 1]), 1.0)
        ref = _oracle().run_oracle(model, one, sigma_thomson=SIGMA_OFF, enable_full_relativity=full_rel, track_last_interaction=False)
        assert ref["counters"]["n_line_events"] == 0 and ref["counters"]["n_escat_events"] == 0 and ref["output_energies"][0] > 0
        assert np.array_equal(ref["j_blue"] != 0, ref["edotlu"] != 0)
        ranges = []
        for s in range(n_shells):
            hit = np.nonzero(ref["j_blue"][:, s])[0]
            a, b = (int(hit[0]), int(hit[-1]) + 1) if len(hit) else (0, 0)
            assert len(hit) == b - a, "a trace covers consecutive lines"
            ranges.append((a, b))
        out.append(ranges)
    return out


class Expected:
    """Exact tables and words of one (packet set, shell count, relativity)."""


@functools.lru_cache(maxsize=None)
def oracle_run(name: str, n_shells: int, full_rel: bool):
    model, packets = packet_set(name, n_shells)
    ref = _oracle().run_oracle(model, packets, sigma_thomson=SIGMA_OFF, enable_full_relativity=full_rel,
                               track_last_interaction=False, nthreads=4)
    assert ref["counters"]["n_line_events"] == 0 and ref["counters"]["n_escat_events"] == 0
    return ref


_expected = {}


def expected(name: str, n_shells: int, full_rel: bool, lab_nus, lab_energies) -> Expected:
    """lab_nus, lab_energies: the packets' lab-frame doubles (a run's output_nus / output_energies)."""
    key = (name, n_shells, full_rel, lab_nus.tobytes(), lab_energies.tobytes())
    if key not in _expected:
        _expected[key] = build_expected(name, n_shells, full_rel, lab_nus, lab_energies)
    return _expected[key]


def build_expected(name: str, n_shells: int, full_rel: bool, lab_nus, lab_energies) -> Expected:
    model, packets = packet_set(name, n_shells)
    assert len(lab_nus) == len(packets) and (lab_energies > 0).all()
    cov = coverage(name, n_shells, full_rel)
    L = model.n_lines
    nu_line = [Fraction(float(x)) for x in model.line_list_nu]
    e = Expected()
    e.scale_j_blue, e.scale_edotlu = model_scales(model.line_list_nu, typical_energy(packets.initial_energies), full_rel)
    # classes of identical packets: (trajectory, lab-frame nu, lab-frame energy) -> count
    classes = {}
    for key in zip((np.arange(len(packets)) % N_TRAJECTORIES).tolist(), lab_nus.tolist(), lab_energies.tolist()):
        classes[key] = classes.get(key, 0) + 1
    # words[variant]: A = E * (1 / nu) and that * (1 / nu) (what trace_range_end computes), B = E / nu and that / nu
    e.words = {v: np.zeros((n_shells, L + 1, 4), dtype=np.int64) for v in "AB"}
    acc = {v: {} for v in "AB"}
    steps = [{} for _ in range(n_shells)]  # shell -> cell -> [d W1, d W2, d terms]
    for (t, nu, en), count in classes.items():
        E = Fraction(en)
        W1 = E * count if full_rel else E * count / Fraction(nu)
        W2 = W1 / Fraction(nu)
        inv = 1.0 / nu
        a1 = en if full_rel else en * inv
        b1 = en if full_rel else en / nu
        terms = {"A": fixed_words(a1, e.scale_edotlu) + fixed_words(a1 * inv, e.scale_j_blue),
                 "B": fixed_words(b1, e.scale_edotlu) + fixed_words(b1 / nu, e.scale_j_blue)}
        for s, (a, b) in enumerate(cov[t]):
            if a == b:
                continue
            for cell, sign in ((a, 1), (b, -1)):
                st = steps[s].setdefault(cell, [Fraction(0), Fraction(0), 0])
                st[0] += sign * W1; st[1] += sign * W2; st[2] += sign * count
                for v in "AB":
                    w = acc[v].setdefault((s, cell), [0, 0, 0, 0])
                    for j in range(4):
                        w[j] += sign * count * terms[v][j]
    for v in "AB":
        for (s, cell), w in acc[v].items():
            e.words[v][s, cell] = [signed64(x) for x in w]
    # tables: the correctly rounded exact value, the number of terms and the exact value's own Fraction per covered cell
    e.edotlu, e.j_blue, e.terms = (np.zeros((n_shells, L)) for _ in range(3))
    for s in range(n_shells):
        run = [Fraction(0), Fraction(0), 0]
        cells = sorted(steps[s])
        for cell, nxt in zip(cells, cells[1:] + [L]):
            run = [x + d for x, d in zip(run, steps[s][cell])]
            for i in range(cell, min(nxt, L)):
                f = Fraction(1) if full_rel else nu_line[i]
                e.edotlu[s, i], e.j_blue[s, i], e.terms[s, i] = float(run[0] * f), float(run[1] * f), run[2]
        assert run == [0, 0, 0]
    e.nu_factor = np.ones(L) if full_rel else np.asarray(model.line_list_nu, dtype=np.float64)
    return e


def conversion_ulps(full_rel: bool) -> dict:
    """Roundings between the inputs and a table cell, each at most one ulp of the cell (the terms are positive, so the sum's
    relative error is at most a term's): w1 = E * (1 / nu) rounds twice (full relativity: w1 = E, not at all), w2 = w1 *
    (1 / nu) once or twice more; the epilogue adds its 2 ulps (1 in full relativity, see above); the reference the cell is
    compared with is the exact value rounded once (1/2)."""
    return {"edotlu": (0 if full_rel else 2) + (1 if full_rel else 2) + 0.5, "j_blue": (2 if full_rel else 3) + (1 if full_rel else 2) + 0.5}


def check_tables(res, e: Expected, full_rel: bool, what: str, rel: float | None = None) -> dict:
    """Jump kernels (rel None): |got - exact| <= terms(cell) / (2 scale) nu_i + conversion_ulps ulp(exact): each term's low
    word is rounded to the nearest unit 1 / scale, a typical term being 2^58 units.  Scan kernel: |got - exact| <= rel exact.
    Cells that no packet covers are exactly 0.0 either way.  -> per table (the largest error beyond the rounding of the low
    words, in ulps; the largest relative error)."""
    seen = {}
    for key, exact, scale in (("edotlu", e.edotlu, e.scale_edotlu), ("j_blue", e.j_blue, e.scale_j_blue)):
        got = np.ascontiguousarray(res[key].T)
        assert np.array_equal(got[exact == 0], np.zeros(int((exact == 0).sum()))), f"{what}: {key}: a cell no packet covers is not 0.0"
        err = np.abs(got - exact)
        units = e.terms * (0.5 / scale) * e.nu_factor[None, :]
        bar = units + conversion_ulps(full_rel)[key] * np.spacing(exact) if rel is None else rel * exact
        bad = np.argwhere(err > bar)
        assert len(bad) == 0, f"{what}: {key}: {len(bad)} cells beyond the bar, first (shell, line) {bad[0]}: {got[tuple(bad[0])]!r} vs {exact[tuple(bad[0])]!r}"
        on = exact != 0
        seen[key] = (float((np.maximum(err - units, 0.0)[on] / np.spacing(exact[on])).max()), float((err[on] / exact[on]).max()))
    return seen


def test_free_packets_do_not_interact_and_reach_both_ends_of_the_line_list():
    """CPU half of part C.  Every trajectory of every set passes through the oracle without an interaction (asserted in
    `coverage`); packets come from above the list, run off its end, and miss it on both sides; the heavy packet is 2^31 or
    2^32 typical terms and the refused one is out of range in both words; and the oracle's own tables, which evaluate
    E (1 - (d + mu r) / (c t)) with its cancellation, lie within 1e-12 of the exact values (printed: the distance that
    DESIGN section 2 quotes)."""
    for name in SETS:
        for n_shells in FREE_SHELLS:
            model, packets = packet_set(name, n_shells)
            for full_rel in (False, True):
                cov = coverage(name, n_shells, full_rel)
                spans = [(min(a for a, b in r if a < b), max(b for a, b in r if a < b)) if any(a < b for a, b in r) else None for r in cov]
                last = model.n_lines - 1  # the reference's trace stops at the last line of the list without an update for it
                assert any(sp and sp[0] == 0 for sp in spans) and max(sp[1] for sp in spans if sp) == last
                assert spans[4] is None and spans[5] is None and spans[8] is None and spans[9] is None
                assert spans[2][0] == 0 and spans[6][1] == last and spans[7][1] == last and spans[1] is not None
                assert sum(sp is not None and 0 < sp[0] and sp[1] < last for sp in spans) > 200
                if n_shells > 1:  # a crossing hands the range on at the same column
                    assert all(r[s][1] == r[s + 1][0] for r in cov for s in range(n_shells - 1) if r[s][0] < r[s][1] and r[s + 1][0] < r[s + 1][1])
                ref = oracle_run(name, n_shells, full_rel)
                e = expected(name, n_shells, full_rel, ref["output_nus"], ref["output_energies"])
                assert np.count_nonzero(e.j_blue) > 500 and e.terms.max() >= 2
                worst = 0.0
                for key, exact in (("edotlu", e.edotlu), ("j_blue", e.j_blue)):
                    got = ref[key].T
                    assert np.array_equal(got != 0, exact != 0)
                    on = exact != 0
                    worst = max(worst, float((np.abs(got[on] - exact[on]) / exact[on]).max()))
                assert worst < 1e-12
                print(f"oracle vs exact: {name} S={n_shells} full_rel={full_rel}: max relative distance {worst:.2e}")
    model, packets = packet_set("heavy", 7)
    k = round(math.log2(packets.initial_energies[1] / packets.initial_energies[0]))
    assert k in (31, 32) and typical_energy(packets.initial_energies) == packets.initial_energies[0]
    for full_rel in (False, True):
        nu_lab, e_lab = lab_frame(model, packets.initial_nus[1], packets.initial_mus[1], 2.0**-17, full_rel)
        assert k <= heaviest_log2(model, nu_lab, e_lab, 2.0**-17, full_rel) < REFUSED_LOG2 - 2
    # powers_of_two: the smallest Edotlu term is a few units of the low word, the largest a few tens of typical ones
    model, packets = packet_set("powers_of_two", 7)
    ref = oracle_run("powers_of_two", 7, False)
    t1 = ref["output_energies"] * (1.0 / ref["output_nus"]) * model_scales(model.line_list_nu, typical_energy(packets.initial_energies), False)[1]
    print(f"powers_of_two: typical energy {typical_energy(packets.initial_energies) * 512:.3e} / 512, Edotlu terms 2^{math.log2(t1.min()):.1f} .. 2^{math.log2(t1.max()):.1f} units")
    assert t1.min() < 2.0**8 and 2.0**60 < t1.max() < 2.0**66


KERNEL_CASES = {"pooled": (POOLED, {}), "lane": (LANE, {}), "volley": ({"algorithm": 1}, {"number_of_vpackets": 1}), "scan": (SCAN, {})}


@pytest.mark.gpu
@pytest.mark.parametrize("full_rel", [False, True], ids=["partial_rel", "full_rel"])
@pytest.mark.parametrize("kernel", sorted(KERNEL_CASES))
@pytest.mark.parametrize("name", SETS)
def test_transport_kernels_match_exact_rationals(engine, name, kernel, full_rel):
    """Pooled jump, lane-resident jump and warp-volley kernel: the accumulator words equal the word model's sums cell for
    cell, all four words (the device forms w1 = E * (1 / nu), w2 = w1 * (1 / nu): variant A; variant B, E / nu and w1 / nu,
    is computed too and would be accepted, since either is a faithful w), and the tables lie within the bar of `check_tables`
    of the exact rationals.  The scan kernel adds doubles with REDs, and the same reference judges it at 1e-12."""
    options, config = KERNEL_CASES[kernel]
    for n_shells in FREE_SHELLS:
        model, packets = packet_set(name, n_shells)
        configure(engine, options)
        engine.set_model_from(model, sigma_thomson=SIGMA_OFF, enable_full_relativity=full_rel, **config)
        res = engine.run_packets(packets)
        e = expected_of_run(res, name, n_shells, full_rel)
        what = f"{name}, {kernel}, {n_shells} shells"
        if kernel == "scan":
            seen = check_tables(res, e, full_rel, what, rel=1e-12)
            print(f"scan kernel vs exact: {what}, full_rel={full_rel}: relative {seen['edotlu'][1]:.2e} / {seen['j_blue'][1]:.2e}")
            continue
        words, scales = device_words(engine)
        assert sorted(scales) == sorted((e.scale_j_blue, e.scale_edotlu)), what
        got = words.cpu().numpy()
        assert not got[:, model.n_lines + 1:].any(), f"{what}: words behind cell n_lines"
        got = got[:, : model.n_lines + 1]
        variant = [v for v in "AB" if np.array_equal(got, e.words[v])]
        assert variant, f"{what}: {int((got != e.words['A']).any(axis=2).sum())} cells differ from the word model"
        seen = check_tables(res, e, full_rel, what)
        print(f"kernel vs exact: {what}, full_rel={full_rel}: words of variant {variant[0]}, Edotlu / J_blue beyond the low words' rounding "
              f"{seen['edotlu'][0]:.2f} / {seen['j_blue'][0]:.2f} ulp, relative {seen['edotlu'][1]:.2e} / {seen['j_blue'][1]:.2e}")
    configure(engine, POOLED)


def expected_of_run(res, name: str, n_shells: int, full_rel: bool) -> Expected:
    """The exact tables for the lab-frame frequencies and energies the run itself reports, which are the oracle's to a few ulps."""
    ref = oracle_run(name, n_shells, full_rel)
    for k in ("output_nus", "output_energies"):
        np.testing.assert_allclose(res[k], ref[k], rtol=1e-14, atol=0, err_msg=k)
    return expected(name, n_shells, full_rel, res["output_nus"], res["output_energies"])


def refused_set(alone: bool = False):
    """The heavy set with its heavy packet at 2^35 typical terms: out of range in both words, and invisible to the typical
    energy.  alone: every other packet passes above the line list, so nothing else is added to the heavy packet's cells (a
    term clipped to the largest word would then neither wrap a word nor unbalance a row: only fixed_term can refuse it)."""
    import dataclasses

    model, packets = packet_set("heavy", 7, REFUSED_LOG2)
    assert typical_energy(packets.initial_energies) == 2.0**-17
    if alone:
        nus = np.full(len(packets), float(model.line_list_nu[0]) * 1.5)
        nus[1] = packets.initial_nus[1]
        packets = dataclasses.replace(packets, initial_nus=nus)
    return model, packets


def arrays_of(packets):
    return (packets.initial_radii, packets.initial_nus, packets.initial_mus, packets.initial_energies, packets.packet_seeds)


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["resident", "run", "run_alone"])
def test_term_out_of_range_is_refused_not_clipped(engine, path):
    """One packet of 2^35 typical energy: EngineError naming the fixed-point accumulator, from the resident launch and from
    tb200_run (host packets), among other packets and as the only one that adds a term; the same engine then runs the heavy
    set that is in range and gives its exact tables."""
    from tardis_b200.engine import EngineError

    model, bad = refused_set(alone=path == "run_alone")
    configure(engine, POOLED)
    engine.set_model_from(model, sigma_thomson=SIGMA_OFF)
    with pytest.raises(EngineError, match="fixed-point line-estimator accumulator out of range"):
        if path == "resident":
            engine.upload_packets(*arrays_of(bad))
            engine.transport(True)
            engine.sync()
        else:
            engine.run(*arrays_of(bad))
    _, good = packet_set("heavy", 7)
    res = engine.run(*arrays_of(good))
    check_tables(res, expected_of_run(res, "heavy", 7, False), False, "after the refusal")


@pytest.mark.gpu
def test_group_names_the_member_whose_term_is_out_of_range():
    from tardis_b200.engine import EngineError, EngineGroup

    model, bad = refused_set()
    _, good = packet_set("heavy", 7)
    g = EngineGroup([0, 0])
    try:
        g.set_model_from(model, sigma_thomson=SIGMA_OFF)
        with pytest.raises(EngineError, match=r"group member 0 \(device 0, global packets \[0, 65536\)\): fixed-point line-estimator accumulator out of range"):
            g.run(*arrays_of(bad))
        res = g.run(*arrays_of(good))
        check_tables(res, expected_of_run(res, "heavy", 7, False), False, "group after the refusal")
    finally:
        g.close()
