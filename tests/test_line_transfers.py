"""Shell-crossing transfers of the jump kernels' line estimators (trace_range_end, fold_transfers_kernel).

A packet that crosses into a neighbouring shell adds its weight once to a transfer row between the two shells instead of
closing its range in one shell's difference row and opening the next in the other; a fold after the launch adds
xfer[s - 1] - xfer[s] to every shell's row.  The words are integers added mod 2^64, so the difference arrays must come out
bit for bit as they were with one direct +w / -w pair per trace.  The digests below were recorded on an H100 from the
engine as it was before the transfers existed; every comparison here is on the raw int64 accumulator words.

Run as a script (`python tests/test_line_transfers.py`, the package importable) to print the digests of the tree it
imports."""
import hashlib
import json

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

# name -> (model, engine configuration, packets, seeds)
WORKLOADS = {
    # the benchmark's model (20 shells, 5e5 lines, macro atom, tau ~ 10^N(-7.5, 2)) at 2e5 packets
    "macroatom_bench": dict(shells=20, lines=500_000, mode="macroatom", mu_tau=-7.5, packets=200_000, seed=None, base_seed=501,
                            config={}),
    "scatter_full_relativity": dict(shells=20, lines=50_000, mode="scatter", mu_tau=-6.0, packets=200_000, seed=502, base_seed=503,
                                    config={"enable_full_relativity": True}),
    # IIP mode: full relativity, continuum processes, 50 shells (~50 crossings per packet)
    "continuum_50_shells": dict(shells=50, lines=100_000, mode="macroatom", mu_tau=-7.5, packets=100_000, seed=504, base_seed=505,
                                config={}, continuum=True),
}

# SHA-256 of {accumulator words, output_nus, output_energies, counters} per workload, from the engine without transfers
DIGESTS = {
    "continuum_50_shells": {
        "words": "ae7bff69995bd1f39ae20ae7dc5252513e37ed94be7c4257f4a730d43ccaa83e",
        "output_nus": "2a6cf6f886818f9d5881d5b996a7365a486639d7e4ff2c0d60206993fe0df882",
        "output_energies": "e4ab6ab65ede667f5643fafaf7a43094cff797c7a1b21ac1622cac0db6064954",
        "counters": "18633c8160f7cfbe14c53e2da8d1d6343b81c3373a6d1359de68d0daabf8d6d7",
    },
    "macroatom_bench": {
        "words": "2ca46a49a3c9735432f8c9d9dd46b95a8c35833620216979f97d6ec88a0a456f",
        "output_nus": "bfc613636429f6112b11fdea91fcdcf8c611ffe16fca08294a8160d779e06f5d",
        "output_energies": "6f2ee69265771eb851b9946fba9c2c67a05983e7f4e6a5eb45db44bf52a6549a",
        "counters": "762a0cee41f1cd20b03deaec6df90de07fb3035a8ccde30566010ebbf0c09218",
    },
    "scatter_full_relativity": {
        "words": "fe3593c23aae2717073213c81638fa289b83466b21a2a8550406b16713bb27fa",
        "output_nus": "dd5d34683c0594b5dcabac12eae892e6d7c7897477151576a0442aca3d61c238",
        "output_energies": "71157ac51254a24ae466729156e691808dc55d12307500c3476902a90d276ada",
        "counters": "367962be675e1ebebcb8eadb03abc9883ba1c82795f6dac9690bc0190d705975",
    },
}


def _model_and_packets(name):
    from tardis_b200 import synthetic as syn

    w = WORKLOADS[name]
    kw = {} if w["seed"] is None else {"seed": w["seed"]}
    model = syn.make_model(w["shells"], w["lines"], w["mode"], mu_tau=w["mu_tau"], **kw)
    if w.get("continuum"):
        syn.add_continuum(model)
    packets = syn.make_packets(w["packets"], model.r_inner[0], base_seed=w["base_seed"])
    return model, packets, w["config"]


def _sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def accumulator_words(engine) -> np.ndarray:
    """The int64 words of the fixed-point difference arrays behind J_blue / Edotlu, copied to the host."""
    from tardis_b200.parallel import line_accumulator_tensor

    words, _ = line_accumulator_tensor(engine)
    return words.cpu().numpy().copy()


def run_digests(name, pooled: int = 1) -> dict:
    from tardis_b200.engine import Engine

    model, packets, config = _model_and_packets(name)
    eng = Engine(0)
    try:
        eng.set_option("algorithm", 1)
        eng.set_option("pooled", pooled)
        eng.set_model_from(model, **config)
        res = eng.run_packets(packets)
        counters = {k: v for k, v in res["counters"].items() if k != "n_search_probes"}  # (search cost, not a result)
        return {"words": _sha(accumulator_words(eng)), "output_nus": _sha(res["output_nus"]),
                "output_energies": _sha(res["output_energies"]),
                "counters": hashlib.sha256(json.dumps(counters, sort_keys=True).encode()).hexdigest()}
    finally:
        eng.close()


@pytest.mark.parametrize("pooled", [1, 0], ids=["pooled", "lane"])
@pytest.mark.parametrize("name", sorted(WORKLOADS))
def test_accumulator_words_match_direct_range_updates(name, pooled):
    """Accumulator words, per-packet outputs and work counters are those of one direct +w / -w pair per trace, for the
    pooled kernel and the lane-resident one alike (the words are integer sums: which kernel ran must not show)."""
    assert run_digests(name, pooled) == DIGESTS[name]


def test_pipelined_run_matches_resident_words():
    """tb200_run splits >= 4e6 packets into ranges and folds the transfers once, after the last range: its words equal
    those of one resident launch over the same packets."""
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import Engine

    model = syn.make_model(12, 6000, "macroatom", mu_tau=-5.0, seed=511)
    packets = syn.make_packets(4_200_000, model.r_inner[0], base_seed=512)
    eng = Engine(0)
    try:
        eng.set_option("algorithm", 1)
        eng.set_model_from(model)
        piped = eng.run_packets(packets)
        piped_words = accumulator_words(eng)
        eng.upload_packets(packets.initial_radii, packets.initial_nus, packets.initial_mus, packets.initial_energies,
                           packets.packet_seeds)
        eng.transport(True)
        eng.sync()
        resident = eng.download()
        assert np.array_equal(piped_words, accumulator_words(eng))
        assert np.array_equal(piped["j_blue"], resident["j_blue"]) and np.array_equal(piped["edotlu"], resident["edotlu"])
        assert np.array_equal(piped["output_nus"], resident["output_nus"])
    finally:
        eng.close()


def test_accumulating_calls_match_one_call():
    """transport(zero_estimators=False) adds to the words: two calls over the halves of a packet set leave exactly the words
    of one call over the whole set (same energies, so the same fixed-point scale)."""
    from tardis_b200 import synthetic as syn
    from tardis_b200.engine import Engine

    model = syn.make_model(20, 20_000, "macroatom", mu_tau=-6.0, seed=521)
    packets = syn.make_packets(300_000, model.r_inner[0], base_seed=522)
    cols = (packets.initial_radii, packets.initial_nus, packets.initial_mus, packets.initial_energies, packets.packet_seeds)
    half = len(packets.initial_nus) // 2
    eng = Engine(0)
    try:
        eng.set_option("algorithm", 1)
        eng.set_model_from(model)
        eng.upload_packets(*cols)
        eng.transport(True)
        eng.sync()
        whole = accumulator_words(eng)
        eng.upload_packets(*(c[:half] for c in cols))
        eng.transport(True)
        eng.upload_packets(*(c[half:] for c in cols))
        eng.transport(False)
        eng.sync()
        assert np.array_equal(accumulator_words(eng), whole)
    finally:
        eng.close()


if __name__ == "__main__":
    print(json.dumps({name: run_digests(name) for name in sorted(WORKLOADS)}, indent=4))
