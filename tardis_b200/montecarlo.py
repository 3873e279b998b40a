"""Host-side mirror of the reference's Monte Carlo transport interface for the classic
(line + Thomson) mode, backed by the CUDA engine.

Same names, argument meaning and side effects as (paths relative to the reference's tardis/ package):

* ``montecarlo_transport_with_vpackets``   transport/montecarlo/modes/montecarlo_transport.py:239-373
* ``MCTransportSolverClassic``             transport/montecarlo/modes/classic/solver.py:49-363
  (here ``MCTransportSolverB200``: ``from_config`` / ``initialize_transport_state`` / ``run``)
* ``MonteCarloTransportState``             transport/montecarlo/montecarlo_transport_state.py:15-317
* ``PacketCollection`` / ``VPacketCollection``  transport/montecarlo/packets/packet_collections.py:14-386
* ``EstimatorsBulk`` / ``EstimatorsLine``  transport/montecarlo/estimators/estimators_{bulk,line}.py
* ``MonteCarloConfiguration`` / ``configuration_initialize``  transport/montecarlo/configuration/base.py:11-78

The classes are plain Python (no Numba jitclasses): the arrays they carry go straight
across the C-ABI.  Everything is duck-typed on attribute names, so the reference's own
``NumbaHomologousRadial1DGeometry`` / ``OpacityStateNumba`` / ``PacketCollection`` objects
(or the host ``OpacityState`` products after ``.to_numba()``) can be passed unchanged; see
INTEGRATION.md for the two injection points the reference already has
(``Simulation.from_config(..., transport=solver)``, ``workflow.transport_solver = solver``).
There is no CPU fallback: without the CUDA library every call raises.
"""
from __future__ import annotations

import logging

import numpy as np

from . import macro_atom
from .engine import SIGMA_THOMSON, Engine, EngineGroup, MacroAtomError, MonteCarloException  # noqa: F401 (re-exported)

logger = logging.getLogger(__name__)

LINE_INTERACTION = {"scatter": 0, "downbranch": 1, "macroatom": 2}
C_SPEED_OF_LIGHT = 2.99792458e10

# InteractionType names, packets/radiative_packet.py:12-35
INTERACTION_TYPE_NAMES = {-1: "NO_INTERACTION", 1: "BOUNDARY", 2: "LINE", 4: "ESCATTERING", 8: "CONTINUUM_PROCESS"}


def _value(x):
    """Plain float/ndarray of a number, ndarray or astropy Quantity (already in cgs in the reference's carriers)."""
    return getattr(x, "value", x)


def _quantity(value, unit):
    """Attach a unit when astropy is importable (the reference's properties return Quantities)."""
    try:
        from astropy import units as u  # noqa: PLC0415

        return value * u.Unit(unit)
    except Exception:
        return value


# --------------------------------------------------------------------------------------
# data carriers
# --------------------------------------------------------------------------------------
class PacketCollection:
    """packets/packet_collections.py:14-76"""

    def __init__(self, initial_radii, initial_nus, initial_mus, initial_energies, packet_seeds, radiation_field_luminosity):
        self.initial_radii = np.ascontiguousarray(initial_radii, dtype=np.float64)
        self.initial_nus = np.ascontiguousarray(initial_nus, dtype=np.float64)
        self.initial_mus = np.ascontiguousarray(initial_mus, dtype=np.float64)
        self.initial_energies = np.ascontiguousarray(initial_energies, dtype=np.float64)
        self.packet_seeds = np.ascontiguousarray(packet_seeds, dtype=np.int64)
        self.radiation_field_luminosity = float(radiation_field_luminosity)
        self.time_of_simulation = 1 / self.radiation_field_luminosity
        self.output_nus = np.ones_like(self.initial_radii, dtype=np.float64) * -99.0
        self.output_energies = np.ones_like(self.initial_radii, dtype=np.float64) * -99.0

    @property
    def number_of_packets(self) -> int:
        return len(self.initial_radii)


class HomologousGeometry:
    """NumbaHomologousRadial1DGeometry, model/geometry/radial1d_homologous.py:199-226 (plain arrays, cgs)."""

    def __init__(self, r_inner, r_outer, v_inner, v_outer, time_explosion):
        self.r_inner = np.ascontiguousarray(r_inner, dtype=np.float64)
        self.r_outer = np.ascontiguousarray(r_outer, dtype=np.float64)
        self.v_inner = np.ascontiguousarray(v_inner, dtype=np.float64)
        self.v_outer = np.ascontiguousarray(v_outer, dtype=np.float64)
        self.time_explosion = float(time_explosion)
        self.velocity_gradient = 1.0 / self.time_explosion
        self.volume = (4 / 3) * np.pi * (self.r_outer**3 - self.r_inner**3)

    def get_velocity(self, r, shell_id):
        return r / self.time_explosion


class OpacityState:
    """Classic-mode fields of OpacityStateNumba (opacities/opacity_state_numba.py:13-72) with the same
    shell slicing (`state[i:j]`, :157-196): shell-dependent tables become (possibly non-contiguous) views."""

    def __init__(self, electron_density, t_electrons, line_list_nu, tau_sobolev, transition_probabilities,
                 line2macro_level_upper, macro_block_edge_index, transition_type, destination_level_id, transition_line_id):
        self.electron_density = electron_density
        self.t_electrons = t_electrons
        self.line_list_nu = line_list_nu
        self.tau_sobolev = tau_sobolev
        self.transition_probabilities = transition_probabilities
        self.line2macro_level_upper = line2macro_level_upper
        self.macro_block_edge_index = macro_block_edge_index
        self.transition_type = transition_type
        self.destination_level_id = destination_level_id
        self.transition_line_id = transition_line_id

    def __getitem__(self, i: slice):
        return OpacityState(self.electron_density[i], self.t_electrons[i], self.line_list_nu, self.tau_sobolev[:, i],
                            self.transition_probabilities[:, i],
                            self.line2macro_level_upper, self.macro_block_edge_index, self.transition_type,
                            self.destination_level_id, self.transition_line_id)

    @classmethod
    def from_model(cls, model):
        """From a `tardis_b200.synthetic.Model`."""
        m = model.macro
        return cls(model.electron_density, model.t_electrons, model.line_list_nu, model.tau_sobolev,
                   m.transition_probabilities, m.line2macro_level_upper, m.macro_block_edge_index, m.transition_type,
                   m.destination_level_id, m.transition_line_id)


class EstimatorsBulk:
    """estimators/estimators_bulk.py:15-104"""

    def __init__(self, mean_intensity_total, mean_frequency):
        self.mean_intensity_total = mean_intensity_total
        self.mean_frequency = mean_frequency

    def increment(self, other):
        self.mean_intensity_total += other.mean_intensity_total
        self.mean_frequency += other.mean_frequency


class EstimatorsLine:
    """estimators/estimators_line.py:15-112"""

    def __init__(self, mean_intensity_blueward, energy_deposition_line_rate):
        self.mean_intensity_blueward = mean_intensity_blueward
        self.energy_deposition_line_rate = energy_deposition_line_rate

    def increment(self, other):
        self.mean_intensity_blueward += other.mean_intensity_blueward
        self.energy_deposition_line_rate += other.energy_deposition_line_rate


class EstimatorsContinuum:
    """estimators/estimators_continuum.py:15-175"""

    FIELDS = ("photo_ion_estimator", "stim_recomb_estimator", "bf_heating_estimator", "stim_recomb_cooling_estimator",
              "ff_heating_estimator", "photo_ion_estimator_statistics")

    def __init__(self, photo_ion_estimator, stim_recomb_estimator, bf_heating_estimator, stim_recomb_cooling_estimator,
                 ff_heating_estimator, photo_ion_estimator_statistics):
        self.photo_ion_estimator = photo_ion_estimator
        self.stim_recomb_estimator = stim_recomb_estimator
        self.bf_heating_estimator = bf_heating_estimator
        self.stim_recomb_cooling_estimator = stim_recomb_cooling_estimator
        self.ff_heating_estimator = ff_heating_estimator
        self.photo_ion_estimator_statistics = photo_ion_estimator_statistics

    def increment(self, other):
        for k in self.FIELDS:
            getattr(self, k).__iadd__(getattr(other, k))


class VPacketCollection:
    """Consolidated virtual-packet tracker (packets/packet_collections.py:103-386).  The six
    "last interaction" arrays are the reference's placeholders (-99, virtual_packet.py:375-386)."""

    def __init__(self, nus, energies, initial_mus, initial_rs, spectrum_frequency_grid=None,
                 v_packet_spawn_start_frequency=0.0, v_packet_spawn_end_frequency=1e200):
        n = len(nus)
        self.nus, self.energies, self.initial_mus, self.initial_rs = nus, energies, initial_mus, initial_rs
        self.last_interaction_in_nu = np.full(n, -99.0)
        self.last_interaction_in_r = np.full(n, -99.0)
        self.last_interaction_type = np.full(n, -99, dtype=np.int64)
        self.last_interaction_in_id = np.full(n, -99, dtype=np.int64)
        self.last_interaction_out_id = np.full(n, -99, dtype=np.int64)
        self.last_interaction_shell_id = np.full(n, -99, dtype=np.int64)
        self.idx = n
        self.length = n
        self.source_rpacket_index = -1
        self.number_of_vpackets = -1
        self.spectrum_frequency_grid = spectrum_frequency_grid
        self.v_packet_spawn_start_frequency = v_packet_spawn_start_frequency
        self.v_packet_spawn_end_frequency = v_packet_spawn_end_frequency


class MonteCarloConfiguration:
    """configuration/base.py:11-49 (same field names and defaults)."""

    def __init__(self):
        self.ENABLE_FULL_RELATIVITY = False
        self.TEMPORARY_V_PACKET_BINS = 0
        self.NUMBER_OF_VPACKETS = 0
        self.MONTECARLO_SEED = 0
        self.LINE_INTERACTION_TYPE = 0
        self.PACKET_SEEDS = np.empty(1, dtype=np.int64)
        self.DISABLE_ELECTRON_SCATTERING = False
        self.DISABLE_LINE_SCATTERING = False
        self.SURVIVAL_PROBABILITY = 0.0
        self.VPACKET_TAU_RUSSIAN = 10.0
        self.INITIAL_TRACKING_ARRAY_LENGTH = 0
        self.LEGACY_MODE_ENABLED = False
        self.VPACKET_SPAWN_START_FREQUENCY = 0
        self.VPACKET_SPAWN_END_FREQUENCY = 1e200
        self.ENABLE_VPACKET_TRACKING = False


def _to_hz(q) -> float:
    """Wavelength/frequency Quantity -> Hz (configuration/base.py:69-74 uses u.spectral())."""
    if hasattr(q, "to"):
        from astropy import units as u  # noqa: PLC0415

        return float(q.to(u.Hz, equivalencies=u.spectral()).value)
    return float(q)


def configuration_initialize(config, transport, number_of_vpackets):
    """configuration/base.py:52-78"""
    if transport.line_interaction_type not in LINE_INTERACTION:
        raise ValueError(
            'Line interaction type must be one of "macroatom","downbranch", or "scatter" but is '
            f"{transport.line_interaction_type}"
        )
    config.LINE_INTERACTION_TYPE = LINE_INTERACTION[transport.line_interaction_type]
    config.NUMBER_OF_VPACKETS = number_of_vpackets
    config.TEMPORARY_V_PACKET_BINS = number_of_vpackets
    config.ENABLE_FULL_RELATIVITY = transport.enable_full_relativity
    config.MONTECARLO_SEED = getattr(transport.packet_source, "base_seed", 0)
    # note the swap: the spawn range is given in wavelength (start < end) -> frequency start = nu(end)
    config.VPACKET_SPAWN_START_FREQUENCY = _to_hz(transport.vpacket_spawn_range.end)
    config.VPACKET_SPAWN_END_FREQUENCY = _to_hz(transport.vpacket_spawn_range.start)
    config.ENABLE_VPACKET_TRACKING = transport.enable_vpacket_tracking


class LastInteractionTrackers:
    """SoA stand-in for the reference's list of ``TrackerLastInteraction`` jitclass objects
    (packets/trackers/tracker_last_interaction.py:7-254): pass one as ``trackers`` and the engine
    fills the columns of ``trackers_last_interaction_to_df`` (tracker_last_interaction_util.py:33-134)."""

    INT_COLUMNS = ("last_interaction_type", "last_event_id", "last_shell_id", "last_line_absorb_id", "last_line_emit_id")
    FLOAT_COLUMNS = ("last_radius", "last_before_nu", "last_before_mu", "last_before_energy",
                     "last_after_nu", "last_after_mu", "last_after_energy")

    def __init__(self, no_of_packets: int):
        self.no_of_packets = no_of_packets
        self.columns = {}

    def __len__(self):
        return self.no_of_packets

    def to_df(self):
        import pandas as pd  # noqa: PLC0415

        c = self.columns
        it = pd.Categorical([INTERACTION_TYPE_NAMES[int(t)] for t in c["last_interaction_type"]],
                            categories=list(INTERACTION_TYPE_NAMES.values()))
        status = pd.Categorical(["IN_PROCESS"] * self.no_of_packets,
                                categories=["IN_PROCESS", "EMITTED", "REABSORBED", "ADIABATIC_COOLING"])
        return pd.DataFrame(
            {
                "event_id": c["last_event_id"], "last_interaction_type": it, "status": status,
                "radius": c["last_radius"], "shell_id": c["last_shell_id"],
                "before_nu": c["last_before_nu"], "before_mu": c["last_before_mu"], "before_energy": c["last_before_energy"],
                "after_nu": c["last_after_nu"], "after_mu": c["last_after_mu"], "after_energy": c["last_after_energy"],
                "line_absorb_id": pd.array(c["last_line_absorb_id"], dtype="int64"),
                "line_emit_id": pd.array(c["last_line_emit_id"], dtype="int64"),
            },
            index=pd.RangeIndex(self.no_of_packets, name="packet_id"),
        )


def generate_tracker_last_interaction_list(no_of_packets: int) -> LastInteractionTrackers:
    """Same name as packets/trackers/tracker_last_interaction_util.py:17."""
    return LastInteractionTrackers(no_of_packets)


# attribute of the reference's TrackerLastInteraction (tracker_last_interaction.py:9-30) <- engine column
_REFERENCE_TRACKER_FIELDS = (
    ("interaction_type", "last_interaction_type"), ("interactions_count", "last_event_id"), ("shell_id", "last_shell_id"),
    ("interaction_line_absorb_id", "last_line_absorb_id"), ("interaction_line_emit_id", "last_line_emit_id"),
    ("radius", "last_radius"), ("before_nu", "last_before_nu"), ("before_mu", "last_before_mu"),
    ("before_energy", "last_before_energy"), ("after_nu", "last_after_nu"), ("after_mu", "last_after_mu"),
    ("after_energy", "last_after_energy"),
)


def _classify_trackers(trackers, n_packets: int) -> str:
    """'soa' (LastInteractionTrackers), 'reference' (a sequence of the reference's TrackerLastInteraction objects, filled
    from the engine's columns after the run), 'none' (None / empty: no tracking).  Anything else -- in particular the
    reference's TrackerFull list of `montecarlo.tracking.track_rpacket` -- is refused instead of being left unfilled."""
    if trackers is None:
        return "none"
    if isinstance(trackers, LastInteractionTrackers):
        return "soa"
    try:
        n = len(trackers)
    except TypeError:
        raise TypeError(f"unsupported `trackers` container {type(trackers).__name__}: pass generate_tracker_last_interaction_list(n) "
                        "from tardis_b200.montecarlo or the reference's list of TrackerLastInteraction") from None
    if n == 0:
        return "none"
    first = trackers[0]
    if all(hasattr(first, a) for a, _ in _REFERENCE_TRACKER_FIELDS):
        if n != n_packets:
            raise ValueError(f"`trackers` has {n} entries for {n_packets} packets")
        return "reference"
    raise NotImplementedError(
        f"`trackers` holds {type(first).__name__} objects: only last-interaction tracking is implemented by the CUDA engine "
        "(full r-packet tracking, montecarlo.tracking.track_rpacket, is out of scope -- DESIGN.md); the list would stay unfilled")


def _fill_reference_trackers(trackers, res) -> None:
    """Write the engine's last-interaction columns into the reference's per-packet tracker objects, so that its own
    trackers_last_interaction_to_df (tracker_last_interaction_util.py:33-134) reports what the packets did."""
    cols = [(a, res[c]) for a, c in _REFERENCE_TRACKER_FIELDS]
    for i, t in enumerate(trackers):
        for attr, col in cols:
            setattr(t, attr, col[i].item())


class FusedPacketSums:
    """What the kernel epilogue already summed over the finished packets (SURVEY.md §8f rank 2), so that the consumers
    need neither the 16 B/packet device-to-host copy nor an O(N) pass on the host:

    * ``spectrum_emitted`` / ``spectrum_reabsorbed``: energy histograms on the spectrum frequency grid
      == ``np.histogram(output_nus[mask], weights=|output_energies[mask]|, bins=grid)`` -- x 1 / time_of_simulation they are
      ``SpectrumSolver.montecarlo_emitted_luminosity`` / ``montecarlo_reabsorbed_luminosity`` (spectrum/base.py:139-159);
    * ``luminosity_sums`` = energy of {emitted, emitted inside the window, reabsorbed, reabsorbed inside the window}
      packets -- x 1 / time_of_simulation the ``emitted_luminosity`` / ``reabsorbed_luminosity`` of ``Simulation.iterate``
      (simulation/base.py:455-466, spectrum/luminosity.py:5-29; window = (luminosity_nu_start, luminosity_nu_end), strict)."""

    def __init__(self, spectrum_emitted, spectrum_reabsorbed, luminosity_sums, luminosity_nu_start, luminosity_nu_end):
        self.spectrum_emitted = spectrum_emitted
        self.spectrum_reabsorbed = spectrum_reabsorbed
        self.luminosity_sums = luminosity_sums
        self.luminosity_nu_start = luminosity_nu_start
        self.luminosity_nu_end = luminosity_nu_end


def _fused_sums(res, luminosity_nu_start, luminosity_nu_end):
    if "luminosity_sums" not in res:
        return None
    return FusedPacketSums(res.get("spectrum_emitted"), res.get("spectrum_reabsorbed"), res["luminosity_sums"],
                           luminosity_nu_start, luminosity_nu_end)


# --------------------------------------------------------------------------------------
# the FFI seam
# --------------------------------------------------------------------------------------
_engines = {}


def get_engine(device=0) -> Engine:
    """One engine (device buffers persist across MC iterations) per device and process.  A sequence of device ids gives
    one cached `EngineGroup` of them (an id may repeat: `[0, 0]` is two engines on device 0)."""
    key = int(device) if isinstance(device, (int, np.integer)) else tuple(int(d) for d in device)
    if key not in _engines:
        _engines[key] = Engine(key) if isinstance(key, int) else EngineGroup(key)
    return _engines[key]


def montecarlo_transport_with_vpackets(
    packet_collection,
    geometry_state_numba,
    time_explosion,
    opacity_state_numba,
    montecarlo_configuration,
    spectrum_frequency_grid,
    trackers,
    number_of_vpackets,
    show_progress_bars=False,
    packet_propagation_function=None,
    *,
    engine: Engine | None = None,
    sigma_thomson: float = SIGMA_THOMSON,
    vlog_capacity: int | None = None,
    luminosity_nu_start: float = 0.0,
    luminosity_nu_end: float = np.inf,
):
    """Drop-in for transport/montecarlo/modes/montecarlo_transport.py:239-373.

    Same positional arguments; returns ``(v_packets_energy_hist, vpacket_tracker, estimators_bulk,
    estimators_line)`` and fills ``packet_collection.output_nus`` / ``output_energies`` in place.
    ``packet_propagation_function`` and ``show_progress_bars`` are accepted and ignored (the classic
    packet propagation is what the kernel implements).  ``sigma_thomson`` replaces the module constant
    the reference reads (configuration/constants.py:3).  ``luminosity_nu_start/end`` (Hz) is the window of the
    filtered luminosities the kernel epilogue sums; the sums and the fused spectra of this call are left in
    ``montecarlo_transport_with_vpackets.last_fused`` (a ``FusedPacketSums``).
    """
    cfg = montecarlo_configuration
    eng = engine or get_engine()
    o = opacity_state_numba
    grid = np.ascontiguousarray(_value(spectrum_frequency_grid), dtype=np.float64)
    # the geometry carrier decides the mode: NumbaRadial1DGeometry (model/geometry/radial1d.py:320-375) holds a per-shell
    # velocity_gradient -> the nonhomologous mode; NumbaHomologousRadial1DGeometry holds the scalar 1 / t_exp
    nonhomologous = np.ndim(getattr(geometry_state_numba, "velocity_gradient", 0.0)) == 1
    line_mode = int(cfg.LINE_INTERACTION_TYPE)
    if int(cfg.NUMBER_OF_VPACKETS) != int(number_of_vpackets):
        logger.debug("number_of_vpackets differs from configuration; using the argument, like the reference")
    eng.set_model(
        r_inner=_value(geometry_state_numba.r_inner), r_outer=_value(geometry_state_numba.r_outer),
        time_explosion=float(_value(time_explosion)),
        electron_density=o.electron_density, line_list_nu=o.line_list_nu, tau_sobolev=o.tau_sobolev,
        line_interaction_type=line_mode,
        transition_probabilities=o.transition_probabilities, line2macro_level_upper=o.line2macro_level_upper,
        macro_block_edge_index=o.macro_block_edge_index, transition_type=o.transition_type,
        destination_level_id=o.destination_level_id, transition_line_id=o.transition_line_id,
        spectrum_frequency_grid=grid,
        enable_full_relativity=bool(cfg.ENABLE_FULL_RELATIVITY),
        disable_line_scattering=bool(cfg.DISABLE_LINE_SCATTERING),
        sigma_thomson=sigma_thomson, number_of_vpackets=int(number_of_vpackets),
        survival_probability=float(cfg.SURVIVAL_PROBABILITY), vpacket_tau_russian=float(cfg.VPACKET_TAU_RUSSIAN),
        vpacket_spawn_start_frequency=float(cfg.VPACKET_SPAWN_START_FREQUENCY),
        vpacket_spawn_end_frequency=float(cfg.VPACKET_SPAWN_END_FREQUENCY),
        luminosity_nu_start=float(_value(luminosity_nu_start)), luminosity_nu_end=float(_value(luminosity_nu_end)),
        nonhomologous=nonhomologous,
        v_inner=_value(geometry_state_numba.v_inner) if nonhomologous else None,
        v_outer=_value(geometry_state_numba.v_outer) if nonhomologous else None,
    )
    pc = packet_collection
    n = len(pc.initial_nus)
    tracker_kind = _classify_trackers(trackers, n)
    track_last = tracker_kind != "none"
    want_vlog = bool(cfg.ENABLE_VPACKET_TRACKING) and number_of_vpackets > 0
    if want_vlog and vlog_capacity is None:
        vlog_capacity = max(1024, 64 * int(number_of_vpackets) * n)
    buffers = {}
    if isinstance(pc.output_nus, np.ndarray) and pc.output_nus.flags["C_CONTIGUOUS"] and pc.output_nus.dtype == np.float64:
        buffers = {"output_nus": pc.output_nus, "output_energies": pc.output_energies}
    res = eng.run(pc.initial_radii, pc.initial_nus, pc.initial_mus, pc.initial_energies, pc.packet_seeds,
                  track_last_interaction=track_last, vlog_capacity=vlog_capacity if want_vlog else 0, buffers=buffers)
    if want_vlog and res["vlog_count"] > vlog_capacity:
        # rare: log buffer too small -> run again with the exact size (results are seed-deterministic)
        res = eng.run(pc.initial_radii, pc.initial_nus, pc.initial_mus, pc.initial_energies, pc.packet_seeds,
                      track_last_interaction=track_last, vlog_capacity=int(res["vlog_count"]), buffers=buffers)
    if not buffers:
        pc.output_nus[:] = res["output_nus"]
        pc.output_energies[:] = res["output_energies"]
    estimators_bulk = EstimatorsBulk(res["j"], res["nu_bar"])
    estimators_line = EstimatorsLine(res["j_blue"], res["edotlu"])
    if tracker_kind == "soa":
        trackers.columns = {k: res[k] for k in LastInteractionTrackers.INT_COLUMNS + LastInteractionTrackers.FLOAT_COLUMNS}
    elif tracker_kind == "reference":
        _fill_reference_trackers(trackers, res)
    if want_vlog:
        m = res["vlog_count"]
        order = np.argsort(res["vlog_packet_index"][:m], kind="stable")  # the reference consolidates in packet order
        vpacket_tracker = VPacketCollection(res["vlog_nus"][:m][order], res["vlog_energies"][:m][order],
                                            res["vlog_initial_mus"][:m][order], res["vlog_initial_rs"][:m][order], grid,
                                            cfg.VPACKET_SPAWN_START_FREQUENCY, cfg.VPACKET_SPAWN_END_FREQUENCY)
    else:
        vpacket_tracker = VPacketCollection(np.empty(1), np.empty(1), np.empty(1), np.empty(1), grid,
                                            cfg.VPACKET_SPAWN_START_FREQUENCY, cfg.VPACKET_SPAWN_END_FREQUENCY)
    montecarlo_transport_with_vpackets.last_counters = res["counters"]
    montecarlo_transport_with_vpackets.last_estimators = (eng, res["j"], res["nu_bar"], res["j_blue"])  # what is resident in HBM
    montecarlo_transport_with_vpackets.last_fused = _fused_sums(res, float(_value(luminosity_nu_start)), float(_value(luminosity_nu_end)))
    return res["vhist"], vpacket_tracker, estimators_bulk, estimators_line


def montecarlo_transport(
    packet_collection,
    geometry_state_numba,
    time_explosion,
    opacity_state_numba,
    montecarlo_configuration,
    n_levels_bf_species_by_n_cells_tuple,
    trackers,
    show_progress_bars=False,
    *,
    engine: Engine | None = None,
    sigma_thomson: float = SIGMA_THOMSON,
    spectrum_frequency_grid=None,
    luminosity_nu_start: float = 0.0,
    luminosity_nu_end: float = np.inf,
):
    """Drop-in for the IIP / continuum main loop, transport/montecarlo/modes/iip/montecarlo_transport.py:40-176.

    `opacity_state_numba` is the reference's ``OpacityStateNumbaIIP`` (or any object with the same attributes,
    opacities/opacity_state_numba_iip.py:8-125).  Returns ``(estimators_bulk, estimators_line, estimators_continuum)``
    and fills ``packet_collection.output_nus / output_energies`` (packets destroyed by adiabatic cooling keep -99).
    Full relativity is always on and no virtual packets are spawned, as in the reference's IIP mode."""
    cfg = montecarlo_configuration
    eng = engine or get_engine()
    o = opacity_state_numba
    # the X that tardis_b200.macro_atom.create_absorbing_probs returned: rebuilt in HBM from its [T, S] input, not uploaded
    rebuild = macro_atom.built_inputs(getattr(o, "absorbing_markov_probabilities", None), o.transition_type)
    montecarlo_transport.last_markov_rebuilt = rebuild is not None
    eng.set_model(
        r_inner=_value(geometry_state_numba.r_inner), r_outer=_value(geometry_state_numba.r_outer),
        time_explosion=float(_value(time_explosion)),
        electron_density=o.electron_density, line_list_nu=o.line_list_nu, tau_sobolev=o.tau_sobolev,
        line_interaction_type=int(cfg.LINE_INTERACTION_TYPE),
        transition_probabilities=o.transition_probabilities, line2macro_level_upper=o.line2macro_level_upper,
        macro_block_edge_index=o.macro_block_edge_index, transition_type=o.transition_type,
        destination_level_id=o.destination_level_id, transition_line_id=o.transition_line_id,
        spectrum_frequency_grid=(None if spectrum_frequency_grid is None
                                 else np.ascontiguousarray(_value(spectrum_frequency_grid), dtype=np.float64)),
        enable_full_relativity=True,
        disable_line_scattering=bool(cfg.DISABLE_LINE_SCATTERING), sigma_thomson=sigma_thomson,
        continuum=o if rebuild is None else macro_atom.WithoutMatrix(o), t_electrons=o.t_electrons,
        luminosity_nu_start=float(_value(luminosity_nu_start)), luminosity_nu_end=float(_value(luminosity_nu_end)),
    )
    if rebuild is not None:
        eng.build_absorbing_markov(**rebuild)
    n_cont = len(o.bf_threshold_list_nu)
    if tuple(n_levels_bf_species_by_n_cells_tuple) not in ((n_cont, len(o.electron_density)), (0, 0)):
        logger.debug("n_levels_bf_species_by_n_cells_tuple %s differs from the continuum tables (%d, %d)",
                     n_levels_bf_species_by_n_cells_tuple, n_cont, len(o.electron_density))
    pc = packet_collection
    tracker_kind = _classify_trackers(trackers, len(pc.initial_nus))
    track_last = tracker_kind != "none"
    buffers = {}
    if isinstance(pc.output_nus, np.ndarray) and pc.output_nus.flags["C_CONTIGUOUS"] and pc.output_nus.dtype == np.float64:
        buffers = {"output_nus": pc.output_nus, "output_energies": pc.output_energies}
    res = eng.run(pc.initial_radii, pc.initial_nus, pc.initial_mus, pc.initial_energies, pc.packet_seeds,
                  track_last_interaction=track_last, buffers=buffers)
    if not buffers:
        pc.output_nus[:] = res["output_nus"]
        pc.output_energies[:] = res["output_energies"]
    if tracker_kind == "soa":
        trackers.columns = {k: res[k] for k in LastInteractionTrackers.INT_COLUMNS + LastInteractionTrackers.FLOAT_COLUMNS}
    elif tracker_kind == "reference":
        _fill_reference_trackers(trackers, res)
    montecarlo_transport.last_counters = res["counters"]
    montecarlo_transport_with_vpackets.last_estimators = (eng, res["j"], res["nu_bar"], res["j_blue"])
    montecarlo_transport.last_fused = _fused_sums(res, float(_value(luminosity_nu_start)), float(_value(luminosity_nu_end)))
    return (EstimatorsBulk(res["j"], res["nu_bar"]), EstimatorsLine(res["j_blue"], res["edotlu"]),
            EstimatorsContinuum(*(res[k] for k in EstimatorsContinuum.FIELDS)))


# --------------------------------------------------------------------------------------
# state object
# --------------------------------------------------------------------------------------
class MonteCarloTransportState:
    """montecarlo_transport_state.py:15-317 (same attribute and property names; HDF writing stays with the
    reference's HDFWriterMixin when this class is mixed into it by the integrator)."""

    hdf_properties = [
        "output_nu", "output_energy", "nu_bar_estimator", "j_estimator", "j_blue_estimator", "packet_luminosity",
        "time_of_simulation", "emitted_packet_mask", "last_interaction_type", "last_interaction_in_nu",
        "last_interaction_in_r", "last_line_interaction_out_id", "last_line_interaction_in_id",
        "last_line_interaction_shell_id",
    ]
    hdf_name = "transport_state"
    last_interaction_type = None
    last_interaction_in_nu = None
    last_interaction_in_r = None
    last_line_interaction_out_id = None
    last_line_interaction_in_id = None
    last_line_interaction_shell_id = None
    virt_logging = False

    def __init__(self, packet_collection, geometry_state_numba, opacity_state_numba, time_explosion,
                 n_levels_bf_species_by_n_cells_tuple=(0, 0), tracker_full_df=None, tracker_last_interaction_df=None,
                 vpacket_tracker=None):
        self.packet_collection = packet_collection
        self.n_levels_bf_species_by_n_cells_tuple = n_levels_bf_species_by_n_cells_tuple
        self.estimators_bulk = None
        self.estimators_line = None
        self.estimators_continuum = None
        self.enable_full_relativity = False
        self.enable_continuum_processes = False
        self.time_explosion = time_explosion
        self.geometry_state_numba = geometry_state_numba
        self.opacity_state_numba = opacity_state_numba
        self.tracker_full_df = tracker_full_df
        self.tracker_last_interaction_df = tracker_last_interaction_df
        self.vpacket_tracker = vpacket_tracker
        self.fused_packet_sums = None  # FusedPacketSums of the last run (CUDA engine only; not in the reference's state)

    # ---- the kernel epilogue's sums, in the units their consumers use (None before the first run) ----
    def _fused_luminosity(self, attr):
        f = self.fused_packet_sums
        if f is None or getattr(f, attr) is None:
            return None
        return getattr(f, attr) / self.packet_collection.time_of_simulation

    @property
    def montecarlo_emitted_luminosity(self):
        """== SpectrumSolver.montecarlo_emitted_luminosity (spectrum/base.py:151-159), erg/s per grid bin, without
        touching the per-packet arrays"""
        v = self._fused_luminosity("spectrum_emitted")
        return None if v is None else _quantity(v, "erg / s")

    @property
    def montecarlo_reabsorbed_luminosity(self):
        """== SpectrumSolver.montecarlo_reabsorbed_luminosity (spectrum/base.py:139-149)"""
        v = self._fused_luminosity("spectrum_reabsorbed")
        return None if v is None else _quantity(v, "erg / s")

    @property
    def emitted_luminosity(self):
        """== calculate_filtered_luminosity(emitted_packet_nu, emitted_packet_luminosity, luminosity_nu_start,
        luminosity_nu_end) of Simulation.iterate (simulation/base.py:455-460)"""
        v = self._fused_luminosity("luminosity_sums")
        return None if v is None else _quantity(v[1], "erg / s")

    @property
    def reabsorbed_luminosity(self):
        """== the reabsorbed twin (simulation/base.py:461-466)"""
        v = self._fused_luminosity("luminosity_sums")
        return None if v is None else _quantity(v[3], "erg / s")

    @property
    def output_nu(self):
        return _quantity(self.packet_collection.output_nus, "Hz")

    @property
    def output_energy(self):
        return _quantity(self.packet_collection.output_energies, "erg")

    @property
    def nu_bar_estimator(self):
        return self.estimators_bulk.mean_frequency

    @property
    def j_estimator(self):
        return self.estimators_bulk.mean_intensity_total

    @property
    def j_blue_estimator(self):
        return self.estimators_line.mean_intensity_blueward

    @property
    def time_of_simulation(self):
        return _quantity(self.packet_collection.time_of_simulation, "s")

    @property
    def packet_luminosity(self):
        return _quantity(self.packet_collection.output_energies / self.packet_collection.time_of_simulation, "erg") / _quantity(1.0, "s")

    @property
    def emitted_packet_mask(self):
        return self.packet_collection.output_energies >= 0

    @property
    def emitted_packet_nu(self):
        return _quantity(self.packet_collection.output_nus[self.emitted_packet_mask], "Hz")

    @property
    def reabsorbed_packet_nu(self):
        return _quantity(self.packet_collection.output_nus[~self.emitted_packet_mask], "Hz")

    @property
    def emitted_packet_luminosity(self):
        return self.packet_luminosity[self.emitted_packet_mask]

    @property
    def reabsorbed_packet_luminosity(self):
        return -self.packet_luminosity[~self.emitted_packet_mask]

    def _vp(self, name, unit=None):
        if self.vpacket_tracker is None or not self.virt_logging:
            return None
        v = getattr(self.vpacket_tracker, name)
        return _quantity(v, unit) if unit else v

    @property
    def virt_packet_nus(self):
        return self._vp("nus", "Hz")

    @property
    def virt_packet_energies(self):
        return self._vp("energies", "erg")

    @property
    def virtual_packet_luminosity(self):
        e = self.virt_packet_energies
        return None if e is None else e / self.packet_collection.time_of_simulation

    @property
    def virt_packet_initial_rs(self):
        return self._vp("initial_rs")

    @property
    def virt_packet_initial_mus(self):
        return self._vp("initial_mus")

    @property
    def virt_packet_last_interaction_in_nu(self):
        return self._vp("last_interaction_in_nu")

    @property
    def virt_packet_last_interaction_in_r(self):
        return self._vp("last_interaction_in_r")

    @property
    def virt_packet_last_interaction_type(self):
        return self._vp("last_interaction_type")

    @property
    def virt_packet_last_line_interaction_in_id(self):
        return self._vp("last_interaction_in_id")

    @property
    def virt_packet_last_line_interaction_out_id(self):
        return self._vp("last_interaction_out_id")

    @property
    def virt_packet_last_line_interaction_shell_id(self):
        return self._vp("last_interaction_shell_id")


# --------------------------------------------------------------------------------------
# estimator -> radiation field (SURVEY.md §8f rank 4)
# --------------------------------------------------------------------------------------
class DilutePlanckianRadiationField:
    """Carrier with the attributes `Simulation.advance_state` reads (plasma/radiation_field/planck_rad_field.py:7-53)."""

    def __init__(self, temperature, dilution_factor):
        self.temperature = temperature
        self.dilution_factor = dilution_factor

    @property
    def temperature_kelvin(self):
        return _value(self.temperature)


class EstimatedRadiationFieldProperties:
    """transport/montecarlo/estimators/base.py:8-11"""

    def __init__(self, dilute_blackbody_radiationfield_state, j_blues):
        self.dilute_blackbody_radiationfield_state = dilute_blackbody_radiationfield_state
        self.j_blues = j_blues


class MCRadiationFieldPropertiesSolverB200:
    """Drop-in for ``MCRadiationFieldPropertiesSolver`` (transport/montecarlo/estimators/mc_rad_field_solver.py:33-144): same
    ``solve`` signature and result attributes.  When the estimators passed in are the very arrays the engine returned from
    its last run on this device, nothing is uploaded: T_rad, W and the normalised / zero-filled J_blue table are computed
    from the copies that are still resident in HBM (``tb200_solve_radiation_field``)."""

    w_epsilon = 1e-10

    def __init__(self, w_epsilon: float = 1e-10, device: int = 0):
        self.w_epsilon = w_epsilon
        self.device = device

    def solve(self, estimators_bulk, estimators_line, time_explosion, time_of_simulation, volume, line_list_nu,
              detailed_optical_window=False):
        eng = get_engine(self.device)
        last = getattr(montecarlo_transport_with_vpackets, "last_estimators", None)
        resident = (last is not None and last[0] is eng and estimators_bulk.mean_intensity_total is last[1]
                    and estimators_bulk.mean_frequency is last[2] and estimators_line.mean_intensity_blueward is last[3])
        t_exp = time_explosion
        t_exp = float(t_exp.cgs.value) if hasattr(t_exp, "cgs") else float(_value(t_exp))
        t_sim = float(_value(time_of_simulation))
        est = None if resident else (estimators_bulk.mean_intensity_total, estimators_bulk.mean_frequency,
                                     estimators_line.mean_intensity_blueward)
        t_rad, w, j_blues = eng.solve_radiation_field(time_explosion=t_exp, time_of_simulation=t_sim, volume=_value(volume),
                                                      w_epsilon=self.w_epsilon, detailed_optical_window=detailed_optical_window,
                                                      estimators=est)
        return EstimatedRadiationFieldProperties(DilutePlanckianRadiationField(_quantity(t_rad, "K"), w), j_blues)


# --------------------------------------------------------------------------------------
# the solver
# --------------------------------------------------------------------------------------
class MCTransportSolverB200:
    """Drop-in for ``MCTransportSolverClassic`` (modes/classic/solver.py:49-363): same constructor
    arguments, ``initialize_transport_state``, ``run`` and ``from_config``; the Numba main loop is
    replaced by the CUDA engine.  ``nthreads`` is accepted for signature compatibility (no host
    threads are used); ``device`` selects the GPU of this process, or, as a list of ids, the `EngineGroup` that runs
    each iteration on several GPUs from this process."""

    hdf_properties = ["transport_state"]
    hdf_name = "transport"

    def __init__(self, radfield_prop_solver, spectrum_frequency_grid, vpacket_spawn_range, enable_full_relativity,
                 line_interaction_type, spectrum_method, packet_source, enable_virtual_packet_logging=False,
                 enable_rpacket_tracking=False, nthreads=1, debug_packets=False, logger_buffer=1, use_gpu=False,
                 montecarlo_configuration=None, device=0, sigma_thomson=SIGMA_THOMSON):
        self.radfield_prop_solver = radfield_prop_solver
        self.spectrum_frequency_grid = spectrum_frequency_grid
        self.vpacket_spawn_range = vpacket_spawn_range
        self.enable_full_relativity = enable_full_relativity
        self.line_interaction_type = line_interaction_type
        self.spectrum_method = spectrum_method
        self.use_gpu = use_gpu
        self.enable_vpacket_tracking = enable_virtual_packet_logging
        self.enable_rpacket_tracking = enable_rpacket_tracking
        self.montecarlo_configuration = montecarlo_configuration or MonteCarloConfiguration()
        self.packet_source = packet_source
        self.rpacket_tracker = None
        self.nthreads = nthreads
        self.device = device
        self.sigma_thomson = sigma_thomson
        self.transport_state = None
        # window of the filtered luminosities summed in the kernel epilogue (Hz); the workflow / Simulation that owns them
        # (simple_tardis_workflow.py:116-131, simulation/base.py:455-466) copies its luminosity_nu_start / _end here
        self.luminosity_nu_start = 0.0
        self.luminosity_nu_end = np.inf
        if enable_rpacket_tracking:
            raise NotImplementedError(
                "montecarlo.tracking.track_rpacket (TrackerFull) is a debugging feature that is out of scope for the "
                "CUDA engine (DESIGN.md); use the reference solver for it")

    def initialize_transport_state(self, simulation_state, opacity_state, macro_atom_state, plasma, no_of_packets,
                                   no_of_virtual_packets=0, iteration=0):
        """modes/classic/solver.py:102-152"""
        species = getattr(plasma, "continuum_interaction_species", None)
        if species is not None and not getattr(species, "empty", True):
            gamma = getattr(plasma, "gamma", None)
            n_levels_bf_species_by_n_cells_tuple = gamma.shape if gamma is not None else plasma.phi_lucy.shape
        else:
            n_levels_bf_species_by_n_cells_tuple = (0, 0)
        packet_collection = self.packet_source.create_packets(no_of_packets, seed_offset=iteration)
        try:  # other host code of the reference branches on this global (opacities/opacity_state.py:212)
            from tardis.transport.montecarlo.configuration import montecarlo_globals  # noqa: PLC0415

            montecarlo_globals.CONTINUUM_PROCESSES_ENABLED = False
        except Exception:
            pass
        geometry_state = simulation_state.geometry.to_numba()
        opacity_state_numba = opacity_state.to_numba(macro_atom_state, self.line_interaction_type)
        geo = simulation_state.geometry
        opacity_state_numba = opacity_state_numba[geo.v_inner_boundary_idx: geo.v_outer_boundary_idx]
        transport_state = MonteCarloTransportState(
            packet_collection, geometry_state_numba=geometry_state, opacity_state_numba=opacity_state_numba,
            time_explosion=simulation_state.time_explosion,
            n_levels_bf_species_by_n_cells_tuple=n_levels_bf_species_by_n_cells_tuple)
        transport_state.enable_full_relativity = self.montecarlo_configuration.ENABLE_FULL_RELATIVITY
        configuration_initialize(self.montecarlo_configuration, self, no_of_virtual_packets)
        return transport_state

    def run(self, transport_state, show_progress_bars=True):
        """modes/classic/solver.py:154-273: returns ``v_packets_energy_hist``; sets the estimators, the
        last-interaction DataFrame and (with virtual-packet logging) the vpacket tracker on the state."""
        self.transport_state = transport_state
        cfg = self.montecarlo_configuration
        number_of_vpackets = cfg.NUMBER_OF_VPACKETS
        n = len(transport_state.packet_collection.initial_nus)
        trackers = generate_tracker_last_interaction_list(n)
        t_exp = transport_state.time_explosion
        t_exp = float(t_exp.cgs.value) if hasattr(t_exp, "cgs") else float(_value(t_exp))
        v_packets_energy_hist, vpacket_tracker, estimators_bulk, estimators_line = montecarlo_transport_with_vpackets(
            transport_state.packet_collection, transport_state.geometry_state_numba, t_exp,
            transport_state.opacity_state_numba, cfg, _value(self.spectrum_frequency_grid), trackers,
            number_of_vpackets, show_progress_bars=show_progress_bars, packet_propagation_function=None,
            engine=get_engine(self.device), sigma_thomson=self.sigma_thomson,
            luminosity_nu_start=self.luminosity_nu_start, luminosity_nu_end=self.luminosity_nu_end)
        transport_state.fused_packet_sums = montecarlo_transport_with_vpackets.last_fused
        transport_state.estimators_bulk = estimators_bulk
        transport_state.estimators_line = estimators_line
        if cfg.ENABLE_VPACKET_TRACKING and number_of_vpackets > 0:
            transport_state.vpacket_tracker = vpacket_tracker
        transport_state.tracker_full_df = None
        transport_state.tracker_last_interaction_df = trackers.to_df()
        transport_state.virt_logging = cfg.ENABLE_VPACKET_TRACKING
        return v_packets_energy_hist

    run_classic = run

    @classmethod
    def from_config(cls, config, packet_source, enable_virtual_packet_logging=False, device=0,
                    honor_disable_electron_scattering=False):
        """modes/classic/solver.py:275-363.

        ``plasma.disable_electron_scattering``: the reference assigns ``constants.SIGMA_THOMSON = 1e-200`` here, but
        its hot path bound the constant at import time (``from ...constants import SIGMA_THOMSON``,
        opacities/opacities.py:10, packets/virtual_packet.py:22), so in a real run the MC loop keeps the physical
        cross-section.  Default: reproduce that effective behaviour; ``honor_disable_electron_scattering=True`` applies
        the intended 1e-200."""
        sigma = SIGMA_THOMSON
        if config.plasma.disable_electron_scattering:
            logger.warning("Disabling electron scattering - this is not physical.")
            if honor_disable_electron_scattering:
                sigma = 1e-200
        stop, start = _to_hz(config.spectrum.stop), _to_hz(config.spectrum.start)
        spectrum_frequency_grid = _quantity(np.linspace(stop, start, num=config.spectrum.num + 1), "Hz")
        mc_cfg = MonteCarloConfiguration()
        mc_cfg.DISABLE_LINE_SCATTERING = config.plasma.disable_line_scattering
        mc_cfg.DISABLE_ELECTRON_SCATTERING = config.plasma.disable_electron_scattering
        mc_cfg.INITIAL_TRACKING_ARRAY_LENGTH = config.montecarlo.tracking.initial_array_length
        try:
            from tardis.transport.montecarlo.estimators.mc_rad_field_solver import (  # noqa: PLC0415
                MCRadiationFieldPropertiesSolver,
            )

            radfield_prop_solver = MCRadiationFieldPropertiesSolver(config.plasma.w_epsilon)
        except Exception:  # the reference's solver is not importable: the engine's own (same surface, runs on the resident estimators)
            radfield_prop_solver = MCRadiationFieldPropertiesSolverB200(config.plasma.w_epsilon, device=device)
        running_mode = str(config.spectrum.integrated.compute).upper()
        if running_mode not in ("GPU", "AUTOMATIC", "CPU"):
            raise ValueError("An invalid option for compute was passed. The three valid values are 'GPU', 'CPU', and 'Automatic'.")
        return cls(
            radfield_prop_solver=radfield_prop_solver, spectrum_frequency_grid=spectrum_frequency_grid,
            vpacket_spawn_range=config.montecarlo.virtual_spectrum_spawn_range,
            enable_full_relativity=config.montecarlo.enable_full_relativity,
            line_interaction_type=config.plasma.line_interaction_type, spectrum_method=config.spectrum.method,
            packet_source=packet_source, debug_packets=config.montecarlo.debug_packets,
            logger_buffer=config.montecarlo.logger_buffer,
            enable_virtual_packet_logging=(config.spectrum.virtual.virtual_packet_logging | enable_virtual_packet_logging),
            enable_rpacket_tracking=config.montecarlo.tracking.track_rpacket, nthreads=config.montecarlo.nthreads,
            use_gpu=running_mode != "CPU", montecarlo_configuration=mc_cfg, device=device, sigma_thomson=sigma)


class MCTransportSolverB200IIP(MCTransportSolverB200):
    """Drop-in for ``MCTransportSolverIIP`` (modes/iip/solver.py): continuum processes always enabled, full relativity
    always on, no shell slicing of the opacity state, no virtual packets; ``run`` returns nothing the spectrum needs
    beyond the transport state (estimators_bulk / _line / _continuum are attached to it)."""

    def initialize_transport_state(self, simulation_state, opacity_state, macro_atom_state, plasma, no_of_packets,
                                   no_of_virtual_packets=0, iteration=0):
        """modes/iip/solver.py:100-160"""
        species = getattr(plasma, "continuum_interaction_species", None)
        n_levels_bf_species_by_n_cells_tuple = (0, 0)
        if species is not None and not getattr(species, "empty", True) and getattr(plasma, "nlte_species", None):
            import pandas as pd  # noqa: PLC0415

            n_levels_bf_species_by_n_cells_tuple = pd.concat(
                [plasma.phi_lucy.loc[sp] for sp in plasma.nlte_species], axis=0).shape
        packet_collection = self.packet_source.create_packets(no_of_packets, seed_offset=iteration)
        try:
            from tardis.transport.montecarlo.configuration import montecarlo_globals  # noqa: PLC0415

            montecarlo_globals.CONTINUUM_PROCESSES_ENABLED = True
        except Exception:
            pass
        geometry_state = simulation_state.geometry.to_numba()
        opacity_state_numba = opacity_state.to_numba(macro_atom_state, self.line_interaction_type)
        transport_state = MonteCarloTransportState(
            packet_collection, geometry_state_numba=geometry_state, opacity_state_numba=opacity_state_numba,
            time_explosion=simulation_state.time_explosion,
            n_levels_bf_species_by_n_cells_tuple=n_levels_bf_species_by_n_cells_tuple)
        transport_state.enable_full_relativity = True
        transport_state.enable_continuum_processes = True
        configuration_initialize(self.montecarlo_configuration, self, no_of_virtual_packets)
        return transport_state

    def run(self, transport_state, show_progress_bars=True):
        self.transport_state = transport_state
        n = len(transport_state.packet_collection.initial_nus)
        trackers = generate_tracker_last_interaction_list(n)
        t_exp = transport_state.time_explosion
        t_exp = float(t_exp.cgs.value) if hasattr(t_exp, "cgs") else float(_value(t_exp))
        bulk, line, cont = montecarlo_transport(
            transport_state.packet_collection, transport_state.geometry_state_numba, t_exp,
            transport_state.opacity_state_numba, self.montecarlo_configuration,
            transport_state.n_levels_bf_species_by_n_cells_tuple, trackers, show_progress_bars=show_progress_bars,
            engine=get_engine(self.device), sigma_thomson=self.sigma_thomson,
            spectrum_frequency_grid=self.spectrum_frequency_grid,
            luminosity_nu_start=self.luminosity_nu_start, luminosity_nu_end=self.luminosity_nu_end)
        transport_state.fused_packet_sums = montecarlo_transport.last_fused
        transport_state.estimators_bulk = bulk
        transport_state.estimators_line = line
        transport_state.estimators_continuum = cont
        transport_state.tracker_full_df = None
        transport_state.tracker_last_interaction_df = trackers.to_df()
        transport_state.virt_logging = False
        return np.zeros_like(np.asarray(_value(self.spectrum_frequency_grid), dtype=np.float64))


# --------------------------------------------------------------------------------------
# the nonhomologous mode (transport/montecarlo/modes/nonhomologous/)
# --------------------------------------------------------------------------------------
class MonteCarloTransportStateB200Nonhomologous(MonteCarloTransportState):
    """modes/nonhomologous/montecarlo_transport_state.py:8-288: the classic state without time_explosion (same
    properties)."""

    def __init__(self, packet_collection, geometry_state_numba, opacity_state_numba, n_levels_bf_species_by_n_cells_tuple,
                 tracker_full_df=None, tracker_last_interaction_df=None, vpacket_tracker=None):
        super().__init__(packet_collection, geometry_state_numba, opacity_state_numba, None,
                         n_levels_bf_species_by_n_cells_tuple=n_levels_bf_species_by_n_cells_tuple,
                         tracker_full_df=tracker_full_df, tracker_last_interaction_df=tracker_last_interaction_df,
                         vpacket_tracker=vpacket_tracker)


class MCRadiationFieldPropertiesSolverB200Nonhomologous(MCRadiationFieldPropertiesSolverB200):
    """Drop-in for the nonhomologous ``MCRadiationFieldPropertiesSolver`` (modes/nonhomologous/mc_rad_field_solver.py:35-131):
    J_blue normalised by (c / velocity_gradient) / (4 pi t_sim V), no optical window."""

    def solve(self, estimators_bulk, estimators_line, velocity_gradient, time_of_simulation, volume, line_list_nu):
        eng = get_engine(self.device)
        last = getattr(montecarlo_transport_with_vpackets, "last_estimators", None)
        resident = (last is not None and last[0] is eng and estimators_bulk.mean_intensity_total is last[1]
                    and estimators_bulk.mean_frequency is last[2] and estimators_line.mean_intensity_blueward is last[3])
        est = None if resident else (estimators_bulk.mean_intensity_total, estimators_bulk.mean_frequency,
                                     estimators_line.mean_intensity_blueward)
        t_rad, w, j_blues = eng.solve_radiation_field(time_explosion=0.0, time_of_simulation=float(_value(time_of_simulation)),
                                                      volume=_value(volume), w_epsilon=self.w_epsilon, estimators=est,
                                                      velocity_gradient=_value(velocity_gradient))
        return EstimatedRadiationFieldProperties(DilutePlanckianRadiationField(_quantity(t_rad, "K"), w), j_blues)


class MCTransportSolverB200Nonhomologous(MCTransportSolverB200):
    """Drop-in for ``MCTransportSolverNonhomologous`` (modes/nonhomologous/solver.py:48-358): the geometry carrier is
    NumbaRadial1DGeometry, the loop runs with time_explosion = 0.0, partial relativity only."""

    def initialize_transport_state(self, simulation_state, opacity_state, macro_atom_state, plasma, no_of_packets,
                                   no_of_virtual_packets=0, iteration=0):
        """modes/nonhomologous/solver.py:101-147 (opacities sliced by the r boundary indices)"""
        species = getattr(plasma, "continuum_interaction_species", None)
        if species is not None and not getattr(species, "empty", True):
            gamma = getattr(plasma, "gamma", None)
            n_levels_bf_species_by_n_cells_tuple = gamma.shape if gamma is not None else plasma.phi_lucy.shape
        else:
            n_levels_bf_species_by_n_cells_tuple = (0, 0)
        packet_collection = self.packet_source.create_packets(no_of_packets, seed_offset=iteration)
        geometry_state = simulation_state.geometry.to_numba()
        opacity_state_numba = opacity_state.to_numba(macro_atom_state, self.line_interaction_type)
        geo = simulation_state.geometry
        opacity_state_numba = opacity_state_numba[geo.r_inner_boundary_index: geo.r_outer_boundary_index]
        transport_state = MonteCarloTransportStateB200Nonhomologous(
            packet_collection, geometry_state_numba=geometry_state, opacity_state_numba=opacity_state_numba,
            n_levels_bf_species_by_n_cells_tuple=n_levels_bf_species_by_n_cells_tuple)
        transport_state.enable_full_relativity = self.montecarlo_configuration.ENABLE_FULL_RELATIVITY
        configuration_initialize(self.montecarlo_configuration, self, no_of_virtual_packets)
        return transport_state

    def run(self, transport_state, show_progress_bars=True):
        """modes/nonhomologous/solver.py:149-268: returns ``v_packets_energy_hist``; the estimators, the last-interaction
        DataFrame and (with virtual-packet logging) the vpacket tracker go on the state."""
        if self.montecarlo_configuration.ENABLE_FULL_RELATIVITY:
            raise NotImplementedError("Full relativity not supported for non-homology.")
        self.transport_state = transport_state
        cfg = self.montecarlo_configuration
        number_of_vpackets = cfg.NUMBER_OF_VPACKETS
        trackers = generate_tracker_last_interaction_list(len(transport_state.packet_collection.initial_nus))
        v_packets_energy_hist, vpacket_tracker, estimators_bulk, estimators_line = montecarlo_transport_with_vpackets(
            transport_state.packet_collection, transport_state.geometry_state_numba, 0.0,
            transport_state.opacity_state_numba, cfg, _value(self.spectrum_frequency_grid), trackers,
            number_of_vpackets, show_progress_bars=show_progress_bars, packet_propagation_function=None,
            engine=get_engine(self.device), sigma_thomson=self.sigma_thomson,
            luminosity_nu_start=self.luminosity_nu_start, luminosity_nu_end=self.luminosity_nu_end)
        transport_state.fused_packet_sums = montecarlo_transport_with_vpackets.last_fused
        transport_state.estimators_bulk = estimators_bulk
        transport_state.estimators_line = estimators_line
        if cfg.ENABLE_VPACKET_TRACKING and number_of_vpackets > 0:
            transport_state.vpacket_tracker = vpacket_tracker
        transport_state.tracker_full_df = None
        transport_state.tracker_last_interaction_df = trackers.to_df()
        transport_state.virt_logging = cfg.ENABLE_VPACKET_TRACKING
        return v_packets_energy_hist

    run_nonhomologous = run

    @classmethod
    def from_config(cls, config, packet_source, enable_virtual_packet_logging=False, device=0,
                    honor_disable_electron_scattering=False):
        """modes/nonhomologous/solver.py:271-358 (as MCTransportSolverB200.from_config, with the nonhomologous
        radiation-field solver)."""
        solver = super().from_config(config, packet_source, enable_virtual_packet_logging=enable_virtual_packet_logging,
                                     device=device, honor_disable_electron_scattering=honor_disable_electron_scattering)
        try:
            from tardis.transport.montecarlo.modes.nonhomologous.mc_rad_field_solver import (  # noqa: PLC0415
                MCRadiationFieldPropertiesSolver,
            )

            solver.radfield_prop_solver = MCRadiationFieldPropertiesSolver(config.plasma.w_epsilon)
        except Exception:  # not importable: the engine's own (same surface)
            solver.radfield_prop_solver = MCRadiationFieldPropertiesSolverB200Nonhomologous(config.plasma.w_epsilon, device=device)
        return solver
