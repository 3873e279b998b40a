"""ctypes declarations of the C-ABI in include/tardis_b200.h (field for field)."""
from __future__ import annotations

import ctypes as C
import os

from . import _build

_pd = C.POINTER(C.c_double)
_pi = C.POINTER(C.c_int64)

EXPORTED_SYMBOLS = [
    "tb200_create", "tb200_destroy", "tb200_last_error", "tb200_version", "tb200_set_model", "tb200_run",
    "tb200_upload_packets", "tb200_transport", "tb200_sync", "tb200_download", "tb200_estimator_buffer",
    "tb200_last_kernel_ms", "tb200_get_counters", "tb200_kernel_launches", "tb200_set_option",
    "tb200_create_packets", "tb200_download_packets", "tb200_get_estimator_layout", "tb200_solve_radiation_field",
    "tb200_set_atomic_data", "tb200_build_opacity", "tb200_download_opacity",
    "tb200_line_accumulators", "tb200_finalize_line_estimators", "tb200_run_resident", "tb200_solve_source_function",
    "tb200_formal_integral", "tb200_formal_integral_ms", "tb200_build_absorbing_markov", "tb200_download_absorbing_markov",
    "tb200_group_create", "tb200_group_destroy", "tb200_group_size", "tb200_group_member", "tb200_group_set_option",
    "tb200_group_set_model", "tb200_group_set_atomic_data", "tb200_group_build_opacity", "tb200_group_upload_packets",
    "tb200_group_create_packets", "tb200_group_run", "tb200_group_run_resident", "tb200_group_sync", "tb200_group_allreduce",
    "tb200_group_allreduce_ms", "tb200_group_formal_integral", "tb200_group_formal_integral_ms",
    "tb200_group_build_absorbing_markov", "tb200_set_plasma_data", "tb200_solve_plasma", "tb200_group_set_plasma_data",
    "tb200_group_solve_plasma",
]


class FormalIntegralParams(C.Structure):
    _fields_ = [
        ("inner_temperature", C.c_double),
        ("n_impact_parameters", C.c_int32), ("interpolate_shells", C.c_int32),
        ("att_S_ul", _pd), ("Jred_lu", _pd), ("Jblue_lu", _pd),
        ("electron_densities", _pd),
        ("sigma_thomson", C.c_double),
    ]


class SourceFunctionParams(C.Structure):
    _fields_ = [
        ("time_explosion", C.c_double), ("time_of_simulation", C.c_double),
        ("volume", _pd), ("wavelength_cm", _pd),
        ("lines_lower_level_idx", _pi), ("lines_upper_level_idx", _pi),
        ("n_levels", C.c_int64),
        ("c", C.c_double),
        ("max_iterations", C.c_int32),
        ("tolerance", C.c_double),
        ("j_blue_estimator", _pd), ("e_dot_lu_estimator", _pd),
    ]


class Model(C.Structure):
    _fields_ = [
        ("n_shells", C.c_int64), ("n_lines", C.c_int64),
        ("r_inner", _pd), ("r_outer", _pd), ("time_explosion", C.c_double),
        ("electron_density", _pd), ("line_list_nu", _pd),
        ("tau_sobolev", _pd), ("tau_line_stride", C.c_int64), ("tau_shell_stride", C.c_int64),
        ("n_transitions", C.c_int64), ("n_blocks", C.c_int64),
        ("transition_probabilities", _pd), ("tp_transition_stride", C.c_int64), ("tp_shell_stride", C.c_int64),
        ("line2macro_level_upper", _pi), ("macro_block_edge_index", _pi), ("transition_type", _pi),
        ("destination_level_id", _pi), ("transition_line_id", _pi),
        ("t_electrons", _pd), ("n_continua", C.c_int64), ("n_phot", C.c_int64),
        ("bf_threshold_list_nu", _pd), ("photo_ion_nu_threshold_mins", _pd), ("photo_ion_nu_threshold_maxs", _pd),
        ("photo_ion_block_references", _pi), ("chi_bf", _pd), ("x_sect", _pd), ("phot_nus", _pd),
        ("ff_opacity_factor", _pd), ("emissivities", _pd), ("photo_ion_activation_idx", _pi),
        ("n_activation", C.c_int64), ("k_packet_idx", C.c_int64), ("n_markov", C.c_int64),
        ("absorbing_markov_probabilities", _pd),
        ("v_inner", _pd), ("v_outer", _pd),
    ]


class Config(C.Structure):
    _fields_ = [
        ("enable_full_relativity", C.c_int32), ("line_interaction_type", C.c_int32),
        ("disable_line_scattering", C.c_int32), ("continuum_processes_enabled", C.c_int32),
        ("sigma_thomson", C.c_double), ("number_of_vpackets", C.c_int64),
        ("survival_probability", C.c_double), ("vpacket_tau_russian", C.c_double),
        ("vpacket_spawn_start_frequency", C.c_double), ("vpacket_spawn_end_frequency", C.c_double),
        ("spectrum_frequency_grid", _pd), ("n_grid", C.c_int64),
        ("luminosity_nu_start", C.c_double), ("luminosity_nu_end", C.c_double),
        ("nonhomologous", C.c_int32),
    ]


class PacketSource(C.Structure):
    """tb200_packet_source (device-side BlackBodySimpleSource, ...Relativistic and BlackBodyWeightedSource)"""
    _fields_ = [
        ("n_packets", C.c_int64), ("seed", C.c_uint64), ("radius", C.c_double), ("temperature", C.c_double),
        ("l_array", _pd), ("n_l", C.c_int64), ("max_seed_val", C.c_uint32), ("relativistic", C.c_int32), ("beta", C.c_double),
        ("weighted", C.c_int32),
    ]


LAYOUT_FIELDS = ("n_doubles", "n_shells", "n_lines", "line_pitch", "n_grid", "n_continua", "off_j", "off_nu_bar", "off_vhist",
                 "off_spectrum_emitted", "off_spectrum_reabsorbed", "off_luminosity", "off_ff_heating", "off_continuum",
                 "n_continuum_doubles", "off_j_blue", "off_edotlu")


class EstimatorLayout(C.Structure):
    """tb200_estimator_layout: where everything lies in the packed estimator buffer (offsets in doubles)"""
    _fields_ = [(n, C.c_int64) for n in LAYOUT_FIELDS]


class RadfieldParams(C.Structure):
    """tb200_radfield_params"""
    _fields_ = [
        ("time_explosion", C.c_double), ("time_of_simulation", C.c_double), ("volume", _pd), ("w_epsilon", C.c_double),
        ("detailed_optical_window", C.c_int32),
        ("t_radiative_estimator_constant", C.c_double), ("sigma_sb", C.c_double), ("c", C.c_double), ("h", C.c_double), ("k_b", C.c_double),
        ("j", _pd), ("nu_bar", _pd), ("j_blue", _pd),
        ("velocity_gradient", _pd),
    ]


_pu8 = C.POINTER(C.c_uint8)


class ContinuumRows(C.Structure):
    """tb200_continuum_rows"""
    _fields_ = [("n_transitions", C.c_int64), ("rate_key", _pi), ("energy", _pd), ("n_rate_rows", C.c_int64 * 6),
                ("n_cooling_rows", C.c_int64 * 3)]


class ContinuumRates(C.Structure):
    """tb200_continuum_rates"""
    _fields_ = [("rate", _pd * 6), ("cooling", _pd * 3), ("electron_densities", _pd), ("ff_cool_rate", _pd), ("fb_cool_rate", _pd),
                ("coll_exc_cool_rate", _pd), ("coll_ion_cool_rate", _pd), ("beta_sobolev", _pd), ("stimulated_emission_factor", _pd)]


class AtomicData(C.Structure):
    """tb200_atomic_data"""
    _fields_ = [
        ("n_lines", C.c_int64), ("n_levels", C.c_int64), ("lines_lower_level_index", _pi), ("lines_upper_level_index", _pi),
        ("g", _pd), ("metastability", _pu8), ("nlte_line", _pu8), ("wavelength_f_lu", _pd), ("f_lu", _pd), ("f_ul", _pd),
        ("energy_lower", _pd), ("energy_upper", _pd),
        ("sobolev_coefficient", C.c_double), ("c_einstein", C.c_double), ("c", C.c_double), ("h", C.c_double),
        ("continuum_rows", C.POINTER(ContinuumRows)),
    ]


class PlasmaState(C.Structure):
    """tb200_plasma_state"""
    _fields_ = [("level_number_density", _pd), ("time_explosion", C.c_double), ("j_blues", _pd), ("velocity_gradient", _pd),
                ("continuum", C.POINTER(ContinuumRates))]


class PlasmaData(C.Structure):
    """tb200_plasma_data"""
    _fields_ = [
        ("n_levels", C.c_int64), ("level_energy", _pd), ("level_ion", _pi), ("n_ions", C.c_int64), ("ion_atomic_number", _pi),
        ("ion_charge", _pi), ("ionization_energy", _pd), ("n_shells", C.c_int64), ("number_density", _pd),
        ("n_zeta_temperatures", C.c_int64), ("zeta_temperatures", _pd), ("zeta", _pd), ("chi_0", C.c_double),
        ("k_b", C.c_double), ("h", C.c_double), ("m_e", C.c_double), ("c", C.c_double),
    ]


class PlasmaParams(C.Structure):
    """tb200_plasma_params"""
    _fields_ = [
        ("t_radiative", _pd), ("dilution_factor", _pd), ("ionization", C.c_int32), ("excitation", C.c_int32),
        ("radiative_rates_type", C.c_int32), ("link_t_rad_t_electron", C.c_double), ("delta_treatment", C.c_double),
        ("departure_coefficient", C.c_double), ("ion_zero_threshold", C.c_double), ("electron_densities", _pd),
    ]


class MarkovInput(C.Structure):
    """tb200_markov_input"""
    _fields_ = [
        ("n_transitions", C.c_int64), ("transition_probabilities", _pd), ("tp_transition_stride", C.c_int64),
        ("tp_shell_stride", C.c_int64), ("source_level_idx", _pi), ("destination_level_idx", _pi), ("transition_type", _pi),
        ("n_states", C.c_int64),
    ]


class Packets(C.Structure):
    _fields_ = [
        ("n_packets", C.c_int64), ("initial_radii", _pd), ("initial_nus", _pd), ("initial_mus", _pd),
        ("initial_energies", _pd), ("packet_seeds", _pi),
    ]


COUNTER_FIELDS = ("n_line_steps", "n_boundary_events", "n_line_events", "n_escat_events", "n_rng_draws",
                  "n_macro_jumps", "n_macro_scanned", "n_vpackets", "n_vpacket_line_steps", "n_continuum_events",
                  "n_bf_estimator_updates", "n_search_probes")


class Counters(C.Structure):
    _fields_ = [(n, C.c_int64) for n in COUNTER_FIELDS]


class Outputs(C.Structure):
    _fields_ = [
        ("output_nus", _pd), ("output_energies", _pd), ("j", _pd), ("nu_bar", _pd), ("j_blue", _pd), ("edotlu", _pd),
        ("vhist", _pd),
        ("last_interaction_type", _pi), ("last_event_id", _pi), ("last_shell_id", _pi), ("last_line_absorb_id", _pi),
        ("last_line_emit_id", _pi),
        ("last_radius", _pd), ("last_before_nu", _pd), ("last_before_mu", _pd), ("last_before_energy", _pd),
        ("last_after_nu", _pd), ("last_after_mu", _pd), ("last_after_energy", _pd),
        ("events", C.c_void_p), ("event_counts", _pi), ("n_tracked_packets", C.c_int64), ("max_events_per_packet", C.c_int64),
        ("vlog_nus", _pd), ("vlog_energies", _pd), ("vlog_initial_mus", _pd), ("vlog_initial_rs", _pd),
        ("vlog_packet_index", _pi), ("vlog_capacity", C.c_int64), ("vlog_count", C.c_int64),
        ("photo_ion_estimator", _pd), ("stim_recomb_estimator", _pd), ("bf_heating_estimator", _pd),
        ("stim_recomb_cooling_estimator", _pd), ("ff_heating_estimator", _pd), ("photo_ion_estimator_statistics", _pi),
        ("spectrum_emitted", _pd), ("spectrum_reabsorbed", _pd), ("luminosity_sums", _pd),
        ("counters", Counters),
    ]


_lib = None


def load(build_if_missing: bool = True):
    """dlopen libtardis_b200.so (building it with nvcc first if it is missing or stale)."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB
    override = os.environ.get("TARDIS_B200_LIB")  # development only: A/B-test another build of the same ABI
    if override:
        path, build_if_missing = override, False
    if build_if_missing and (_build.is_stale()):
        _build.build()
    if not os.path.exists(path):
        raise ImportError(f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` (needs nvcc). "
                          "tardis_b200 has no CPU fallback.")
    lib = C.CDLL(path)
    missing = [name for name in EXPORTED_SYMBOLS if not hasattr(lib, name)]
    if missing:
        raise ImportError(f"{path} is stale: it does not export {missing}. Rebuild it: "
                          "`python -c 'import __graft_entry__ as g; g.build()'`.")
    E = C.c_void_p
    lib.tb200_create.argtypes = [C.c_int, C.POINTER(E)]
    lib.tb200_destroy.argtypes = [E]
    lib.tb200_destroy.restype = None
    lib.tb200_last_error.restype = C.c_char_p
    lib.tb200_version.restype = C.c_char_p
    lib.tb200_set_model.argtypes = [E, C.POINTER(Model), C.POINTER(Config)]
    lib.tb200_run.argtypes = [E, C.POINTER(Packets), C.POINTER(Outputs)]
    lib.tb200_upload_packets.argtypes = [E, C.POINTER(Packets)]
    lib.tb200_transport.argtypes = [E, C.c_int]
    lib.tb200_sync.argtypes = [E]
    lib.tb200_download.argtypes = [E, C.POINTER(Outputs)]
    lib.tb200_estimator_buffer.argtypes = [E, C.POINTER(C.c_void_p), C.POINTER(C.c_int64)]
    lib.tb200_last_kernel_ms.argtypes = [E, C.POINTER(C.c_double)]
    lib.tb200_get_counters.argtypes = [E, C.POINTER(Counters)]
    lib.tb200_kernel_launches.argtypes = [E]
    lib.tb200_kernel_launches.restype = C.c_int64
    lib.tb200_set_option.argtypes = [E, C.c_char_p, C.c_int64]
    lib.tb200_create_packets.argtypes = [E, C.POINTER(PacketSource)]
    lib.tb200_download_packets.argtypes = [E, _pd, _pd, _pd, _pd, _pi]
    lib.tb200_get_estimator_layout.argtypes = [E, C.POINTER(EstimatorLayout)]
    lib.tb200_solve_radiation_field.argtypes = [E, C.POINTER(RadfieldParams), _pd, _pd, _pd]
    lib.tb200_set_atomic_data.argtypes = [E, C.POINTER(AtomicData)]
    lib.tb200_build_opacity.argtypes = [E, C.POINTER(PlasmaState)]
    lib.tb200_download_opacity.argtypes = [E, _pd, _pd, _pd, _pd]
    lib.tb200_line_accumulators.argtypes = [E, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), _pd, _pd]
    lib.tb200_finalize_line_estimators.argtypes = [E]
    lib.tb200_run_resident.argtypes = [E, C.POINTER(Outputs)]
    lib.tb200_solve_source_function.argtypes = [E, C.POINTER(SourceFunctionParams), _pd, _pd, _pd, _pd, C.POINTER(C.c_int32)]
    lib.tb200_formal_integral.argtypes = [E, C.POINTER(FormalIntegralParams), _pd, C.c_int64, _pd, _pd]
    lib.tb200_formal_integral_ms.argtypes = [E, _pd, _pd]
    lib.tb200_build_absorbing_markov.argtypes = [E, C.POINTER(MarkovInput)]
    lib.tb200_download_absorbing_markov.argtypes = [E, _pd, _pd]
    lib.tb200_group_build_absorbing_markov.argtypes = [E, C.POINTER(MarkovInput)]
    lib.tb200_set_plasma_data.argtypes = [E, C.POINTER(PlasmaData)]
    lib.tb200_solve_plasma.argtypes = [E, C.POINTER(PlasmaParams), _pd, _pd, _pd, _pd, C.POINTER(C.c_int32)]
    lib.tb200_group_set_plasma_data.argtypes = [E, C.POINTER(PlasmaData)]
    lib.tb200_group_solve_plasma.argtypes = [E, C.POINTER(PlasmaParams), _pd, _pd, _pd, _pd, C.POINTER(C.c_int32)]
    lib.tb200_group_create.argtypes = [C.POINTER(C.c_int), C.c_int, C.POINTER(E)]
    lib.tb200_group_destroy.argtypes = [E]
    lib.tb200_group_destroy.restype = None
    lib.tb200_group_size.argtypes = [E]
    lib.tb200_group_member.argtypes = [E, C.c_int, C.POINTER(E)]
    lib.tb200_group_set_option.argtypes = [E, C.c_char_p, C.c_int64]
    lib.tb200_group_set_model.argtypes = [E, C.POINTER(Model), C.POINTER(Config)]
    lib.tb200_group_set_atomic_data.argtypes = [E, C.POINTER(AtomicData)]
    lib.tb200_group_build_opacity.argtypes = [E, C.POINTER(PlasmaState)]
    lib.tb200_group_upload_packets.argtypes = [E, C.POINTER(Packets)]
    lib.tb200_group_create_packets.argtypes = [E, C.POINTER(PacketSource)]
    lib.tb200_group_run.argtypes = [E, C.POINTER(Packets), C.POINTER(Outputs)]
    lib.tb200_group_run_resident.argtypes = [E, C.POINTER(Outputs)]
    lib.tb200_group_sync.argtypes = [E]
    lib.tb200_group_allreduce.argtypes = [E, C.POINTER(C.c_int)]
    lib.tb200_group_allreduce_ms.argtypes = [E, _pd]
    lib.tb200_group_formal_integral.argtypes = [E, C.POINTER(FormalIntegralParams), _pd, C.c_int64, _pd, _pd]
    lib.tb200_group_formal_integral_ms.argtypes = [E, _pd, _pd]
    for name in ("tb200_create", "tb200_set_model", "tb200_run", "tb200_upload_packets", "tb200_transport", "tb200_sync",
                 "tb200_download", "tb200_estimator_buffer", "tb200_last_kernel_ms", "tb200_get_counters", "tb200_set_option",
                 "tb200_create_packets", "tb200_download_packets", "tb200_get_estimator_layout", "tb200_solve_radiation_field",
                 "tb200_set_atomic_data", "tb200_build_opacity", "tb200_download_opacity", "tb200_line_accumulators",
                 "tb200_finalize_line_estimators", "tb200_run_resident",
                 "tb200_solve_source_function", "tb200_formal_integral", "tb200_formal_integral_ms",
                 "tb200_build_absorbing_markov", "tb200_download_absorbing_markov", "tb200_set_plasma_data", "tb200_solve_plasma",
                 *(n for n in EXPORTED_SYMBOLS if n.startswith("tb200_group_") and n != "tb200_group_destroy")):
        getattr(lib, name).restype = C.c_int
    _lib = lib
    return lib
