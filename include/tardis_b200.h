/*
 * tardis_b200.h -- C-ABI of the H100 (sm_90a) Monte Carlo packet-propagation engine.
 *
 * This is the drop-in boundary for ONE call of the reference (paths relative
 * to /root/reference/tardis/):
 *
 *   montecarlo_transport_with_vpackets(packet_collection, geometry_state_numba,
 *       time_explosion, opacity_state_numba, montecarlo_configuration,
 *       spectrum_frequency_grid, trackers, number_of_vpackets, show_progress_bars,
 *       packet_propagation_function)
 *     -> (v_packets_energy_hist, vpacket_tracker, estimators_bulk, estimators_line)
 *   transport/montecarlo/modes/montecarlo_transport.py:239-373,
 *   called from MCTransportSolverClassic.run_classic,
 *   transport/montecarlo/modes/classic/solver.py:223-234.
 *
 * Plain pointers and sizes only; all host arrays are caller-owned (NumPy
 * buffers in the Python shim), the library never frees or keeps them beyond
 * the call that receives them.  Device memory is library-owned and persists
 * across MC iterations.  Every function returns TB200_OK (0) or an error code;
 * tb200_last_error() gives the message.  One engine drives one GPU from one
 * host thread.  Multi-GPU from one process: an engine group (tb200_group_*,
 * end of this file) drives one engine per listed device and sums their
 * estimators itself.  Across processes or nodes: one engine per rank, packets
 * sharded by the caller, estimators summed through the device buffer exposed
 * by tb200_estimator_buffer() (see INTEGRATION.md).
 */
#ifndef TARDIS_B200_H
#define TARDIS_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TB200_OK 0
/* physics errors, same conditions under which the reference raises */
#define TB200_ERR_NU_DIFF 1      /* MonteCarloException("nu difference is less than 0.0"), transport/geometry/calculate_distances.py:106 */
#define TB200_ERR_MACRO_ATOM 2   /* MacroAtomError, transport/montecarlo/macro_atom.py:95 / interaction_event_callers.py:89-91 */
#define TB200_ERR_VPACKET_LOOP 3 /* virtual packet never leaves the grid (the reference would spin in virtual_packet.py:191-243) */
#define TB200_ERR_CONTINUUM 5    /* continuum tables inconsistent (index out of range; the reference would read out of bounds) */
#define TB200_ERR_PLASMA_IONIZATION 6 /* PlasmaIonizationError('n_electron just turned "nan" - aborting'), plasma/properties/ion_population.py:363-366;
                                         also the n_e fixed point not converged within its iteration cap (tb200_solve_plasma) */
/* host-side errors */
#define TB200_ERR_CUDA 100
#define TB200_ERR_INVALID 101
#define TB200_ERR_NO_MODEL 102

typedef struct tb200_engine tb200_engine;

/* Replaces NumbaHomologousRadial1DGeometry (model/geometry/radial1d_homologous.py:199-226)
 * + OpacityStateNumba (opacities/opacity_state_numba.py:13-72), classic-mode fields.
 * 2-D tables carry element strides so the reference's shell-sliced, non-contiguous
 * views (modes/classic/solver.py:132-134, opacity_state_numba.py:157-196) can be passed as they are. */
typedef struct {
    int64_t n_shells, n_lines;
    const double *r_inner, *r_outer; /* [S] cm */
    double time_explosion;           /* s */
    const double *electron_density;  /* [S] cm^-3 */
    const double *line_list_nu;      /* [L] Hz, non-increasing */
    const double *tau_sobolev;       /* element (line, shell) at [line*tau_line_stride + shell*tau_shell_stride]; NULL: built on
                                        the device by tb200_build_opacity (as is transition_probabilities when NULL) */
    int64_t tau_line_stride, tau_shell_stride;
    /* macro atom (1-element dummies for `scatter`, opacities/opacity_state.py:199-209) */
    int64_t n_transitions, n_blocks;
    const double *transition_probabilities; /* (transition, shell) at [t*tp_transition_stride + s*tp_shell_stride] */
    int64_t tp_transition_stride, tp_shell_stride;
    const int64_t *line2macro_level_upper; /* [L] */
    const int64_t *macro_block_edge_index; /* [n_blocks + 1] */
    const int64_t *transition_type;        /* [T] */
    const int64_t *destination_level_id;   /* [T] */
    const int64_t *transition_line_id;     /* [T] */
    /* Continuum (IIP mode) fields of OpacityStateNumbaIIP (opacities/opacity_state_numba_iip.py:8-125); read only when
     * config.continuum_processes_enabled.  All 2-D tables C-contiguous. */
    const double *t_electrons;                   /* [S] K */
    int64_t n_continua, n_phot;                  /* bound-free continua; total number of cross-section points */
    const double *bf_threshold_list_nu;          /* [n_continua] */
    const double *photo_ion_nu_threshold_mins;   /* [n_continua] */
    const double *photo_ion_nu_threshold_maxs;   /* [n_continua] */
    const int64_t *photo_ion_block_references;   /* [n_continua + 1] */
    const double *chi_bf;                        /* [n_phot, S] */
    const double *x_sect, *phot_nus;             /* [n_phot] */
    const double *ff_opacity_factor;             /* [S] */
    const double *emissivities;                  /* [n_phot, S] */
    const int64_t *photo_ion_activation_idx;     /* [n_activation] */
    int64_t n_activation, k_packet_idx;
    int64_t n_markov;                            /* absorbing_markov_probabilities is [S, n_markov, n_markov] */
    const double *absorbing_markov_probabilities;
    /* NumbaRadial1DGeometry (model/geometry/radial1d.py:320-375): shell-edge velocities, cm / s.  Read only when
     * config.nonhomologous; the engine computes velocity_gradient = (v_outer - v_inner) / (r_outer - r_inner) itself. */
    const double *v_inner, *v_outer;             /* [S] */
} tb200_model;

/* Replaces MonteCarloConfiguration (transport/montecarlo/configuration/base.py:11-49)
 * + the module constant SIGMA_THOMSON (configuration/constants.py:3) + spectrum_frequency_grid. */
typedef struct {
    int32_t enable_full_relativity;
    int32_t line_interaction_type;   /* 0 scatter, 1 downbranch, 2 macroatom (interaction_events.py:220-223) */
    int32_t disable_line_scattering;
    int32_t continuum_processes_enabled; /* IIP mode (modes/iip/packet_propagation.py:55-270): continuum opacities and
                                            events, full relativity forced, no virtual packets */
    double sigma_thomson;
    int64_t number_of_vpackets;
    double survival_probability;     /* SURVIVAL_PROBABILITY */
    double vpacket_tau_russian;      /* VPACKET_TAU_RUSSIAN */
    double vpacket_spawn_start_frequency, vpacket_spawn_end_frequency;
    const double *spectrum_frequency_grid; /* [n_grid] Hz, uniform spacing */
    int64_t n_grid;
    /* window of Simulation.iterate's calculate_filtered_luminosity (simulation/base.py:455-466, spectrum/luminosity.py:5-29;
     * config supernova.luminosity_wavelength_start/end converted to Hz), strict on both sides.  0 / +inf = everything. */
    double luminosity_nu_start, luminosity_nu_end;
    /* 1: the nonhomologous transport mode (transport/montecarlo/modes/nonhomologous/): piecewise-linear velocity law from
     * model.v_inner / v_outer, line distances from the quartic of calculate_distance_line_nonhomologous, two-way line scan;
     * time_explosion is not used (0 is accepted).  Refused with full relativity ("Full relativity not supported for
     * non-homology."), with continuum processes and without v_inner / v_outer.  Runs its own kernel whatever the
     * options "algorithm" / "pooled" say; tb200_line_accumulators is refused and engine groups sum in f64 (exact = 0). */
    int32_t nonhomologous;
} tb200_config;

/* Replaces PacketCollection inputs (transport/montecarlo/packets/packet_collections.py:14-76). */
typedef struct {
    int64_t n_packets;
    const double *initial_radii, *initial_nus, *initial_mus, *initial_energies; /* [N] */
    const int64_t *packet_seeds; /* [N], low 32 bits used (np.random.seed) */
} tb200_packets;

/* Integer work counters; functions of the seeds only, so the oracle reports the same numbers. */
typedef struct {
    int64_t n_line_steps, n_boundary_events, n_line_events, n_escat_events, n_rng_draws;
    int64_t n_macro_jumps, n_macro_scanned, n_vpackets, n_vpacket_line_steps;
    int64_t n_continuum_events, n_bf_estimator_updates;
    int64_t n_search_probes; /* engine-only: evaluations of the trace stopping predicate by the "jump" algorithm */
} tb200_counters;

/* One row of the reference's TrackerFull (packets/trackers/tracker_full.py:19-110). */
typedef struct {
    int64_t packet_id, interaction_type, status, before_shell_id, after_shell_id, line_absorb_id, line_emit_id;
    double radius, before_nu, before_mu, before_energy, after_nu, after_mu, after_energy;
} tb200_event;

/* Host destinations; any pointer may be NULL to skip that output. */
typedef struct {
    double *output_nus, *output_energies; /* [N]  PacketCollection.output_* (sign convention modes/montecarlo_transport.py:85-90) */
    double *j, *nu_bar;                   /* [S]  EstimatorsBulk (estimators/estimators_bulk.py:15-104) */
    double *j_blue, *edotlu;              /* [L,S] C-order  EstimatorsLine (estimators/estimators_line.py:15-112) */
    double *vhist;                        /* [n_grid]  v_packets_energy_hist */
    /* TrackerLastInteraction columns (packets/trackers/tracker_last_interaction_util.py:33-134); all [N] */
    int64_t *last_interaction_type, *last_event_id, *last_shell_id, *last_line_absorb_id, *last_line_emit_id;
    double *last_radius, *last_before_nu, *last_before_mu, *last_before_energy;
    double *last_after_nu, *last_after_mu, *last_after_energy;
    /* TrackerFull rows for packets [0, n_tracked_packets) */
    tb200_event *events;   /* [n_tracked_packets * max_events_per_packet] */
    int64_t *event_counts; /* [n_tracked_packets] (may exceed max_events_per_packet: rows beyond the cap are dropped) */
    int64_t n_tracked_packets, max_events_per_packet;
    /* virtual packet log (spectrum.virtual.virtual_packet_logging), unordered across packets */
    double *vlog_nus, *vlog_energies, *vlog_initial_mus, *vlog_initial_rs;
    int64_t *vlog_packet_index;
    int64_t vlog_capacity, vlog_count;
    /* EstimatorsContinuum (estimators/estimators_continuum.py:15-175): [n_continua, S] C-order, ff_heating [S] */
    double *photo_ion_estimator, *stim_recomb_estimator, *bf_heating_estimator, *stim_recomb_cooling_estimator;
    double *ff_heating_estimator;
    int64_t *photo_ion_estimator_statistics;
    /* Fused spectrum (SURVEY.md §8f rank 2): energy histograms of the emitted / reabsorbed packets on the spectrum
     * frequency grid, [n_grid - 1] bins each, with numpy.histogram's bin rule (last bin closed).  Multiply by
     * 1 / time_of_simulation to get SpectrumSolver.montecarlo_emitted_luminosity (tardis/spectrum/base.py:151-159). */
    double *spectrum_emitted, *spectrum_reabsorbed;
    /* [4] energy sums of the finished packets: {emitted, emitted inside the luminosity window, reabsorbed, reabsorbed inside
     * the window}; x 1 / time_of_simulation = the emitted_luminosity / reabsorbed_luminosity of Simulation.iterate */
    double *luminosity_sums;
    tb200_counters counters;
} tb200_outputs;

/* ---- lifetime ---- */
int tb200_create(int device_id, tb200_engine **engine);
void tb200_destroy(tb200_engine *engine);
const char *tb200_last_error(void);
const char *tb200_version(void);

/* ---- per-iteration table upload: geometry_state.to_numba() + opacity_state.to_numba()
 *      (modes/classic/solver.py:126-134) + configuration_initialize (configuration/base.py:52-78) ---- */
int tb200_set_model(tb200_engine *engine, const tb200_model *model, const tb200_config *config);

/* ---- the reference-facing call: host packets in, host results out (H2D, kernels, D2H). ---- */
int tb200_run(tb200_engine *engine, const tb200_packets *packets, tb200_outputs *outputs);

/* The same pipeline for packets that already lie in HBM (tb200_upload_packets, or tb200_create_packets -- the device-side
 * BlackBodySimpleSource): nothing goes up, the per-packet outputs of packet range c-1 travel back while range c computes. */
int tb200_run_resident(tb200_engine *engine, tb200_outputs *outputs);

/* ---- the same work as separate stages, for callers that keep data resident in HBM ---- */
int tb200_upload_packets(tb200_engine *engine, const tb200_packets *packets); /* H2D (each transport expands the seeds) */

/* ---- device-side packet source (SURVEY.md §8f rank 1): the packets never exist on the host ----
 * Fills the engine's resident packet arrays with what BlackBodySimpleSource.create_packets(no_of_packets, seed_offset)
 * returns (tardis/transport/montecarlo/packet_source/base.py:195-253, black_body.py:122-220) for
 * np.random.default_rng(seed), seed = base_seed + seed_offset: seeds = rng.choice(2**32 - 1, N), nus by the
 * Carter-Cashwell sampler from rng.random((5, N)), mus = sqrt(rng.random(N)), radii = radius, energies = 1 / N.
 * Integer outputs and mus / radii / energies are bit-identical to numpy's; nus to one ulp of `log`.
 * l_array = cumsum(arange(1, l_samples) ** -4.0) is supplied by the caller (so that it carries numpy's own pow).
 * After this call tb200_transport / tb200_download work as after tb200_upload_packets. */
typedef struct {
    int64_t n_packets;
    uint64_t seed;           /* base_seed + seed_offset */
    double radius;           /* cm: r_inner[0] */
    double temperature;      /* K */
    const double *l_array;   /* [n_l] */
    int64_t n_l;
    uint32_t max_seed_val;   /* population of rng.choice: BasePacketSource.MAX_SEED_VAL = 2**32 - 1 (0 = that default) */
    /* BlackBodySimpleSourceRelativistic (packet_source/black_body_relativistic.py:92-177; the continuum / full-relativity
     * modes use it): beta = (radius / time_explosion) / c; mus = -beta + sqrt(beta^2 + 2 beta z + z), energies =
     * 1 / N * (2 beta + 1) / (1 - beta^2) / gamma.  relativistic = 0: the plain source, beta ignored. */
    int32_t relativistic;
    double beta;
    /* BlackBodyWeightedSource (packet_source/black_body_weighted.py:9-108): the stream after the seeds is 5 N doubles for
     * Carter-Cashwell nus that only give their min and max, then nus = rng.uniform(min, max, N) (= min + (max - min) *
     * rng.random()), then mus = sqrt(rng.random(N)); energies = I / I.sum() with I = intensity_black_body(nus, T)
     * (util/base.py:279-302) and the sum in numpy's pairwise order.  Seeds, radii and mus are bit-identical to numpy's;
     * nus and energies differ from numpy's by the ulps of log, pow and exp (INTEGRATION.md gives the measured bounds).
     * Refused together with relativistic (the reference has no such source) and for n_packets = 0 (numpy raises on the
     * zero-size min).  weighted = 0: the sources above. */
    int32_t weighted;
} tb200_packet_source;
int tb200_create_packets(tb200_engine *engine, const tb200_packet_source *source);
/* resident input arrays -> host (diagnostics / tests / callers that want the PacketCollection); any pointer may be NULL */
int tb200_download_packets(tb200_engine *engine, double *radii, double *nus, double *mus, double *energies, int64_t *seeds);
int tb200_transport(tb200_engine *engine, int zero_estimators);               /* the propagation kernel, asynchronous */
int tb200_sync(tb200_engine *engine);                                         /* wait, then report physics errors */
int tb200_download(tb200_engine *engine, tb200_outputs *outputs);             /* D2H (estimators transposed to [L,S]) */

/* Packed device buffer of everything that is summed over packets (all float64; offsets in doubles):
 *   [ j(S) | nu_bar(S) | vhist(n_grid) | spectrum_emitted(n_grid-1) | spectrum_reabsorbed(n_grid-1) | luminosity sums (4)
 *     | continuum mode only: ff_heating(S), continuum estimator block | pad to 32 | j_blue(S x line_pitch, shell-major)
 *     | edotlu(S x line_pitch) ].
 * The exact offsets of the current model are reported by tb200_get_estimator_layout -- slice by them, not by this comment.
 * One all-reduce over the buffer (ncclAllReduce sum f64 / torch.distributed.all_reduce on a tensor aliasing the pointer)
 * is the only collective of a multi-GPU iteration.  The pointer is valid until the next tb200_set_model (which may
 * reallocate it): fetch it again after every tb200_set_model. */
typedef struct {
    int64_t n_doubles;                 /* length of the buffer */
    int64_t n_shells, n_lines, line_pitch, n_grid, n_continua;
    int64_t off_j, off_nu_bar, off_vhist, off_spectrum_emitted, off_spectrum_reabsorbed, off_luminosity;
    int64_t off_ff_heating, off_continuum, n_continuum_doubles; /* -1 / 0 outside continuum mode */
    int64_t off_j_blue, off_edotlu;    /* element (shell, line) at off + shell * line_pitch + line */
} tb200_estimator_layout;
int tb200_estimator_buffer(tb200_engine *engine, void **device_ptr, int64_t *n_doubles);
int tb200_get_estimator_layout(tb200_engine *engine, tb200_estimator_layout *layout);

/* ---- exact line estimators across GPUs ----
 * With algorithm = 1 (jump) J_blue and Edotlu are accumulated as 128-bit fixed-point difference arrays of 64-bit integer
 * words ([n_shells][line_pitch + 1][4]); tb200_transport turns them into the doubles of the estimator buffer at its end.
 * Integer sums do not depend on the order of the addends, so a multi-GPU iteration that all-reduces THESE words
 * (ncclAllReduce sum int64 / torch.distributed.all_reduce on an int64 tensor aliasing the pointer) and then calls
 * tb200_finalize_line_estimators gets J_blue and Edotlu bit-identical on every rank and bit-identical to a single-GPU run
 * over the same packets, whatever the number of GPUs -- the reference's prange sum (modes/montecarlo_transport.py:239-349)
 * has no such property.  Every rank must hold the same scales (they follow from the packets' typical energy and the model's
 * typical frequency); the caller compares them and falls back to the f64 all-reduce of the estimator buffer if they differ.
 * The f64 all-reduce of the remaining estimators then covers [0, off_j_blue) of the estimator buffer only. */
int tb200_line_accumulators(tb200_engine *engine, void **device_ptr, int64_t *n_words, double *scale_j_blue, double *scale_edotlu);
int tb200_finalize_line_estimators(tb200_engine *engine);

/* ---- estimator -> radiation field solve on the device (SURVEY.md §8f rank 4) ----
 * Replaces MCRadiationFieldPropertiesSolver.solve (transport/montecarlo/estimators/mc_rad_field_solver.py:37-144), which
 * Simulation.advance_state calls right after the MC iteration (simulation/base.py:281-288): T_rad and W per shell from
 * J / nu_bar, and the normalised J_blue table with its zero cells filled by w_epsilon x the dilute Planck intensity.
 * With j == NULL the estimators of the engine's last transport are used where they lie in HBM (after the caller's
 * all-reduce in a multi-GPU run); otherwise the given host arrays are uploaded first.  The results also stay resident. */
typedef struct {
    double time_explosion, time_of_simulation;       /* s */
    const double *volume;                            /* [S] cm^3: geometry_state_numba.volume */
    double w_epsilon;                                /* MCRadiationFieldPropertiesSolver.w_epsilon */
    int32_t detailed_optical_window;                 /* keep the estimated J_blue only inside (2500, 10000) Angstrom */
    /* constants exactly as the reference's module computes them (mc_rad_field_solver.py:20-30, util/base.py:21-23) */
    double t_radiative_estimator_constant, sigma_sb, c, h, k_b;
    const double *j, *nu_bar;                        /* [S], or NULL = resident estimators */
    const double *j_blue;                            /* [L,S] C-order (with j) */
    /* [S] or NULL.  The nonhomologous mode's solver (modes/nonhomologous/mc_rad_field_solver.py:35-131): J_blue is normalised
     * by (c / velocity_gradient) / ((4 pi t_sim) V) instead of c t_exp / (4 pi t_sim V), and there is no optical window.
     * Required (and only accepted) when the model was set with config.nonhomologous = 1. */
    const double *velocity_gradient;
} tb200_radfield_params;
int tb200_solve_radiation_field(tb200_engine *engine, const tb200_radfield_params *params, double *t_radiative /* [S] */,
                                double *dilution_factor /* [S] */, double *j_blues /* [L,S] C-order, or NULL */);

/* ---- formal-integral source function on the device (SURVEY.md §8f rank 4) ----
 * Replaces SourceFunctionSolver.solve (spectrum/formal_integral/source_function.py:27-358), which FormalIntegralSolver runs on
 * the host after the last Monte Carlo iteration: e_dot_u (group-by over the lines of every upper level), for macroatom the
 * per-shell system (I - Q)^T C = e_dot_u -- scipy spsolve there, the fixed point C <- e_dot_u + Q^T C here, iterated until
 * max |change| <= tolerance x max |C| in every shell --, att_S_ul, Jblue_lu and Jred_lu [L,S].  Reads tau_sobolev and the
 * line estimators where they lie in HBM (after the caller's all-reduce in a multi-GPU run) and the NORMALISED transition
 * probabilities, which the engine keeps only with the option keep_opacity_tables = 1 set before tb200_set_model /
 * tb200_build_opacity (the transport kernels read running sums).  Level indices are rows of MacroAtomState.references_index.
 * Only the bound-bound macro atom (row types -1 / 0 / 1); every line needs its emission row, as in the reference. */
typedef struct {
    double time_explosion, time_of_simulation;       /* s */
    const double *volume;                            /* [S] cm^3 */
    const double *wavelength_cm;                     /* [L] atom_data.lines.wavelength_cm */
    const int64_t *lines_lower_level_idx, *lines_upper_level_idx; /* [L] */
    int64_t n_levels;                                /* len(macro_atom_state.references_index) */
    double c;                                        /* const.c.cgs */
    int32_t max_iterations;                          /* 0 = 100000 */
    double tolerance;                                /* 0 = 1e-15 */
    const double *j_blue_estimator, *e_dot_lu_estimator; /* [L,S] C-order, or both NULL = the resident estimators */
} tb200_source_function_params;
int tb200_solve_source_function(tb200_engine *engine, const tb200_source_function_params *params, double *att_S_ul /* [L,S] or NULL */,
                                double *Jred_lu /* [L,S] or NULL */, double *Jblue_lu /* [L,S] or NULL */,
                                double *e_dot_u /* [n_levels,S] or NULL: C of every level */, int32_t *iterations /* or NULL */);

/* ---- formal integral on the device (SURVEY.md §8f rank 4: "the reference's Numba-CUDA formal integral ... beaten in place") ----
 * Replaces what FormalIntegralSolver.solve does after the source function (spectrum/formal_integral/formal_integral_solver.py:208-285):
 * interpolate_integrator_quantities (:305-430, scipy interp1d over the shell mid-points: nearest for tau_sobolev and the electron
 * densities, linear with extrapolation and a clip at 0 for att_S_ul / Jred_lu / Jblue_lu) and the integrator itself --
 * numba_formal_integral (formal_integral_numba.py:377-567) or its Numba-CUDA twin cuda_formal_integral
 * (formal_integral_cuda.py:272-621).  Reads tau_sobolev, the line list, the geometry and the electron densities of the resident
 * model and, by default, the att_S_ul / Jred_lu / Jblue_lu tables tb200_solve_source_function left in HBM; the interpolated
 * [L, S2] tables exist only on the device, as one 32-byte cell per (shell, line).  One warp integrates 32 neighbouring impact
 * parameters of one frequency in a single sweep over the line list; every ray performs the reference's operations in the
 * reference's order.  luminosity_densities[k] = 8 pi^2 trapezoid(I_nu_p[k, :], dx = r_max / n_impact_parameters) -- multiply by the
 * frequency step for the luminosity, as the reference does (:281-284).
 * Constants: C_INV, KB_CGS, H_CGS of spectrum/formal_integral/base.py:12-14 are compiled in; sigma_thomson defaults to
 * transport/montecarlo/configuration/constants.py:3.  Not for the continuum mode, not for line_interaction_type scatter
 * (check_formal_integral_requirements, base.py:26-83).  Rays whose window reaches beyond the reddest line: see
 * tardis_b200/csrc/formal_integral.cuh (the reference reads behind its arrays there). */
typedef struct {
    double inner_temperature;            /* simulation_state.t_inner [K] */
    int32_t n_impact_parameters;         /* FormalIntegralSolver.points (>= 2) */
    int32_t interpolate_shells;          /* > 1: number of radii of the linspace (that many - 1 shells); 0: max(2 S, 80); < 0: the model's shells */
    const double *att_S_ul, *Jred_lu, *Jblue_lu;  /* [L,S] C-order, or all NULL = the tables of the last tb200_solve_source_function */
    const double *electron_densities;    /* [S], or NULL = the model's */
    double sigma_thomson;                /* 0 = 6.652458734e-25 */
} tb200_formal_integral_params;
int tb200_formal_integral(tb200_engine *engine, const tb200_formal_integral_params *params, const double *frequencies /* [n] Hz */,
                          int64_t n_frequencies, double *luminosity_densities /* [n] erg / s / Hz */,
                          double *intensities_nu_p /* [n, n_impact_parameters] (each already times its impact parameter), or NULL */);
/* CUDA-event times of the last tb200_formal_integral: building the cells (interpolation), the rays + trapezoid */
int tb200_formal_integral_ms(tb200_engine *engine, double *interpolation_ms, double *integral_ms);

/* ---- opacity build on the device (SURVEY.md §8f rank 3) ----
 * Replaces, per iteration, StimulatedEmissionFactor.calculate (plasma/properties/radiative_properties.py:66-116),
 * calculate_sobolev_line_opacity / numba_calculate_beta_sobolev (opacities/tau_sobolev.py:21-88), the macro-atom
 * probabilities of BoundBoundMacroAtomSolver._solve_next_macroatom_iteration (opacities/macro_atom/macroatom_solver.py:491-585,
 * macroatom_line_transitions.py) and the [L,S] / [T,S] host tables of OpacityState.to_numba (opacities/opacity_state.py:157-342).
 * Usage: tb200_set_model with tau_sobolev == NULL (and transition_probabilities == NULL) uploads everything else and
 * leaves the opacity tables pending; tb200_set_atomic_data once; then every iteration tb200_build_opacity fills the
 * tables in HBM (shell-major, with the prefix sums / running sums / guide tables the kernels read) from the level
 * populations and from J_blue -- the copy tb200_solve_radiation_field left resident, or a host array. */
/* The continuum mode's static row map (given once, with the atomic data): for every macro-atom row, which row of which
 * per-iteration table of tb200_continuum_rates it reads, and its energy factor, resolved on the host exactly as
 * ContinuumMacroAtomSolver._solve_next_macroatom_iteration (opacities/macro_atom/macroatom_solver.py:1533-1631) looks them
 * up: by label (.loc) for PHOTOIONIZATION_INTERNAL (2) / PHOTO_RECOMB_INTERNAL (3), by collision_key_idx (.iloc) for the
 * collisional rows (11, 5, 4, 6, 7, 14), by position inside the type for PHOTO_RECOMB_EMISSION (-7) and the cooling rows
 * (-20, 21, 22; normalize_cooling_block_by_rate_fractions, :1817-1833).  The map belongs to the model current when it is
 * given: tb200_set_model discards it, and the continuum build refuses to run until tb200_set_atomic_data gives it again.  The table follows from the row's transition_type
 * (the model's): 2 -> rate[0], 3 / -7 -> rate[1], 11 / 5 -> rate[2], 4 -> rate[3], 6 -> rate[4], 7 / 14 -> rate[5],
 * -20 -> cooling[0], 21 -> cooling[1], 22 -> cooling[2]; line rows (-1 / 0 / 1) and FF_COOLING (-21) read none.  Rows of
 * any other type are refused.  tardis_b200.macro_atom derives the map from the reference's own metadata. */
typedef struct {
    int64_t n_transitions;                   /* T: must equal the model's */
    const int64_t *rate_key;                 /* [T] row of the row's table (not read for line and free-free rows) */
    const double *energy;                    /* [T] erg: the energy factor of rows 2, 3, -7, 11, 5, 4, 6, 7, 14 (level energy,
                                                delta_E_yg or ionization energy difference, as the reference picks it) */
    int64_t n_rate_rows[6];                  /* heights of tb200_continuum_rates.rate[k] */
    int64_t n_cooling_rows[3];               /* heights of tb200_continuum_rates.cooling[k] */
} tb200_continuum_rows;
/* The continuum mode's per-iteration inputs of the macro atom's rows (arguments of ContinuumMacroAtomSolver.solve,
 * macroatom_solver.py:861-882).  Row (key, shell) of every table at [key * S + shell]. */
typedef struct {
    /* [n_rate_rows[k], S]: stim_recomb_corrected_photoionization_rate_coeff, spontaneous_recombination_coeff, coll_deexc_coeff,
     * coll_exc_coeff, coll_ion_coeff, coll_recomb_coeff.  Unnormalised rows: 2 / 3 / -7: rate * energy
     * (macroatom_continuum_transitions.py:29,103,178); 11 / 5 / 4 / 6 / 7 / 14: (rate * n_e) * energy (:343,430,514,599,682,763) */
    const double *rate[6];
    /* [n_cooling_rows[k], S]: fb_cool_probs_arr.T, coll_exc_cool_arr.T, coll_ion_cool_arr.T; row = cool_rate[s] * cooling[k][key, s] */
    const double *cooling[3];
    const double *electron_densities;        /* [S] */
    const double *ff_cool_rate, *fb_cool_rate, *coll_exc_cool_rate, *coll_ion_cool_rate; /* [S]; FF_COOLING rows = ff_cool_rate */
    /* [L,S] C-order, both or neither: the beta_Sobolev and stimulated-emission factor the line rows read, as
     * _solve_next_macroatom_iteration receives them (macroatom_solver.py:1358-1378).  Given, tb200_plasma_state's
     * level_number_density must be NULL and tau is not rebuilt: the model needs its tau_sobolev from tb200_set_model. */
    const double *beta_sobolev, *stimulated_emission_factor;
} tb200_continuum_rates;
typedef struct {
    int64_t n_lines, n_levels;
    const int64_t *lines_lower_level_index, *lines_upper_level_index; /* [L] rows of the level arrays */
    const double *g;                         /* [n_levels] statistical weights */
    const uint8_t *metastability;            /* [n_levels] */
    const uint8_t *nlte_line;                /* [L] line belongs to an NLTE species (radiative_properties.py:103-115), or NULL */
    const double *wavelength_f_lu;           /* [L] lines.wavelength_cm * lines.f_lu (tau_sobolev.py:56) */
    const double *f_lu, *f_ul;               /* [L] */
    const double *energy_lower, *energy_upper; /* [L] erg: levels.energy of the line's lower / upper level */
    /* constants as the reference's modules compute them (tau_sobolev.py:9-18, macroatom_line_transitions.py:7-11) */
    double sobolev_coefficient, c_einstein, c, h;
    /* Continuum mode (config.continuum_processes_enabled): required there, refused on any other model.  Checked (types,
     * keys against the table heights, T) before anything is allocated. */
    const tb200_continuum_rows *continuum_rows;
} tb200_atomic_data;
typedef struct {
    const double *level_number_density;      /* [n_levels, S] C-order (NULL with tb200_continuum_rates.beta_sobolev); NULL outside
                                                the continuum mode: the populations of the last tb200_solve_plasma since
                                                tb200_set_model (refused when there are none) */
    double time_explosion;                   /* s (not read in the nonhomologous mode) */
    const double *j_blues;                   /* [L,S] C-order, or NULL = the table tb200_solve_radiation_field left in HBM
                                                (only read by the macro atom's internal-up rows) */
    /* Nonhomologous mode (config.nonhomologous): required, and refused on a homologous model.  The active shells'
     * dv/dr; tau = lambda f_lu COEFF / velocity_gradient * stim * n_lower (modes/nonhomologous/tau_sobolev.py:55-61)
     * instead of ... * time_explosion * ...  A shell with velocity_gradient < 0 has tau < 0 (and beta > 1), as in the
     * reference; velocity_gradient == 0 is the reference's "Some tau_sobolevs are nan, inf, -inf" error. */
    const double *velocity_gradient;         /* [S], 1/s */
    /* Continuum mode: required there, refused on any other model.  tau / beta / stim are built as in the homologous mode;
     * then every row of the macro atom (line rows as above, continuum rows from these tables and the row map of
     * tb200_set_atomic_data) and their normalisation (macroatom_solver.py:709-739: pandas' Kahan group sum per source
     * block, NaN addends skipped, then p / sum with NaN -> 0).  The normalised table stays in HBM for
     * tb200_build_absorbing_markov with transition_probabilities == NULL; until that runs, transport refuses to run. */
    const tb200_continuum_rates *continuum;
} tb200_plasma_state;
int tb200_set_atomic_data(tb200_engine *engine, const tb200_atomic_data *atomic);
int tb200_build_opacity(tb200_engine *engine, const tb200_plasma_state *plasma);
/* the tables as the reference would hold them on the host (tests / callers that want them); any pointer may be NULL.
 * transition_probabilities needs the option "keep_opacity_tables" = 1 (the kernels turn the table into running sums in place).
 * In the continuum mode it is the normalised table of the last tb200_build_opacity, refused if that build kept none (the
 * deactivation table is tb200_download_absorbing_markov's). */
int tb200_download_opacity(tb200_engine *engine, double *tau_sobolev /* [L,S] */, double *beta_sobolev /* [L,S] */,
                           double *stimulated_emission_factor /* [L,S] */, double *transition_probabilities /* [T,S] */);

/* ---- the classic plasma on the device ----
 * Replaces the plasma update of Simulation.advance_state (simulation/base.py:363-415) for the graphs without NLTE, helium NLTE
 * or continuum-interaction species: ionization nebular | lte, excitation dilute-lte | lte, radiative_rates_type
 * dilute-blackbody | blackbody | detailed.  The chain (plasma/properties/general.py:20-121, partition_function.py:32-353,
 * ion_population.py:37-390, level_population.py:13-70) and its layout: tardis_b200/csrc/plasma.cuh.
 * Usage: tb200_set_plasma_data once, after tb200_set_atomic_data (g and metastability come from there, same level rows);
 * then every iteration, after tb200_set_model (which uploads the host's electron densities), tb200_solve_plasma with the
 * damped T_rad and W, and tb200_build_opacity with level_number_density == NULL.
 * tb200_set_plasma_data refuses, before anything is allocated: levels not grouped by ion (level_ion non-decreasing, every
 * ion with a level), ions not grouped by element in ascending atomic number with charges 0, 1, 2, ... from 0, an element
 * with a single ion (the reference's Phi blocks would misalign), an ion of charge >= 1 without an ionisation energy, a zeta
 * grid that is not strictly ascending or has fewer than 2 points, and the continuum mode (its plasma is the IIP one). */
typedef struct {
    int64_t n_levels;                 /* must equal tb200_atomic_data.n_levels */
    const double *level_energy;       /* [n_levels] erg: levels.energy (the excitation energy) */
    const int64_t *level_ion;         /* [n_levels] row of the level's ion in the ion table */
    int64_t n_ions;                   /* the rows of the partition function: (atomic_number, ion_number) of the levels */
    const int64_t *ion_atomic_number, *ion_charge; /* [n_ions] */
    const double *ionization_energy;  /* [n_ions] erg: ionization_data of (Z, charge), the energy into this ion (charge 0: not read) */
    int64_t n_shells;                 /* must equal the model's */
    const double *number_density;     /* [n_elements, S] C-order, elements in the order of the ion table */
    int64_t n_zeta_temperatures;      /* 0: no zeta table (nebular ionisation is then refused) */
    const double *zeta_temperatures;  /* [n_zeta_temperatures] K, strictly ascending */
    const double *zeta;               /* [n_ions, n_zeta_temperatures] C-order (rows of charge 0 not read) */
    double chi_0;                     /* RadiationFieldCorrection's chi_0: 1.9020591570241798e-11 (Ca II), or a species' energy */
    double k_b, h, m_e, c;            /* cgs, as tardis.constants gives them */
} tb200_plasma_data;
int tb200_set_plasma_data(tb200_engine *engine, const tb200_plasma_data *data);
/* One plasma update from T_rad and W [S] (damped on the host, as in the reference).  Effects: the level populations stay in
 * HBM for tb200_build_opacity(level_number_density == NULL); n_e becomes the model's resident electron densities (transport's
 * chi_e, the formal integral); for dilute-blackbody / blackbody the J_blue table tb200_build_opacity(j_blues == NULL) reads
 * is overwritten with W B_nu(T_rad) (W = 1 for blackbody); detailed keeps the table tb200_solve_radiation_field left.
 * The n_e fixed point runs on the device in one launch and stops after 1000 iterations with TB200_ERR_PLASMA_IONIZATION
 * (the reference's loop is unbounded); a NaN n_e gives the same code.  After an error the model's n_e and the J_blue table are
 * unchanged and no level populations are resident.
 * Outputs may be NULL: electron_densities [S], ion_number_density [n_ions, S], level_number_density [n_levels, S],
 * j_blues [L, S] (the table build_opacity will read; refused if none is resident), n_e iterations (0 with fixed n_e). */
typedef struct {
    const double *t_radiative, *dilution_factor; /* [S] */
    int32_t ionization;               /* 0 nebular, 1 lte */
    int32_t excitation;               /* 0 dilute-lte, 1 lte */
    int32_t radiative_rates_type;     /* 0 dilute-blackbody, 1 blackbody, 2 detailed */
    double link_t_rad_t_electron;     /* T_e = link * T_rad (config plasma.link_t_rad_t_electron, 0.9) */
    double delta_treatment;           /* NaN: delta computed; otherwise delta = this constant */
    double departure_coefficient;     /* NaN: 1 / W */
    double ion_zero_threshold;        /* populations below are set to 0 (1e-20) */
    const double *electron_densities; /* [S] fixed n_e (no fixed point), or NULL */
} tb200_plasma_params;
int tb200_solve_plasma(tb200_engine *engine, const tb200_plasma_params *params, double *electron_densities, double *ion_number_density,
                       double *level_number_density, double *j_blues, int32_t *iterations);

/* ---- the continuum mode's macro atom on the device ----
 * Replaces steps 2-3 of ContinuumMacroAtomSolver._solve_next_macroatom_iteration (opacities/macro_atom/macroatom_solver.py:1648-1662):
 * create_absorbing_probs (opacities/macro_atom/absorbing_markov_chain.py:19-134), which solves (I - Q) X = diag(1 - rowsum Q)
 * per shell with scipy's splu, and the normalisation of the deactivating rows (internal rows zeroed; pandas' Kahan group sum
 * per source block, NaN -> 0).  Usage: tb200_set_model in continuum mode with absorbing_markov_probabilities == NULL (or
 * transition_probabilities == NULL) leaves the macro atom pending -- transport refuses to run -- and then every iteration
 * tb200_build_absorbing_markov writes X (as the running sums the kernels read) and the normalised deactivation table into
 * HBM.  Rows must be grouped by source as the model's macro_block_edge_index says (block b holds the rows of state b).
 * Refused, before anything is allocated: an index out of range, rows not grouped as the block edges say, a table that does
 * not fit on the device.  A chain that is not absorbing (a pivot <= 0 or not finite: splu's "singular matrix") is an error
 * that names the shell and the state; the macro atom then stays pending.  See tardis_b200/csrc/markov_build.cuh. */
typedef struct {
    int64_t n_transitions;                       /* T, as in the model */
    const double *transition_probabilities;      /* normalised (macroatom_solver.py:709-739): (row, shell) at
                                                    [t*tp_transition_stride + s*tp_shell_stride] */
    int64_t tp_transition_stride, tp_shell_stride;   /* transition_probabilities == NULL: the table tb200_build_opacity left
                                                    in HBM (refused if none was built since the last tb200_set_model) */
    const int64_t *source_level_idx, *destination_level_idx, *transition_type; /* [T]; rows with type >= 0 are internal.
                                                    transition_type must equal the model's (the transport reads the rows by it);
                                                    destination_level_idx is read for the internal rows only */
    int64_t n_states;                            /* max(source_level_idx) + 1 */
} tb200_markov_input;
int tb200_build_absorbing_markov(tb200_engine *engine, const tb200_markov_input *input);
/* X [S, n_states, n_states] as create_absorbing_probs returns it, and the normalised deactivation table [T,S] the transport
 * reads; either pointer may be NULL.  Needs the option keep_opacity_tables = 1 before tb200_build_absorbing_markov (the
 * kernels turn both tables into running sums in place). */
int tb200_download_absorbing_markov(tb200_engine *engine, double *matrix, double *deactivating);

/* ---- measurement ---- */
int tb200_last_kernel_ms(tb200_engine *engine, double *ms);          /* CUDA-event time of the last tb200_transport kernel */
int tb200_get_counters(tb200_engine *engine, tb200_counters *counters);
int64_t tb200_kernel_launches(tb200_engine *engine);                 /* kernels launched by this engine so far */
/* Tuning only (no option changes a result): "algorithm" (1 jump, default; 0 scan), "pooled" (1: per-warp packet pool in the
 * classic mode), "ctas_per_sm" / "park_min" (0 = the measured best for the kernel that will run; each kernel is compiled for
 * its default CTAs per SM, so another ctas_per_sm only sizes the grid, at most to what fits), "threads_per_cta" (256 | 128),
 * "vol_min", "refill_min", "sort_packets", "sort_bits", "pipeline_chunks", "pipeline_edges" (1, default: the first and the last
 * packet range of tb200_run are a quarter of the others, their copies being the ones no kernel hides), "keep_opacity_tables".
 * Any other name is an error. */
int tb200_set_option(tb200_engine *engine, const char *name, int64_t value);

/* ---- engine groups: one MC iteration on several GPUs from one host call ----
 * A group owns one ordinary engine per entry of device_ids; an id may repeat ({0, 0} is two engines on device 0).
 * tb200_group_member exposes the members, so every single-engine call stays usable on one.  The tb200_group_* calls
 * below apply to every member, one host thread per member; an error names the member (and, for runs, its global packet
 * range: the kernels record an error code, not the index of the packet that raised it) and leaves the group usable.
 * Members on the same device transport one after the other.
 *
 * tb200_group_run: member g transports packets [g N / G, (g + 1) N / G) of the caller's arrays (no host copies) at the
 * fixed-point scales of the whole set, and writes its per-packet outputs and last-interaction columns straight into the
 * caller's arrays at that offset.  TrackerFull rows cover global packets [0, n_tracked_packets) with global packet_id;
 * the virtual-packet log is concatenated in member order with global vlog_packet_index, vlog_count is the total (rows
 * beyond vlog_capacity are dropped, as with one engine; every member keeps a device log of vlog_capacity rows, and only the
 * rows that fit are copied to the caller).  Then tb200_group_allreduce, and the estimators come back as
 * from one engine: J_blue / Edotlu and the counters bit-identical to one engine over the same packets, the other sums
 * to rounding.
 * tb200_group_create_packets: member g generates exactly packets [g N / G, (g + 1) N / G) of what tb200_create_packets
 * gives one engine, in place (the set never passes through one device).  tb200_group_run_resident then runs them.
 * tb200_group_allreduce: the collective alone (for callers that drive tb200_transport per member), once per transport: a
 * second call without a transport in between fails (it would add the sums again).  Every member ends up with the same
 * estimator buffer.  *exact = 1: every member ran the jump algorithm at the same fixed-point scales, so
 * the line accumulators were summed as integers and finalized, and [0, off_j_blue) of the estimator buffer was summed
 * in f64 in member order; *exact = 0: the whole buffer was summed in f64 in member order.  Members whose devices have
 * peer access read each other's memory; the others (and all, with the option "peer_access" = 0) are staged through
 * cudaMemcpyPeerAsync.
 * tb200_group_formal_integral: member g integrates frequencies [g n / G, (g + 1) n / G); every member needs the
 * source-function tables (tb200_solve_source_function on each member: identical inputs give identical tables). */
typedef struct tb200_group tb200_group;
int tb200_group_create(const int *device_ids, int n, tb200_group **group);
void tb200_group_destroy(tb200_group *group);
int tb200_group_size(tb200_group *group);
int tb200_group_member(tb200_group *group, int i, tb200_engine **engine);
int tb200_group_set_option(tb200_group *group, const char *name, int64_t value); /* "peer_access" (1), or any engine option */
int tb200_group_set_model(tb200_group *group, const tb200_model *model, const tb200_config *config);
int tb200_group_set_atomic_data(tb200_group *group, const tb200_atomic_data *atomic);
int tb200_group_build_opacity(tb200_group *group, const tb200_plasma_state *plasma);
int tb200_group_set_plasma_data(tb200_group *group, const tb200_plasma_data *data);
/* every member solves the same plasma (bit-identical results); the host outputs are member 0's */
int tb200_group_solve_plasma(tb200_group *group, const tb200_plasma_params *params, double *electron_densities, double *ion_number_density,
                             double *level_number_density, double *j_blues, int32_t *iterations);
int tb200_group_build_absorbing_markov(tb200_group *group, const tb200_markov_input *input); /* every member, bit-identical tables */
int tb200_group_upload_packets(tb200_group *group, const tb200_packets *packets);
int tb200_group_create_packets(tb200_group *group, const tb200_packet_source *source);
int tb200_group_run(tb200_group *group, const tb200_packets *packets, tb200_outputs *outputs);
int tb200_group_run_resident(tb200_group *group, tb200_outputs *outputs);
int tb200_group_sync(tb200_group *group);
int tb200_group_allreduce(tb200_group *group, int *exact);
int tb200_group_allreduce_ms(tb200_group *group, double *ms); /* host time of the last collective, device work included */
int tb200_group_formal_integral(tb200_group *group, const tb200_formal_integral_params *params, const double *frequencies,
                                int64_t n_frequencies, double *luminosity_densities, double *intensities_nu_p);
int tb200_group_formal_integral_ms(tb200_group *group, double *interpolation_ms, double *integral_ms); /* slowest member's */

#ifdef __cplusplus
}
#endif
#endif /* TARDIS_B200_H */
