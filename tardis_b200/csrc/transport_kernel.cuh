// transport_kernel.cuh -- the packet-propagation kernel for sm_90a (H100).
//
// What it replaces (paths relative to /root/reference/tardis/):
//   montecarlo_transport_with_vpackets   transport/montecarlo/modes/montecarlo_transport.py:239-373
//   packet_propagation (classic)         transport/montecarlo/modes/classic/packet_propagation.py:53-251
//   trace_packet                         transport/montecarlo/modes/homologous_rad_packet_transport.py:30-174
//   + the leaf functions cited next to each device function below.
//
// Three kernels share the physics below (DESIGN.md §3).  All are persistent (one grid of resident CTAs), pull packets
// from a global counter in batches and give every packet its own lazily generated MT19937 stream:
//   transport_scan_kernel   the streaming formulation: the line scan of trace_packet is done by the WHOLE WARP for one
//                           lane's packet at a time -- 32 consecutive lines per step, coalesced 256-byte reads of
//                           nu_line / tau (shell-major), a warp prefix sum, one ballot, two coalesced fp64 reductions
//                           into the shell-major J_blue / Edotlu rows.  HBM/L2-bandwidth bound.
//   transport_jump_kernel   no scan: the end of a trace is searched in the double-double tau prefix table and the
//                           per-line estimator updates become two range updates in exact fixed point; one packet per
//                           lane, parked packets wait for company (continuum mode; classic with virtual packets).
//   transport_pool_kernel   the same algorithm with a per-warp pool of packet contexts in shared memory (classic mode).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "continuum_bins.cuh"

namespace tb {

constexpr double C_LIGHT = 2.99792458e10;        // configuration/constants.py:5 (CODATA-2010 via tardis/constants.py:1)
constexpr double INV_C = 1 / C_LIGHT;            // frame_transformations.py:27 `inv_c = 1 / C_SPEED_OF_LIGHT`
constexpr double CLOSE_LINE_THRESHOLD = 1e-14;   // configuration/constants.py:4
constexpr double MISS_DISTANCE = 1e99;           // configuration/constants.py:6
constexpr unsigned FULL = 0xffffffffu;

// InteractionType / PacketStatus, packets/radiative_packet.py:12-43
constexpr int IT_BOUNDARY = 1, IT_LINE = 2, IT_ESCATTERING = 4, IT_CONTINUUM_PROCESS = 8;
constexpr int ST_IN_PROCESS = 0, ST_EMITTED = 1, ST_REABSORBED = 2, ST_ADIABATIC_COOLING = 4;
constexpr double K_BOLTZMANN = 1.3806488e-16, H_PLANCK = 6.62606957e-27;  // CODATA-2010 cgs (tardis/constants.py:1)

constexpr int ERR_NU_DIFF = 1, ERR_MACRO_ATOM = 2, ERR_VPACKET_LOOP = 3, ERR_FIXED_POINT = 4, ERR_CONTINUUM = 5, ERR_STUCK = 6, ERR_OPACITY = 7;
constexpr int MAX_EVENTS_PER_PACKET = 4000000;  // watchdog: a packet that does this many events is reported, not waited for

constexpr int MT_N = 624;
constexpr int NU_KEY_SHIFT = 36;  // frequency-bucket key = sign, exponent and 16 mantissa bits of the binary64 pattern

enum Counter {
    CNT_LINE_STEPS = 0, CNT_BOUNDARY, CNT_LINE_EVENTS, CNT_ESCAT_EVENTS, CNT_RNG_DRAWS,
    CNT_MACRO_JUMPS, CNT_MACRO_SCANNED, CNT_VPACKETS, CNT_VPACKET_LINE_STEPS, CNT_CONT_EVENTS, CNT_BF_UPDATES, CNT_PROBES, CNT_COUNT
};

// Where a classic macro-atom transition leads, one int2 per transition (macro_next_kernel), independent of the shell:
// {start, end} of the destination block for an internal jump (start >= 0), {MNEXT_EMIT, line} for an emission,
// {MNEXT_BAD_LEVEL, 0} for an internal jump to a level outside the table, {MNEXT_BAD_TYPE, 0} for any other type.  The same
// encoding, per line, gives the block that absorbing the line activates (macro_entry).  One load then gives a jump both
// its outcome and the next block, where dest / ttype / tline and block_edge took two dependent loads.
constexpr int MNEXT_EMIT = -1, MNEXT_BAD_LEVEL = -2, MNEXT_BAD_TYPE = -3;

struct Event {  // == tb200_event
    long long packet_id, interaction_type, status, before_shell_id, after_shell_id, line_absorb_id, line_emit_id;
    double radius, before_nu, before_mu, before_energy, after_nu, after_mu, after_energy;
};

// Everything a packet's start needs, written at the packet's processing slot by the ordering pass (start_record_kernel /
// order_scatter_kernel): the lab-to-comoving transform of r, mu, nu, energy, the first line id, the 32-bit seed and x[397] of
// its generator, and the packet id.  A refill then takes consecutive slots with one coalesced 48-byte load per lane where
// it took a dependent chain (order -> six scattered gathers -> frame transform -> line search).
struct __align__(16) StartRecord {
    double r, mu, nu, energy;
    int next_line;
    unsigned seed, x397;
    int pid;
};
static_assert(sizeof(StartRecord) == 48, "StartRecord is three 16-byte loads");

struct KParams {
    // ---- geometry + opacity tables (device) ----
    int n_shells, n_lines, lpad;
    const double *r_inner, *r_outer, *n_e;   // [S]
    const double *nu_line;                   // [lpad], entries >= n_lines are 0
    const double *tau_t;                     // [S][lpad] shell-major
    const double2 *tau_prefix;               // [S][lpad+1] double-double (hi, lo) exclusive prefix sums of tau along the line list
    const int *nu_first_le;                  // [n_keys] first line index whose frequency key is <= k (frequency -> line index guess)
    long long nu_key_min; int n_keys;
    double t_exp, ct, inv_ct, sigma_thomson;
    // ---- macro atom ----
    int n_transitions, tpad, n_blocks;
    const double *tp_t;                      // [S][tpad] shell-major; per block: running sums of the transition probabilities
    const int *line2macro, *block_edge, *ttype, *dest, *tline;
    // ---- continuum / IIP mode (OpacityStateNumbaIIP, opacities/opacity_state_numba_iip.py:8-125) ----
    int continuum, n_continua, n_phot, phot_pad, n_activation, k_packet_idx, n_markov;
    const double *t_e, *bf_thr, *pi_min, *pi_max, *x_sect, *phot_nus, *ff_factor;
    const int *pi_refs, *pi_act;
    const double *chi_bf_t, *emiss_t;        // [S][phot_pad] shell-major
    const double *markov_cum;                // [S][n_markov][n_markov], running sums along the last axis
    double ff_opac_const;
    // global frequency bins of the bound-free opacity / estimators (continuum_bins.cuh); cont_bins == 0: literal path only
    int cont_bins, cb_n_gkeys;
    long long cb_gkey_min;
    const double *cb_B;                      // [n_phot] ascending union of the phot_nus blocks
    const int *cb_guide, *cb_nact;           // [cb_n_gkeys + 1]; [n_phot + 1] active continua per bin
    const int *cb_act_start;                 // [n_phot + 2]: bin g's {continuum, lower phot_nus index} pairs are
    const int2 *cb_act;                      //   cb_act[cb_act_start[g] .. cb_act_start[g + 1]) (HostBins::act)
    const double2 *cb_chi_lin;               // [S][n_phot + 1] {chi_bf_tot at the bin's left edge, slope}
    double *cb_mom;                          // [S][n_phot + 1][8] moments (tbc::trace_moments)
    double *cont_lit;                        // [5][n_continua][S] {photo_ion, stim_recomb, bf_heating, stim_recomb_cooling, statistics}
                                             // accumulated by the literal per-continuum path (breakpoint ties, odd tables)
    // ---- configuration ----
    int full_rel, line_mode, disable_line, n_vpackets;
    double survival_probability, tau_russian, spawn_start, spawn_end;
    const double *grid; int n_grid;
    // ---- packets ----
    long long n_packets;
    const double *in_r, *in_nu, *in_mu, *in_energy;
    const unsigned *seed, *seed_x397;        // by packet id: what rng_replay_tier1 replays a packet's first outputs from
    const StartRecord *start;                // by processing slot (StartRecord)
    int refill_min;                          // refill a warp when this many lanes are free
    int park_min;                           // jump kernel: run the slow phase when this many lanes are parked
    double *out_nu, *out_energy;
    // ---- estimators (device, packed buffer) ----
    double *J, *nubar, *vhist, *jblue_t, *edotlu_t;
    double *spec_emitted, *spec_reabsorbed;  // [n_grid - 1] fused energy histograms of the finished packets (or nullptr)
    // ---- jump algorithm: fixed-point difference arrays, [S][lpad+1][4] = {w1 hi, w1 lo, w2 hi, w2 lo} ----
    unsigned long long *diff;
    unsigned long long *xfer;                // [S-1][lpad+1][4] transfers across the interface between shells s and s+1,
                                             // folded into diff by fold_transfers_kernel (trace_range_end)
    double scale1, scale2;                   // powers of two
    // ---- scratch / control ----
    unsigned *rng_buf;                       // [n_warps][624][32]
    unsigned long long *next_packet;
    int *error;
    unsigned long long *counters;            // [CNT_COUNT]
    double grid0, grid_last, inv_dgrid;      // spectrum grid: first / last edge, 1 / (edge[1] - edge[0]) (binning guess only)
    const int *macro_guide;                  // [S][tpad] bracket table of the classic macro atom (macro_guide_kernel), or null
    const int2 *macro_next, *macro_entry;    // [T] / [L] classic macro atom: where a transition leads / the block a line
                                             //    activates (macro_next_kernel), or null in continuum mode
    unsigned long long *cnt_rep;             // [bulk_reps][CNT_COUNT] replicas of the rare-path counters
    double *bulk_rep;                        // [bulk_reps][rep_stride] replicas {J(S) | nu_bar(S) | luminosity sums(4) | ff_heating(S, continuum)}
    int bulk_reps;                           // power of two
    int rep_stride;
    int vol_off, vol_min;                    // warp-cooperative volleys: vol_off: first double of the item area in smem;
                                             //    vol_min: run the volleys when this many lanes wait for one
    double lum_nu_start, lum_nu_end;         // calculate_filtered_luminosity window (spectrum/luminosity.py:5-29), strict on both sides
    int park_off;                            // jump kernels: first double of the parked-packet area in dynamic shared memory
    int pool_slots;                          // pooled jump kernel: packet contexts per warp (32 + park_min)
    int rng_units;                           // MT rings per warp (32 lanes, + pool_slots in the pooled kernel)
    // ---- optional tracking ----
    long long *last_type, *last_event_id, *last_shell, *last_absorb, *last_emit;
    double *last_radius, *last_before_nu, *last_before_mu, *last_before_energy, *last_after_nu, *last_after_mu, *last_after_energy;
    Event *events; long long *event_counts; long long n_tracked, max_events;
    // ---- optional virtual packet log ----
    double *vlog_nu, *vlog_energy, *vlog_mu, *vlog_r; long long *vlog_pid; long long vlog_capacity;
    unsigned long long *vlog_count;
    // ---- nonhomologous mode (nonhomologous.cuh): NumbaRadial1DGeometry's per-shell velocities [S] ----
    const double *v_inner, *v_outer, *dvdr;
};

// Launch parameters live in constant memory: every field is a warp-uniform broadcast read, and the
// out-of-line helpers (virtual packets, macro atom, trackers) need no parameter block on the stack.
__constant__ KParams cP;

// ------------------------------------------------------------------------------------------
// MT19937 exactly as Numba seeds and draws it (numba/_random.c:37-75, numba/cpython/randomimpl.py:109-147),
// but generated lazily in three tiers so that a packet never pays the 624-word init + twist up front:
//   outputs   0..226 : x[n], x[n+1], x[n+397] all come from the Knuth init recurrence -> two running cursors
//   outputs 227..623 : x[n+397] is an already generated word, read back from the per-lane ring
//   outputs 624..    : the textbook in-place recurrence on the ring
// x[397] of each packet's seed is precomputed by the ordering pass (start_fields).
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned mt_init_next(unsigned x, unsigned k) { return 1812433253u * (x ^ (x >> 30)) + k; }

// Outputs 0..226 are pure functions of the seed, so the common short packet never writes the ring (which
// would cost ~1.4 kB of scattered DRAM traffic per packet).  A packet that does reach output 227 replays
// them once into the ring.  (Free function with by-value arguments: a noinline MEMBER would take `this`, and an
// object whose address reaches a real call is kept in local memory for its whole life.)
__device__ __noinline__ void rng_replay_tier1(unsigned seed0, unsigned b0, unsigned *buf, unsigned stride) {
    unsigned ra = seed0, rb = b0;
#pragma unroll 1
    for (unsigned k = 0; k < 227u; k++) {
        const unsigned xn1 = mt_init_next(ra, k + 1u);
        const unsigned y = (ra & 0x80000000u) | (xn1 & 0x7fffffffu);
        buf[k * stride] = rb ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
        ra = xn1; rb = mt_init_next(rb, k + 398u);
    }
}

// Tiers 2 and 3 of the generator (a packet's outputs 227 and later: ring read-back, then the in-place recurrence),
// out of line and by value so that the hot loop carries neither their code nor an address-taken Rng.
// Returns {untempered output, updated cursor a}.
__device__ __noinline__ uint2 rng_slow_next(unsigned n, unsigned a, unsigned pid, unsigned ring) {
    const size_t gwarp = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const unsigned st = (unsigned)cP.rng_units;
    unsigned *rg = cP.rng_buf + gwarp * (size_t)MT_N * st + ring;  // word k of this packet's ring at rg[k * st]
    unsigned xn, xn1, xm, k;
    if (n == 227u && !cP.continuum) rng_replay_tier1(cP.seed[pid], cP.seed_x397[pid], rg, st);
    if (n < 624u) {
        k = n; xn = a;
        if (n < 623u) { xn1 = mt_init_next(a, n + 1u); a = xn1; } else { xn1 = rg[0]; }
        xm = rg[(n - 227u) * st];
    } else {
        k = n % 624u;
        const unsigned k1 = (k == 623u) ? 0u : k + 1u;
        const unsigned km = (k >= 227u) ? k - 227u : k + 397u;
        xn = rg[k * st]; xn1 = rg[k1 * st]; xm = rg[km * st];
    }
    const unsigned y = (xn & 0x80000000u) | (xn1 & 0x7fffffffu);
    const unsigned v = xm ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
    rg[k * st] = v;
    return make_uint2(v, a);
}

// One out-of-line copy of the generator for the continuum-mode call sites: that kernel's hot code is ~70 kB against a 32 kB
// instruction cache and fetch is its largest stall; inlining the two-output draw at its ~20 sites made it slower, while the
// classic kernels, whose hot loop nearly fits, are faster with the draw inlined.  Two consecutive outputs (one double) of a
// packet's generator, by value:
// {out0 >> 5, out1 >> 6, cursor a, cursor b}.
__device__ __noinline__ uint4 rng_draw_pair(unsigned n, unsigned a, unsigned b, unsigned pid, unsigned ring) {
    unsigned out[2];
#pragma unroll
    for (int h = 0; h < 2; h++) {
        unsigned v;
        if (__builtin_expect(n < 227u, 1)) {
            const unsigned xn = a, xn1 = mt_init_next(a, n + 1u), xm = b;
            a = xn1; b = mt_init_next(b, n + 398u);
            const unsigned y = (xn & 0x80000000u) | (xn1 & 0x7fffffffu);
            v = xm ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
            if (cP.continuum) {  // tier-1 words go to the ring as they are drawn: output 227 then needs no replay
                const size_t gwarp = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
                cP.rng_buf[(gwarp * (size_t)MT_N + n) * (unsigned)cP.rng_units + ring] = v;
            }
        } else {
            const uint2 r = rng_slow_next(n, a, pid, ring);
            v = r.x; a = r.y;
        }
        n++;
        v ^= v >> 11; v ^= (v << 7) & 0x9d2c5680u; v ^= (v << 15) & 0xefc60000u; v ^= v >> 18;
        out[h] = v;
    }
    return make_uint4(out[0] >> 5, out[1] >> 6, a, b);
}

struct Rng {
    unsigned n, a, b;
    unsigned pid;   // index of the packet's seed / x[397] (n_packets <= 2e9): tier 1 is replayed from them, not stored
    unsigned ring;  // which of the warp's rng_units rings belongs to the packet (travels with it; start() keeps it)
    __device__ __forceinline__ void start(unsigned seed, unsigned x397, unsigned pid_) { n = 0; a = seed; b = x397; pid = pid_; }
    __device__ __forceinline__ unsigned next_u32() {
        unsigned v;
        if (__builtin_expect(n < 227u, 1)) {
            const unsigned xn = a, xn1 = mt_init_next(a, n + 1u), xm = b;
            a = xn1; b = mt_init_next(b, n + 398u);
            const unsigned y = (xn & 0x80000000u) | (xn1 & 0x7fffffffu);
            v = xm ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
        } else {
            const uint2 r = rng_slow_next(n, a, pid, ring);
            v = r.x; a = r.y;
        }
        n++;
        v ^= v >> 11; v ^= (v << 7) & 0x9d2c5680u; v ^= (v << 15) & 0xefc60000u; v ^= v >> 18;
        return v;
    }
    // STORE = continuum-mode call site (tens of draws per packet): the out-of-line copy, which in continuum mode also writes
    // every tier-1 word to the packet's ring as it is drawn, so that reaching output 227 needs no replay.  The
    // classic kernels' call sites inline the draw and carry none of that (it slows the headline kernel down).
    template <bool STORE = false>
    __device__ __forceinline__ double next_double() {
        unsigned hi, lo;
        if (STORE) {  // continuum-mode site: the shared out-of-line copy (see rng_draw_pair)
            const uint4 r = rng_draw_pair(n, a, b, pid, ring);
            n += 2u; a = r.z; b = r.w;
            hi = r.x; lo = r.y;
        } else {
            hi = next_u32() >> 5; lo = next_u32() >> 6;
        }
        // (a * 67108864.0 + b) / 9007199254740992.0 -- every step is exact in binary64
        return ((double)lo + (double)hi * 67108864.0) * (1.0 / 9007199254740992.0);
    }
};

// the generator's 32-bit seed and x[397] (Rng::start) from a packet's 64-bit seed
__device__ __forceinline__ uint2 seed_expand(long long seed64) {
    const unsigned s = (unsigned)(seed64 & 0xffffffffll);  // np.random.seed takes uint32 (randomimpl.py:213-225)
    unsigned x = s;
#pragma unroll 4
    for (unsigned k = 1; k <= 397u; k++) x = mt_init_next(x, k);
    return make_uint2(s, x);
}

// ------------------------------------------------------------------------------------------
// frame transformations, transport/frame_transformations.py:12-109 (literal operation order)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ double doppler_factor_fr(double velocity, double mu) {
    double beta = velocity * INV_C;
    return (1.0 - mu * beta) / sqrt(1 - beta * beta);
}
__device__ __forceinline__ double inverse_doppler_factor_fr(double velocity, double mu) {
    double beta = velocity * INV_C;
    return (1.0 + mu * beta) / sqrt(1 - beta * beta);
}
template <bool FR> __device__ __forceinline__ double doppler_factor(double velocity, double mu) {
    if (FR) return doppler_factor_fr(velocity, mu);
    double beta = velocity * INV_C;
    return 1.0 - mu * beta;
}
template <bool FR> __device__ __forceinline__ double inverse_doppler_factor(double velocity, double mu) {
    if (FR) return inverse_doppler_factor_fr(velocity, mu);
    double beta = velocity * INV_C;
    return 1.0 / (1.0 - mu * beta);
}
__device__ __forceinline__ double aberration_cmf_to_lf(double r, double t_exp, double mu) {
    double ct = C_LIGHT * t_exp;
    double beta = r / ct;
    return (mu + beta) / (1.0 + beta * mu);
}
__device__ __forceinline__ double aberration_lf_to_cmf(double r, double t_exp, double mu) {
    double ct = C_LIGHT * t_exp;
    double beta = r / ct;
    return (mu - beta) / (1.0 - beta * mu);
}

// transport/geometry/calculate_distances.py:25-62
__device__ __forceinline__ double distance_boundary(double r, double mu, double r_inner, double r_outer, int &delta_shell) {
    double distance;
    if (mu > 0.0) {
        distance = sqrt(r_outer * r_outer + ((mu * mu - 1.0) * r * r)) - (r * mu);
        delta_shell = 1;
    } else {
        double check = r_inner * r_inner + (r * r * (mu * mu - 1.0));
        if (check >= 0.0) {
            distance = -r * mu - sqrt(check);
            delta_shell = -1;
        } else {
            distance = sqrt(r_outer * r_outer + ((mu * mu - 1.0) * r * r)) - (r * mu);
            delta_shell = 1;
        }
    }
    return distance;
}

// transport/geometry/calculate_distances.py:198-219
// (out of line on purpose: a square root and three divisions, used at a dozen call sites of kernels that are bound by
//  instruction fetch)
__device__ __noinline__ double distance_line_full_relativity(double nu_line, double nu, double t_exp, double r, double mu) {
    double nu_r = nu_line / nu;
    double ct = C_LIGHT * t_exp;
    return -mu * r + (ct - nu_r * nu_r * sqrt(ct * ct - (1 + r * r * (1 - mu * mu) * (1 + 1.0 / (nu_r * nu_r))))) / (1 + nu_r * nu_r);
}

// transport/geometry/calculate_distances.py:66-112, literal (used once per LINE event and by the virtual packets)
template <bool FR>
__device__ __forceinline__ double distance_line_literal(double r, double mu, double nu, double comov_nu, bool is_last_line,
                                                        double nu_line, double t_exp, int *error) {
    if (is_last_line) return MISS_DISTANCE;
    double nu_diff = comov_nu - nu_line;
    if (fabs(nu_diff / nu) < CLOSE_LINE_THRESHOLD) return 0.0;
    if (!(nu_diff >= 0)) { atomicMax(error, ERR_NU_DIFF); return 0.0; }
    if (FR) return distance_line_full_relativity(nu_line, nu, t_exp, r, mu);
    return (nu_diff / nu) * C_LIGHT * t_exp;
}

// Partial relativity inside the trace loops: the distance to a line as nu_diff * d_scale with d_scale = c t * (1 / nu),
// computed once per trace, instead of the reference's (nu_diff / nu) * c * t.  The product carries four roundings
// (1 / nu, c t, d_scale, the product), the reference's expression three, each <= u = 2^-53 relative, so the two differ
// by at most ~7u = 8e-16 relative (4 ulps seen in practice) -- enough to decide `d_boundary <= d` the other way when
// the line sits at the boundary.  Within PR_TIE_MARGIN = 1e-14 (> 12 x 7u) of d_boundary the reference's expression is
// recomputed and decides (scan kernel); outside it both lie on the same side of d_boundary.  The jump kernels search with
// the plain product and redo the search with the reference's expression when its result lies at such a tie
// (trace_phase_a, event_phase_b): a check in every probe costs the pooled kernel ~4 %.
// (The recomputation is out of line: it is rarely taken, and a division inlined at every call site bloats the hot loops.)
constexpr double PR_TIE_MARGIN = 1e-14;
__device__ __noinline__ double line_distance_partial_literal(double nu_diff, double nu) { return (nu_diff / nu) * C_LIGHT * cP.t_exp; }
__device__ __forceinline__ double line_distance_partial(double nu_diff, double d_scale, double nu, double d_boundary) {
    const double d = nu_diff * d_scale;
    if (__builtin_expect(fabs(d - d_boundary) <= PR_TIE_MARGIN * d_boundary, 0)) return line_distance_partial_literal(nu_diff, nu);
    return d;
}

__device__ __forceinline__ double shfl_d(double v, int src) { return __shfl_sync(FULL, v, src); }
__device__ __forceinline__ double shfl_up_d(double v, int d) { return __shfl_up_sync(FULL, v, d); }

// (a.x + a.y) - (b.x + b.y) in double-double arithmetic, rounded to one double
__device__ __forceinline__ double dd_diff(const double2 a, const double2 b) {
    double s = a.x - b.x;
    double bb = s - a.x;
    double err = (a.x - (s - bb)) - (b.x + bb);
    return s + (err + (a.y - b.y));
}

// add w * scale (scale = 2^k) to a 104-bit fixed-point accumulator made of two 64-bit words:
// Reductions into GLOBAL memory, stated as such.  The tables' addresses come out of the __constant__ parameter block,
// so the compiler only knows them as generic pointers: a generic fp64 atomicAdd carries a run-time "is this shared
// memory?" branch with a compare-and-swap loop behind it, and a generic integer one returns a value nobody reads.
__device__ __forceinline__ void red_f64(double *addr, double v) {
    asm volatile("red.global.add.f64 [%0], %1;" ::"l"(__cvta_generic_to_global(addr)), "d"(v) : "memory");
}
__device__ __forceinline__ void red_u64(unsigned long long *addr, unsigned long long v) {
    asm volatile("red.global.add.u64 [%0], %1;" ::"l"(__cvta_generic_to_global(addr)), "l"(v) : "memory");
}

// word0 += floor(t / 2^29), word1 += round(t mod 2^29), with the typical term scaled to 2^58 (engine.cu).  Integer adds are
// exact and order-independent, so the sums are bit-reproducible and cells that no packet touched stay exactly zero.
// Headroom: a cell's low word holds 2^34 same-sign terms, its high word 2^33 typical ones (2^27 of the heaviest that equal
// energies and a line list spanning a factor 40 in frequency can produce) before the signed reading in
// finalize_line_estimators_kernel would be off by 2^64 -- and that kernel notices: every trace adds +w at its first line and
// -w behind its last, so each row must sum to exactly zero and no prefix is negative (ERR_FIXED_POINT otherwise).
// fixed_term converts w once (false, with ERR_FIXED_POINT raised, when w * scale is out of range); fixed_add adds it or its
// negative to one cell.
constexpr double FIXED_SPLIT = 536870912.0;  // 2^29
constexpr int FIXED_TYPICAL_LOG2 = 58;
struct FixedTerm { long long hi, lo; };
__device__ __forceinline__ bool fixed_term(double w, double scale, FixedTerm &f, int *error) {
    const double t = w * scale;
    const double th = t * (1.0 / FIXED_SPLIT);
    if (__builtin_expect(!(th < 4.0e18) || !(t >= 0.0), 0)) { atomicMax(error, ERR_FIXED_POINT); return false; }
    f.hi = __double2ll_rd(th);
    f.lo = __double2ll_rn(t - (double)f.hi * FIXED_SPLIT);
    return true;
}
__device__ __forceinline__ void fixed_add(unsigned long long *cell, const FixedTerm &f, bool negative) {
    red_u64(cell, (unsigned long long)(negative ? -f.hi : f.hi));
    red_u64(cell + 1, (unsigned long long)(negative ? -f.lo : f.lo));
}

struct Counters {
    unsigned long long line_steps = 0, boundary = 0, line_ev = 0, escat_ev = 0, draws = 0;
    unsigned long long jumps = 0, scanned = 0, vp = 0, vsteps = 0, probes = 0, cont_ev = 0, bf_upd = 0;
};
constexpr int CNT_SLOTS = CNT_COUNT;
// The counters of a rare path go straight to one of cnt_reps global replicas [CNT_COUNT] (u64 RED, summed by
// reduce_bulk_kernel): adding them to the hot loop's register-resident Counters would keep all twelve 64-bit fields live
// across the loop, and 64-bit shared-memory atomics are compare-and-swap loops (5 % of the pooled kernel's samples).
__device__ __forceinline__ unsigned long long *counter_replica() {
    const KParams &P = cP;
    return P.cnt_rep + (size_t)((blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) & (P.bulk_reps - 1)) * CNT_SLOTS;
}
__device__ __forceinline__ void flush_rare(const Counters &o) {
    const unsigned long long v[CNT_SLOTS] = {o.line_steps, o.boundary, o.line_ev, o.escat_ev, o.draws, o.jumps, o.scanned,
                                             o.vp, o.vsteps, o.cont_ev, o.bf_upd, o.probes};
    unsigned long long *rep = counter_replica();
#pragma unroll
    for (int k = 0; k < CNT_SLOTS; k++) if (v[k]) red_u64(&rep[k], v[k]);
}

// Calling convention for the rare, out-of-line paths below: a *_impl function is a real call that takes the packet
// state by reference, and an object whose address reaches a real call lives in local memory for its WHOLE life
// (every p.r / p.mu in the hot loop becomes a local load).  So the inlined wrappers hand the call copies made inside
// the rare branch and copy the result back: the hot loop's Lane / Rng / Counters / TraceSetup stay in registers.

// first index with nu_line < nu (== number of lines with nu_line >= nu), bracketed by the frequency-bucket table
__device__ __forceinline__ int first_line_below(double nu) {
    const KParams &P = cP;
    const int L = P.n_lines;
    int lo = 0, hi = L;
    if (nu > 0.0) {
        const long long kb = (__double_as_longlong(nu) >> NU_KEY_SHIFT) - P.nu_key_min;
        if (kb >= (long long)P.n_keys) { hi = 0; }
        else if (kb >= 0) { lo = P.nu_first_le[kb]; hi = (kb > 0) ? P.nu_first_le[kb - 1] : L; }
        else { lo = L; }
    }
    if (hi - lo <= 8) {  // the usual bucket: independent loads instead of a dependent chain (rows are padded)
        int cnt = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) cnt += (lo + k < hi && P.nu_line[lo + k] >= nu);
        return lo + cnt;
    }
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (P.nu_line[mid] >= nu) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// (out of line: faster for the classic kernels' packet start and virtual-packet literal walk, slower at the continuum
//  emission sites)
__device__ __noinline__ int first_line_below_call(double nu) { return first_line_below(nu); }

// first index with nu_line <= nu, L - 1 when there is none or nu is not positive (guess helper; clamped by the callers)
__device__ __forceinline__ int first_line_at_or_below(double nu) {
    const KParams &P = cP;
    const int L = P.n_lines;
    if (!(nu > 0.0)) return L - 1;
    const long long kb = (__double_as_longlong(nu) >> NU_KEY_SHIFT) - P.nu_key_min;
    if (kb >= (long long)P.n_keys) return 0;
    if (kb < 0) return L - 1;
    int glo = P.nu_first_le[kb];
    int ghi = (kb > 0) ? P.nu_first_le[kb - 1] : L;
    if (ghi - glo <= 8) {  // a bucket holds ~2 lines on average: eight independent loads, no dependent chain
        // (a lane that needs the bisection below holds up its whole warp: with <= 4 that was 7 % of the traces)
        int cnt = 0;  // number of bracket entries that are still > nu (the list is sorted; rows are padded)
#pragma unroll
        for (int k = 0; k < 8; k++) cnt += (glo + k < ghi && P.nu_line[glo + k] > nu);
        return glo + cnt;
    }
    while (glo < ghi) {
        const int mid = (glo + ghi) >> 1;
        if (P.nu_line[mid] <= nu) ghi = mid; else glo = mid + 1;
    }
    return glo;
}

// ------------------------------------------------------------------------------------------
// Per-lane packet state.  RPacket, packets/radiative_packet.py:47-110, plus the tracker counters.
// ------------------------------------------------------------------------------------------
struct Lane {
    double r, mu, nu, energy;
    int pid;  // n_packets <= 2e9 (tb200_upload_packets)
    int next_line, shell, status;
    int icount, bbuf;  // TrackerLastInteraction.interactions_count / _boundary_interactions_buffer
    int nev;           // rows written to the TrackerFull log
    int nsteps;        // events of this packet so far (watchdog)
    int seg_open;      // jump kernels: the +w that opens this trace's estimator range was already added by the transfer at the
                       // shell crossing that ended the previous trace (trace_range_end)
};

// the state of a lane that holds no packet yet
__device__ __forceinline__ Lane idle_lane() {
    Lane p;
    p.status = -1; p.pid = -1; p.r = p.mu = p.nu = p.energy = 0.0; p.next_line = 0; p.shell = 0; p.icount = 0; p.bbuf = 0; p.nev = 0; p.nsteps = 0; p.seg_open = 0;
    return p;
}

__device__ __noinline__ void log_boundary_slow(Lane &p, int from_shell, int to_shell) {
    const KParams &P = cP;
    if (P.events && p.pid < P.n_tracked) {
        if (p.nev < P.max_events) {
            Event &e = P.events[(size_t)p.pid * P.max_events + p.nev];
            e.packet_id = p.pid; e.interaction_type = IT_BOUNDARY; e.status = p.status;
            e.before_shell_id = from_shell; e.after_shell_id = to_shell; e.line_absorb_id = -1; e.line_emit_id = -1;
            e.radius = p.r; e.before_nu = p.nu; e.before_mu = p.mu; e.before_energy = p.energy;
            e.after_nu = p.nu; e.after_mu = p.mu; e.after_energy = p.energy;
        }
        p.nev++;
    }
}

__device__ __forceinline__ void log_boundary(Lane &p, int from_shell, int to_shell) {
    const KParams &P = cP;
    p.bbuf += 1;  // tracker_last_interaction.py:209-231
    if (P.events) { Lane lp = p; log_boundary_slow(lp, from_shell, to_shell); p.nev = lp.nev; }  // the copy keeps p in registers
}

__device__ __noinline__ void log_interaction_before(Lane &p, int type) {
    const KParams &P = cP;
    if (P.last_type) {  // tracker_last_interaction.py:84-99,127-143
        P.last_before_nu[p.pid] = p.nu; P.last_before_mu[p.pid] = p.mu; P.last_before_energy[p.pid] = p.energy;
        if (type == IT_LINE) { P.last_absorb[p.pid] = p.next_line; }
        else { P.last_absorb[p.pid] = -1; P.last_emit[p.pid] = -1; }
    }
    if (P.events && p.pid < P.n_tracked && p.nev < P.max_events) {
        Event &e = P.events[(size_t)p.pid * P.max_events + p.nev];
        e.packet_id = p.pid; e.interaction_type = type; e.status = p.status;
        e.before_shell_id = p.shell; e.after_shell_id = p.shell;
        e.line_absorb_id = (type == IT_LINE) ? p.next_line : -1; e.line_emit_id = -1;
        e.radius = p.r; e.before_nu = p.nu; e.before_mu = p.mu; e.before_energy = p.energy;
    }
}

__device__ __noinline__ void log_interaction_after_slow(Lane &p, int type) {
    const KParams &P = cP;
    if (P.last_type) {
        P.last_after_nu[p.pid] = p.nu; P.last_after_mu[p.pid] = p.mu; P.last_after_energy[p.pid] = p.energy;
        if (type == IT_LINE) P.last_emit[p.pid] = p.next_line - 1;
        P.last_event_id[p.pid] = p.icount;
        P.last_radius[p.pid] = p.r; P.last_shell[p.pid] = p.shell; P.last_type[p.pid] = type;
    }
    if (P.events && p.pid < P.n_tracked) {
        if (p.nev < P.max_events) {
            Event &e = P.events[(size_t)p.pid * P.max_events + p.nev];
            e.after_nu = p.nu; e.after_mu = p.mu; e.after_energy = p.energy;
            if (type == IT_LINE) e.line_emit_id = p.next_line - 1;
        }
        p.nev++;
    }
}

__device__ __forceinline__ void log_interaction_after(Lane &p, int type) {
    const KParams &P = cP;
    p.icount += 1 + p.bbuf;  // tracker_last_interaction.py:100-125,144-165
    p.bbuf = 0;
    if (P.last_type || P.events) log_interaction_after_slow(p, type);
}

// interaction_events.py:227-258
template <bool FR> __device__ __forceinline__ void line_emission(Lane &p, int emission_line_id) {
    const KParams &P = cP;
    double velocity = p.r / P.t_exp;
    double inv_doppler = inverse_doppler_factor<FR>(velocity, p.mu);
    p.nu = P.nu_line[emission_line_id] * inv_doppler;
    p.next_line = emission_line_id + 1;
    if (FR) p.mu = aberration_cmf_to_lf(p.r, P.t_exp, p.mu);
}

// line_emission of the homologous modes, as the emitter of macro_atom_event
template <bool FR> struct HomologousEmission {
    __device__ __forceinline__ void operator()(Lane &p, int emission_line_id) const { line_emission<FR>(p, emission_line_id); }
};

// macro_atom.py:52-104 + interaction_event_callers.py:31-91 (classic branch).  `entry`: P.macro_entry of the absorbed line.
// The walk does not depend on the velocity law; EMIT is the line_emission of the caller's mode (nonhomologous.cuh has its own).
template <bool FR, typename EMIT = HomologousEmission<FR>>
__device__ __noinline__ void macro_atom_event(Lane &p, Rng &rng, int2 entry,
                                                 unsigned long long &n_jumps, unsigned long long &n_scanned) {
    const KParams &P = cP;
    // P.tp_t holds, per shell, the running sum of the transition probabilities inside each block, accumulated in
    // the reference's order (macro_cumsum_kernel): cum[tid] is bit-for-bit the `probability` the reference compares
    // with its random number after adding transition tid, so the first tid with cum[tid] > xi is found by bisection.
    const double *cum = P.tp_t + (size_t)p.shell * P.tpad;
    const int *guide = P.macro_guide + (size_t)p.shell * P.tpad;
    int2 next = entry;  // the block this jump draws from, or what ends the walk
    while (next.x >= 0 || next.x == MNEXT_BAD_LEVEL) {
        double xi = rng.next_double();
        n_jumps++;
        if (next.x < 0) { atomicMax(P.error, ERR_MACRO_ATOM); return; }  // a level outside the table
        const int block_start = next.x, block_end = next.y;
        if (block_end <= block_start || !(cum[block_end - 1] > xi)) {  // "MacroAtom ran out of the block"
            n_scanned += (unsigned long long)(block_end - block_start);
            atomicMax(P.error, ERR_MACRO_ATOM);
            return;
        }
        // bracket from the guide table: the answer lies between the entries of buckets k-1 and k+2 (one bucket of
        // slack on each side covers the rounding of xi * n); cum is non-decreasing, so bisection inside is exact
        const int n = block_end - block_start;
        int k = (int)(xi * (double)n);
        k = k < 0 ? 0 : (k > n - 1 ? n - 1 : k);
        int lo = guide[block_start + (k > 0 ? k - 1 : 0)];
        int hi = (k + 2 < n) ? guide[block_start + k + 2] : block_end - 1;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (cum[mid] > xi) hi = mid; else lo = mid + 1;
        }
        n_scanned += (unsigned long long)(lo - block_start + 1);
        next = P.macro_next[lo];
    }
    if (next.x == MNEXT_EMIT) EMIT()(p, next.y);
    else atomicMax(P.error, ERR_MACRO_ATOM);
}


// ------------------------------------------------------------------------------------------
// Continuum processes (IIP mode).  References: opacities/opacities.py:89-246, radfield_estimator_calcs.py:57-124,
// interaction_events.py:21-180,262-299, interaction_event_callers.py:31-183, macro_atom.py:108-184.
// ------------------------------------------------------------------------------------------
struct PhotInterp { int lo, hi; double high_weight, low_weight, interval; };  // indices into the phot_nus / chi_bf rows

// np.searchsorted(phot_nus[start:end], nu) and the linear-interpolation weights of chi_bf_interpolator (:139-161)
__device__ __forceinline__ PhotInterp phot_interp(int k, double nu) {
    const KParams &P = cP;
    const int start = P.pi_refs[k], n = P.pi_refs[k + 1] - start;
    const double *pn = P.phot_nus + start;
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (pn[mid] < nu) lo = mid + 1; else hi = mid;
    }
    int idx = lo;
    if (idx >= n) { atomicMax(P.error, ERR_CONTINUUM); idx = n - 1; }
    const int im1 = (idx == 0) ? n - 1 : idx - 1;  // python's [-1] wrap
    PhotInterp r;
    r.hi = start + idx; r.lo = start + im1;
    r.interval = pn[idx] - pn[im1];
    r.high_weight = nu - pn[im1];
    r.low_weight = pn[idx] - nu;
    return r;
}

// chi_continuum_calculator, literally: total bound-free opacity (cumsum order = continuum order).  Used where the global
// bins do not apply (a frequency exactly on a breakpoint, tables without the expected structure) and by continuum_event.
__device__ __noinline__ double chi_bf_literal(double nu, int shell, int *n_active) {
    const KParams &P = cP;
    const double *chi_row = P.chi_bf_t + (size_t)shell * P.phot_pad;
    double running = 0.0;
    int n_act = 0;
    for (int k = 0; k < P.n_continua; k++) {
        if (nu >= P.pi_min[k] && nu <= P.pi_max[k]) {
            const PhotInterp w = phot_interp(k, nu);
            running += (chi_row[w.hi] * w.high_weight + chi_row[w.lo] * w.low_weight) / w.interval;
            n_act++;
        }
    }
    *n_active = n_act;
    return running;
}

// update_estimators_bound_free, literally (same cases as chi_bf_literal): five reductions per active continuum into
// cont_lit = [5][n_continua][S]; continuum_finalize_kernel adds them to what the moments give.
__device__ __noinline__ void bf_estimators_literal(double comov_nu, double comov_energy, int shell, double distance, double boltzmann_factor) {
    const KParams &P = cP;
    const size_t ncs = (size_t)P.n_continua * P.n_shells;
    for (int k = 0; k < P.n_continua; k++) {
        if (comov_nu >= P.pi_min[k] && comov_nu <= P.pi_max[k]) {
            const PhotInterp w = phot_interp(k, comov_nu);
            const double xs = (P.x_sect[w.hi] * w.high_weight + P.x_sect[w.lo] * w.low_weight) / w.interval;
            const size_t cell = (size_t)k * P.n_shells + shell;
            const double inc = comov_energy * distance * xs / comov_nu;
            red_f64(&P.cont_lit[cell], inc);
            red_f64(&P.cont_lit[ncs + cell], inc * boltzmann_factor);
            const double bfh = comov_energy * distance * xs * (1 - P.bf_thr[k] / comov_nu);
            red_f64(&P.cont_lit[2 * ncs + cell], bfh);
            red_f64(&P.cont_lit[3 * ncs + cell], bfh * boltzmann_factor);
            red_f64(&P.cont_lit[4 * ncs + cell], 1.0);  // exact integer counts in binary64; converted to int64 on download
        }
    }
}

// What trace_setup keeps of the continuum opacities for the estimator update after the trace
struct ContTrace { double boltz; int g, n_active; };  // g: global bin, or -1 = literal path

// chi_bf_tot and chi_ff of a trace (opacities/opacities.py:89-246).  The exponential is shared with the stimulated-
// recombination estimators: exp(-H nu / (k T)) here and exp(-(H nu) / (k T)) there are the same number.
__device__ __forceinline__ void chi_continuum(double nu, int shell, double &chi_bf_tot, double &chi_ff, ContTrace &ct) {
    const KParams &P = cP;
    bool tie = false;
    int g = -1;
    if (P.cont_bins) {
        tbc::BinView v;
        v.B = P.cb_B; v.guide = P.cb_guide; v.gkey_min = P.cb_gkey_min; v.n_gkeys = P.cb_n_gkeys; v.n_phot = P.n_phot;
        g = tbc::find_bin(v, nu, &tie);
    }
    if (__builtin_expect(g < 0 || tie, 0)) {
        int n_act = 0;
        chi_bf_tot = chi_bf_literal(nu, shell, &n_act);
        ct.g = -1; ct.n_active = n_act;
    } else {
        const double2 cd = P.cb_chi_lin[(size_t)shell * (P.n_phot + 1) + g];
        const double left = g >= 1 ? P.cb_B[g - 1] : 0.0;
        chi_bf_tot = cd.x + cd.y * (nu - left);
        ct.g = g; ct.n_active = P.cb_nact[g];
    }
    ct.boltz = exp(-H_PLANCK * nu / (K_BOLTZMANN * P.t_e[shell]));
    chi_ff = P.ff_opac_const * P.ff_factor[shell] / (nu * nu * nu) * (1 - ct.boltz);
}

// update_estimators_bound_free (radfield_estimator_calcs.py:57-124): free-free heating to the replica row, and the
// trace's seven moments to its (shell, bin) cell -- or the literal per-continuum reductions (ct.g < 0).
__device__ __forceinline__ void bf_estimators(double comov_nu, double comov_energy, int shell, double distance, double chi_ff,
                                              const ContTrace &ct, double *ffh, unsigned long long &n_updates) {
    const KParams &P = cP;
    red_f64(&ffh[shell], comov_energy * distance * chi_ff);
    n_updates += (unsigned long long)ct.n_active;
    if (ct.n_active == 0) return;
    if (__builtin_expect(ct.g < 0, 0)) { bf_estimators_literal(comov_nu, comov_energy, shell, distance, ct.boltz); return; }
    const tbc::TraceMoments tm = tbc::trace_moments(comov_nu, comov_energy, distance, ct.boltz, P.cb_B[ct.g - 1]);  // n_active > 0 => g >= 1
    double *m = P.cb_mom + ((size_t)shell * (P.n_phot + 1) + ct.g) * tbc::N_MOMENTS;
#pragma unroll
    for (int q = 0; q < 7; q++) red_f64(m + q, tm.m[q]);
}


// bound_free_emission + sample_nu_free_bound (interaction_events.py:40-92)
__device__ __forceinline__ void bound_free_emission(Lane &p, Rng &rng, int continuum_id) {
    const KParams &P = cP;
    if (continuum_id < 0 || continuum_id >= P.n_continua) { atomicMax(P.error, ERR_CONTINUUM); return; }
    const double velocity = p.r / P.t_exp;
    const double inv_doppler = inverse_doppler_factor<true>(velocity, p.mu);
    const int start = P.pi_refs[continuum_id], n = P.pi_refs[continuum_id + 1] - start;
    const double *pn = P.phot_nus + start;
    const double *em = P.emiss_t + (size_t)p.shell * P.phot_pad + start;
    const double zrand = rng.next_double<true>();
    int lo = 0, hi = n;  // searchsorted(em, zrand, side='right'): first idx with em[idx] > zrand
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (em[mid] <= zrand) lo = mid + 1; else hi = mid;
    }
    int idx = lo;
    if (idx >= n) { atomicMax(P.error, ERR_CONTINUUM); idx = n - 1; }
    const int im1 = (idx == 0) ? n - 1 : idx - 1;
    const double comov_nu = pn[idx] - (em[idx] - zrand) / (em[idx] - em[im1]) * (pn[idx] - pn[im1]);
    p.nu = comov_nu * inv_doppler;
    p.next_line = first_line_below(comov_nu);  // get_current_line_id (:21-37), not clamped
    p.mu = aberration_cmf_to_lf(p.r, P.t_exp, p.mu);
}

// free_free_emission + sample_nu_free_free (interaction_events.py:141-180)
__device__ __forceinline__ void free_free_emission(Lane &p, Rng &rng) {
    const KParams &P = cP;
    const double velocity = p.r / P.t_exp;
    const double inv_doppler = inverse_doppler_factor<true>(velocity, p.mu);
    const double temperature = P.t_e[p.shell];
    const double zrand = rng.next_double<true>();
    const double comov_nu = -K_BOLTZMANN * temperature / H_PLANCK * log(zrand);
    p.nu = comov_nu * inv_doppler;
    p.next_line = first_line_below(comov_nu);
    p.mu = aberration_cmf_to_lf(p.r, P.t_exp, p.mu);
}

// macro_atom_event, CONTINUUM_PROCESSES_ENABLED branch: one jump of the absorbing Markov chain, then one deactivation
// channel of the absorbing state (macro_atom_interaction_iip).  Both searches bisect running sums that are accumulated
// in the reference's order, so the selected indices are the reference's.
__device__ __noinline__ void macro_atom_event_iip(Lane &p, Rng &rng, int level, unsigned long long &n_jumps, unsigned long long &n_scanned) {
    const KParams &P = cP;
    if (level < 0 || level >= P.n_markov) { atomicMax(P.error, ERR_MACRO_ATOM); return; }
    const double xi = rng.next_double<true>();
    n_jumps++;
    const double *row = P.markov_cum + ((size_t)p.shell * P.n_markov + level) * P.n_markov;
    if (!(row[P.n_markov - 1] > xi)) { n_scanned += (unsigned long long)P.n_markov; atomicMax(P.error, ERR_MACRO_ATOM); return; }
    int lo = 0, hi = P.n_markov - 1;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (row[mid] > xi) hi = mid; else lo = mid + 1;
    }
    const int absorbing = lo;
    n_scanned += (unsigned long long)(absorbing + 1);
    if (absorbing >= P.n_blocks) { atomicMax(P.error, ERR_MACRO_ATOM); return; }
    const int block_start = P.block_edge[absorbing], block_end = P.block_edge[absorbing + 1];
    const double *cum = P.tp_t + (size_t)p.shell * P.tpad;
    const double xe = rng.next_double<true>();
    n_jumps++;
    if (block_end <= block_start || !(cum[block_end - 1] > xe)) {
        n_scanned += (unsigned long long)(block_end - block_start);
        atomicMax(P.error, ERR_MACRO_ATOM);
        return;
    }
    lo = block_start; hi = block_end - 1;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (cum[mid] > xe) hi = mid; else lo = mid + 1;
    }
    n_scanned += (unsigned long long)(lo - block_start + 1);
    const int ttype = P.ttype[lo], tid = P.tline[lo];
    if (ttype == -3 || ttype == -21) free_free_emission(p, rng);                                   // FF_EMISSION, FF_COOLING
    else if (ttype == -2 || ttype == -20 || ttype == -7) bound_free_emission(p, rng, tid);          // BF_EMISSION, FB_COOLING, PHOTO_RECOMB_EMISSION
    else if (ttype == -4) p.status = ST_ADIABATIC_COOLING;                                         // adiabatic_cooling
    else if (ttype == -1) line_emission<true>(p, tid);
    else atomicMax(P.error, ERR_MACRO_ATOM);
}

// One term of chi_bf_contributions on the bins path: entry {k, lo} of the trace's bin (HostBins::act), interpolated with
// phot_interp's weights and operation order, so the value is chi_bf_literal's term for continuum k.
__device__ __forceinline__ double bin_chi_term(int2 e, double nu, const double *chi_row) {
    const KParams &P = cP;
    const double lo = P.phot_nus[e.y], hi = P.phot_nus[e.y + 1];
    return (chi_row[e.y + 1] * (nu - lo) + chi_row[e.y] * (hi - nu)) / (hi - lo);
}

// continuum_event + determine_continuum_macro_activation_idx + determine_bf_macro_activation_idx
// `trace_nu` is the comoving frequency at the START of the trace: the reference draws the absorbing continuum from the
// chi_bf_contributions it computed there (modes/iip/packet_propagation.py:118-128,231-240), while the ionisation
// fraction uses the comoving frequency at the interaction point.  fraction_bf and the normalisation of the draw use the
// literal cumulative sum at trace_nu in continuum order, the reference's chi_bf_contributions[-1].  The trace's bins
// value C + D (nu - B[g-1]) can differ from it in the last bits, or by far more where chi_bf cancels inside a bin, and
// a draw above sum / bins value would find no continuum.  The trace distance and escat_prob stay on the bins value
// (DESIGN section 2).  `trace_g` is the trace's bin, or -1 when the trace took the literal path (breakpoint tie, tables
// without the bins' structure): then the active continua are searched as chi_bf_literal does, else they are read from
// the bin's list.
__device__ __noinline__ void continuum_event_impl(Lane &p, Rng &rng, double trace_nu, int trace_g, double chi_ff, Counters &c) {
    const KParams &P = cP;
    if (P.last_type || P.events) log_interaction_before(p, IT_CONTINUUM_PROCESS);
    const double velocity = p.r / P.t_exp;
    const double old_dop = doppler_factor<true>(velocity, p.mu);
    p.mu = 2.0 * rng.next_double<true>() - 1.0;
    const double inv_dop = inverse_doppler_factor<true>(velocity, p.mu);
    const double comov_energy = p.energy * old_dop;
    const double comov_nu = p.nu * old_dop;
    p.energy = comov_energy * inv_dop;
    int destination = P.k_packet_idx;
    const double *chi_row = P.chi_bf_t + (size_t)p.shell * P.phot_pad;
    const int2 *act = nullptr;
    int n_list = 0;
    double chi_bf_tot = 0.0;
    if (trace_g >= 0) {
        act = P.cb_act + P.cb_act_start[trace_g];
        n_list = P.cb_act_start[trace_g + 1] - P.cb_act_start[trace_g];
        for (int i = 0; i < n_list; i++) chi_bf_tot += bin_chi_term(act[i], trace_nu, chi_row);
    } else {
        int n_act;
        chi_bf_tot = chi_bf_literal(trace_nu, p.shell, &n_act);
    }
    const double fraction_bf = chi_bf_tot / (chi_bf_tot + chi_ff);
    if (rng.next_double<true>() < fraction_bf) {
        // np.searchsorted(chi_bf_contributions, z): first active continuum with cumsum_i / chi_bf_tot >= z
        const double z = rng.next_double<true>();
        double running = 0.0;
        int active = -1;
        if (trace_g >= 0) {
            for (int i = 0; i < n_list; i++) {
                const int2 e = act[i];
                running += bin_chi_term(e, trace_nu, chi_row);
                if (!(running / chi_bf_tot < z)) { active = e.x; break; }
            }
        } else {
            for (int k = 0; k < P.n_continua; k++) {
                if (trace_nu >= P.pi_min[k] && trace_nu <= P.pi_max[k]) {
                    const PhotInterp w = phot_interp(k, trace_nu);
                    running += (chi_row[w.hi] * w.high_weight + chi_row[w.lo] * w.low_weight) / w.interval;
                    if (!(running / chi_bf_tot < z)) { active = k; break; }
                }
            }
        }
        if (active < 0) { atomicMax(P.error, ERR_CONTINUUM); return; }
        const double fraction_ionization = P.pi_min[active] / comov_nu;
        if (rng.next_double<true>() < fraction_ionization) {
            if (active >= P.n_activation) { atomicMax(P.error, ERR_CONTINUUM); return; }
            destination = P.pi_act[active];
        }
    }
    macro_atom_event_iip(p, rng, destination, c.jumps, c.scanned);
    log_interaction_after(p, IT_CONTINUUM_PROCESS);
    c.cont_ev++;
}
__device__ __forceinline__ void continuum_event(Lane &p, Rng &rng, double trace_nu, int trace_g, double chi_ff, Counters &c) {
    Lane lp = p; Rng lr = rng; Counters lc;
    continuum_event_impl(lp, lr, trace_nu, trace_g, chi_ff, lc);
    p = lp; rng = lr; flush_rare(lc);
}


// ------------------------------------------------------------------------------------------
// Virtual packets, packets/virtual_packet.py:77-386.  Lane-parallel: every lane traces the volley of
// its own packet.  The per-shell line scan of trace_vpacket_within_shell (a pure sum of tau over the
// lines crossed) is replaced by a binary search for the first line beyond the shell boundary -- using
// the reference's own distance formula at every probe, so the break index is identical -- and a
// difference of double-double prefix sums of tau (error << 1 ulp of the sum).
// ------------------------------------------------------------------------------------------
// trace_vpacket (virtual_packet.py:168-245) of ONE virtual packet, literally: the shell-by-shell geometry, the line scan of
// every shell (as a search that uses the reference's own distance formula at every probe, so the break index is the
// reference's) and the Russian roulette.  Returns the energy the packet contributes (already x exp(-tau)).
template <bool FR>
__device__ __noinline__ double trace_vpacket_literal(double p_r, int p_shell, int p_next_line, double v_mu, double v_nu, double v_energy,
                                                     Rng &rng, unsigned long long &n_vsteps) {
    const KParams &P = cP;
    double v_r = p_r;
    int v_shell = p_shell, v_line = p_next_line, v_status = ST_IN_PROCESS;
    double tau_total = 0.0;
    int guard = 0;
    while (true) {
        // trace_vpacket_within_shell, virtual_packet.py:77-165
        int delta_shell;
        double d_b = distance_boundary(v_r, v_mu, P.r_inner[v_shell], P.r_outer[v_shell], delta_shell);
        double chi = P.n_e[v_shell] * P.sigma_thomson;
        double velocity = v_r / P.t_exp;
        double dop = doppler_factor<FR>(velocity, v_mu);
        double comov_nu = v_nu * dop;
        if (FR) chi *= dop;
        double tau_shell = chi * d_b;
        // first line index >= v_line with d_b <= d_line(idx); d_line is non-decreasing in idx
        int lo = v_line, hi = P.n_lines;  // answer in [lo, hi]; hi == n_lines means "no break"
        if (lo < hi) {
            // The last line always breaks (MISS_DISTANCE), so the answer is <= n_lines - 1.  Every probe uses
            // the reference's own distance formula, so the index is the one the sequential scan stops at; the
            // frequency-bucket table only supplies the starting guess (nu_line <= nu_cmf - d_b nu / (c t)).
            const int last = P.n_lines - 1;
            auto pred = [&](int i) -> bool {
                if (i >= last) return true;
                return d_b <= distance_line_literal<FR>(v_r, v_mu, v_nu, comov_nu, false, P.nu_line[i], P.t_exp, P.error);
            };
            int gss = first_line_at_or_below(comov_nu - d_b * v_nu * P.inv_ct);
            gss = gss < lo ? lo : (gss > last ? last : gss);
            if (pred(gss)) {
                hi = gss;
                int step = 1;
                while (hi > lo) {  // walk / gallop down to the first true
                    int probe = hi - step; if (probe < lo) probe = lo;
                    if (pred(probe)) { hi = probe; step <<= 1; }
                    else { lo = probe + 1; break; }
                }
                if (hi <= lo) lo = hi;
            } else {
                lo = gss + 1; hi = gss;
                int step = 1;
                bool found = false;
                while (!found) {  // gallop up; terminates at `last`
                    hi = (hi + step < last) ? hi + step : last;
                    step <<= 1;
                    found = pred(hi);
                    if (!found) lo = hi + 1;
                }
            }
            while (lo < hi) {
                int mid = (lo + hi) >> 1;
                if (pred(mid)) hi = mid; else lo = mid + 1;
            }
            int end = lo;
            n_vsteps += (unsigned long long)(end - v_line + 1);
            const double2 *prow = P.tau_prefix + (size_t)v_shell * (P.lpad + 1);
            double sum_lines = dd_diff(prow[end], prow[v_line]);
            tau_shell = tau_shell + sum_lines;
            v_line = end;
        }
        tau_total += tau_shell;
        // move_packet_across_shell_boundary, packets/movement.py:80-102
        int next_shell = v_shell + delta_shell;
        if (next_shell >= P.n_shells) v_status = ST_EMITTED;
        else if (next_shell < 0) v_status = ST_REABSORBED;
        else v_shell = next_shell;
        if (tau_total > P.tau_russian) {
            double event_random = rng.next_double();
            if (event_random > P.survival_probability) {
                v_energy = 0.0;
                v_status = ST_EMITTED;
            } else {
                v_energy = v_energy / P.survival_probability * exp(-tau_total);
                tau_total = 0.0;
            }
        }
        double new_r = sqrt(v_r * v_r + d_b * d_b + 2.0 * v_r * d_b * v_mu);
        v_mu = (v_mu * v_r + d_b) / new_r;
        v_r = new_r;
        if (v_status == ST_EMITTED) break;
        if (++guard > 4 * P.n_shells + 64) { atomicMax(P.error, ERR_VPACKET_LOOP); break; }
    }
    return v_energy * exp(-tau_total);
}

// add_vpacket_collection_to_histogram (modes/montecarlo_transport.py:166-195) + the optional virtual-packet log
__device__ __forceinline__ void record_vpacket(double v_nu, double v_energy, double init_mu, double p_r, int pid) {
    const KParams &P = cP;
    if (!((v_nu < P.grid0) || (v_nu > P.grid_last))) {
        const double delta_nu = P.grid[1] - P.grid[0];
        const long long idx = (long long)floor((v_nu - P.grid0) / delta_nu);
        red_f64(&P.vhist[idx], v_energy);
    }
    if (P.vlog_nu) {
        const unsigned long long slot = atomicAdd(P.vlog_count, 1ull);
        if ((long long)slot < P.vlog_capacity) {
            P.vlog_nu[slot] = v_nu; P.vlog_energy[slot] = v_energy; P.vlog_mu[slot] = init_mu;
            P.vlog_r[slot] = p_r; P.vlog_pid[slot] = pid;
        }
    }
}

// What trace_vpacket_volley (virtual_packet.py:248-345) fixes once per volley
struct VolleySetup { double mu_min, mu_bin, beta_inner, rp_velocity, rp_doppler; bool on_inner; };
template <bool FR> __device__ __forceinline__ VolleySetup volley_setup(const Lane &p) {
    const KParams &P = cP;
    VolleySetup v;
    const double r_inner0 = P.r_inner[0];
    v.beta_inner = 0.0;
    if (p.r > r_inner0) {
        const double q = r_inner0 / p.r;
        v.mu_min = -sqrt(1 - q * q);
        v.on_inner = false;
        if (FR) v.mu_min = aberration_lf_to_cmf(p.r, P.t_exp, v.mu_min);
    } else {
        v.on_inner = true;
        v.mu_min = 0.0;
        if (FR) { const double inv_t = 1 / P.t_exp; v.beta_inner = r_inner0 * inv_t * INV_C; }
    }
    v.mu_bin = (1.0 - v.mu_min) / P.n_vpackets;
    v.rp_velocity = p.r / P.t_exp;
    v.rp_doppler = doppler_factor<FR>(v.rp_velocity, p.mu);
    return v;
}
// direction, frequency and energy of virtual packet i of the volley (one draw), virtual_packet.py:302-345
struct VpacketStart { double v_mu, v_nu, v_energy; };
template <bool FR> __device__ __forceinline__ VpacketStart vpacket_start(const Lane &p, const VolleySetup &v, int i, Rng &rng) {
    const KParams &P = cP;
    const int nv = P.n_vpackets;
    const double v_mu0 = v.mu_min + i * v.mu_bin + rng.next_double() * v.mu_bin;
    double weight;
    if (v.on_inner) {
        if (!FR) weight = 2 * v_mu0 / nv;
        else weight = 2 * (v_mu0 + v.beta_inner) / (2 * v.beta_inner + 1) / nv;
    } else {
        weight = (1 - v.mu_min) / (2 * nv);
    }
    VpacketStart s;
    s.v_mu = v_mu0;
    if (FR) s.v_mu = aberration_cmf_to_lf(p.r, P.t_exp, s.v_mu);
    const double v_doppler = doppler_factor<FR>(v.rp_velocity, s.v_mu);
    const double ratio = v.rp_doppler / v_doppler;
    s.v_nu = p.nu * ratio;
    s.v_energy = p.energy * weight * ratio;
    return s;
}

// Per-lane volley (scan kernel): every lane traces the volley of its own packet.
template <bool FR>
__device__ __noinline__ void vpacket_volley(const Lane &p, Rng &rng, unsigned long long &n_vp, unsigned long long &n_vsteps) {
    const KParams &P = cP;
    if ((p.nu < P.spawn_start) || (p.nu > P.spawn_end)) return;
    const int nv = P.n_vpackets;
    if (nv == 0) return;
    const VolleySetup vs = volley_setup<FR>(p);
    for (int i = 0; i < nv; i++) {
        const VpacketStart st = vpacket_start<FR>(p, vs, i, rng);
        const double e = trace_vpacket_literal<FR>(p.r, p.shell, p.next_line, st.v_mu, st.v_nu, st.v_energy, rng, n_vsteps);
        n_vp++;
        record_vpacket(st.v_nu, e, st.v_mu, p.r, p.pid);
    }
}


// ------------------------------------------------------------------------------------------
// Virtual packets, warp-cooperative form (jump kernel with virtual packets).
//
// A virtual packet flies straight: its impact parameter b^2 = r^2 (1 - mu^2) is conserved, so at a shell boundary of radius
// R its  mu R = +-sqrt(R^2 - b^2)  is known without walking there.  With s = mu R (signed) at the entry and exit of a shell,
//   d_boundary = s_exit - s_entry,   comoving nu at a point = v_nu (1 - s / (c t))   [x gamma(R) with full relativity],
// the SHELLS A VIRTUAL PACKET CROSSES ARE INDEPENDENT ITEMS: every (virtual packet, shell) pair needs one square root or two,
// one search in the line list (first line at or below the comoving frequency at the exit) and one prefix difference.  What
// stays sequential is the packet's random-number stream: virtual packet i draws its direction after the Russian-roulette
// draws of virtual packets 0..i-1 (virtual_packet.py:221,314).  So the warp advances all its waiting packets by ONE virtual
// packet per step -- lane = packet for the draw and the bookkeeping, lane = ITEM (all shells of all packets, packed) for the
// work:
//   A  lane = packet : draw the direction of virtual packet i; path description {b^2, v_nu, s at the start, first / turning
//                      shell}; the number of shells it will cross
//   B  lane = item   : geometry of the shell, line search (bucket table + one 64-byte window of the line list)
//   D  lane = item   : tau of the lines crossed = double-double prefix difference, + tau of the continuum
//   E  lane = packet : sum tau in shell order, Russian roulette (draws), histogram / log
// The reference walks the same path step by step, rounding r and mu at every boundary (virtual_packet.py:168-245); the
// closed form differs from that walk by ~1e-16 relative in d_boundary and nu, i.e. in tau by ~1e-15 -- and not at all in
// the INDICES, which are decided by a frequency window: a line within 1e-12 nu of the comoving frequency at a boundary (the
// only place where the two roundings could disagree about "crossed or not"; probability ~1e-7 per shell), a non-monotone
// sequence of break indices, or a path that touches the inner boundary sends that virtual packet through
// trace_vpacket_literal -- the reference's arithmetic -- instead.
// ------------------------------------------------------------------------------------------
constexpr int VOL_ITEMS = 320;              // item slots per warp and sub-batch (8 packets x 2 x 20 shells)
// doubles per warp: tau[VOL_ITEMS] | e int[VOL_ITEMS] | who u16[VOL_ITEMS] | b2, vnu, s0, r0 [32] each | meta int[32]
__host__ __device__ constexpr int vol_doubles_per_warp(bool) { return VOL_ITEMS + VOL_ITEMS / 2 + VOL_ITEMS / 4 + 4 * 32 + 16; }

struct VolView {
    double *tau;                 // [VOL_ITEMS] tau of the continuum, then of the whole shell
    int *e;                      // [VOL_ITEMS] break index
    unsigned short *who;         // [VOL_ITEMS] owner lane | k << 5
    double *b2, *vnu, *s0, *r0;  // [32] per packet: impact parameter^2, frequency, mu r and r at the start
    int *meta;                   // [32] start shell | turning shell << 8 | K << 16 | no line scan << 30 | literal << 31
};
__device__ __forceinline__ VolView vol_view() {
    extern __shared__ double s_bulk[];
    double *base = s_bulk + cP.vol_off + (size_t)(threadIdx.x >> 5) * vol_doubles_per_warp(false);
    VolView v;
    v.tau = base;
    v.e = reinterpret_cast<int *>(base + VOL_ITEMS);
    v.who = reinterpret_cast<unsigned short *>(base + VOL_ITEMS + VOL_ITEMS / 2);
    v.b2 = base + VOL_ITEMS + VOL_ITEMS / 2 + VOL_ITEMS / 4; v.vnu = v.b2 + 32; v.s0 = v.vnu + 32; v.r0 = v.s0 + 32;
    v.meta = reinterpret_cast<int *>(v.r0 + 32);
    return v;
}

// first line index in [0, L-1] with nu_line <= nu_stop -- the first line the virtual packet does NOT reach in this shell --
// or -1 when a line lies within 1e-12 nu_stop of nu_stop (only the reference's own arithmetic may decide that case)
__device__ __noinline__ int vp_first_break_search(double nu_stop, int glo, int ghi) {  // bucket larger than the window
    const KParams &P = cP;
    const int last = P.n_lines - 1;
    while (glo < ghi) {
        const int mid = (glo + ghi) >> 1;
        if (P.nu_line[mid] <= nu_stop) ghi = mid; else glo = mid + 1;
    }
    const int g = glo > last ? last : glo;
    const bool sure = (g == last || P.nu_line[g] <= nu_stop * (1.0 - 1e-12)) && (g == 0 || P.nu_line[g - 1] >= nu_stop * (1.0 + 1e-12));
    return sure ? g : -1;
}
__device__ __forceinline__ int vp_first_break(double nu_stop) {
    const KParams &P = cP;
    const int L = P.n_lines, last = L - 1;
    if (!(nu_stop > 0.0)) return -1;
    const long long kb = (__double_as_longlong(nu_stop) >> NU_KEY_SHIFT) - P.nu_key_min;
    if (kb < 0) return last;                          // redder than the whole list: every line is crossed, line L-1 always breaks
    if (kb >= (long long)P.n_keys) return vp_first_break_search(nu_stop, 0, 1);  // bluer than the whole list
    const int glo = P.nu_first_le[kb];
    const int ghi = (kb > 0) ? P.nu_first_le[kb - 1] : L;
    // the window [a, a + 8) starts one or two entries before the bucket (the predecessor of the answer must be seen
    // too): four 16-byte loads; the line list is padded by 32 entries, so the window is always mapped
    const int a = (glo > 0 ? glo - 1 : 0) & ~1;
    if (__builtin_expect(ghi - a > 7, 0)) return vp_first_break_search(nu_stop, glo, ghi);  // (ghi itself must be inside the window)
    const double2 *w2 = reinterpret_cast<const double2 *>(P.nu_line + a);
    const double2 q0 = w2[0], q1 = w2[1], q2 = w2[2], q3 = w2[3];
    const double w[8] = {q0.x, q0.y, q1.x, q1.y, q2.x, q2.y, q3.x, q3.y};
    int cnt = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) cnt += (a + k >= glo && a + k < ghi && w[k] > nu_stop);
    int g = glo + cnt;  // first index with nu_line <= nu_stop (== ghi when the whole bucket lies above nu_stop)
    if (g > last) g = last;
    const int ig = g - a, im = g - 1 - a;  // window positions of the answer (<= 7) and of its predecessor (>= 0 unless g == 0)
    double nu_g = w[0], nu_m = w[0];
#pragma unroll
    for (int k = 1; k < 8; k++) { if (ig == k) nu_g = w[k]; if (im == k) nu_m = w[k]; }
    const bool sure = (g == last || nu_g <= nu_stop * (1.0 - 1e-12)) && (g == 0 || nu_m >= nu_stop * (1.0 + 1e-12));
    return sure ? g : -1;
}

// Called by ALL lanes of the warp, converged.  `active`: this lane's packet owes a volley (packet_propagation.py:109-118 at
// birth, :176-230 after an interaction); p / rng are that packet's state (rng advances by the volley's draws).
template <bool FR>
__device__ __noinline__ void warp_volley(bool active, const Lane &p, Rng &rng, unsigned long long &n_vp_out, unsigned long long &n_vsteps_out) {
    const KParams &P = cP;
    extern __shared__ double s_bulk[];  // [4 S] shell table {r_inner, r_outer, chi_e, 1 / chi_e}
    const int lane = threadIdx.x & 31;
    const int nv = P.n_vpackets;
    const int S = P.n_shells, L = P.n_lines;
    active = active && nv > 0 && !((p.nu < P.spawn_start) || (p.nu > P.spawn_end));  // virtual_packet.py:262-266
    if (__ballot_sync(FULL, active) == 0u) return;
    const VolView V = vol_view();
    VolleySetup vs;
    vs.mu_min = 0.0; vs.mu_bin = 0.0; vs.beta_inner = 0.0; vs.rp_velocity = 0.0; vs.rp_doppler = 1.0; vs.on_inner = true;
    if (active) vs = volley_setup<FR>(p);
    // Sub-batches: the items of consecutive lanes are packed into the VOL_ITEMS slots; a lane belongs to sub-batch
    // floor(first item / cap) with cap = VOL_ITEMS - 2 S, so that a sub-batch never holds more than cap + 2 S items
    // (a virtual packet crosses fewer than 2 S shells).  Typically one or two sub-batches per step.
    const int cap = VOL_ITEMS - 2 * S;
    const bool too_many_shells = cap < 1 || S > 255;
    unsigned long long n_vp = 0, n_vsteps = 0;

    for (int i = 0; i < nv; i++) {
        // ---------------- A: lane = packet ----------------
        VpacketStart st;
        st.v_mu = 0.0; st.v_nu = 0.0; st.v_energy = 0.0;
        int K = 0, k_turn = 0;
        bool literal = false;
        if (active) {
            st = vpacket_start<FR>(p, vs, i, rng);
            const double b2 = p.r * p.r * (1.0 - st.v_mu * st.v_mu);
            k_turn = p.shell;
            if (!(st.v_mu > 0.0)) {  // inward while the inner boundary of the shell is reached (calculate_distances.py:40-58)
                while (k_turn >= 0 && s_bulk[k_turn] * s_bulk[k_turn] - b2 >= 0.0) k_turn--;
                if (k_turn < 0) { literal = true; k_turn = 0; }  // would reach the photosphere: not a path virtual packets are launched on
            }
            literal = literal || too_many_shells;
            if (!literal) K = (p.shell - k_turn) + (S - k_turn);
            V.b2[lane] = b2; V.vnu[lane] = st.v_nu; V.s0[lane] = st.v_mu * p.r; V.r0[lane] = p.r;
            V.meta[lane] = p.shell | (k_turn << 8) | (K << 16) | ((p.next_line >= L) ? (1 << 30) : 0);
        } else {
            V.meta[lane] = 0;
        }
        __syncwarp();
        // exclusive scan of K over the warp -> sub-batch of every lane and its first item inside it
        int incl = K;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(FULL, incl, o); if (lane >= o) incl += v; }
        const int excl = incl - K;
        const int my_batch = too_many_shells ? 0 : excl / cap;
        const int n_batches = too_many_shells ? 1 : __shfl_sync(FULL, my_batch, 31) + 1;
        for (int batch = 0; batch < n_batches; batch++) {
            const bool mine = my_batch == batch;
            const unsigned members = __ballot_sync(FULL, mine);
            if (members == 0u) continue;
            const int lead = __ffs(members) - 1, tail = 31 - __clz(members);
            const int first = excl - __shfl_sync(FULL, excl, lead);                      // this lane's first slot in the sub-batch
            const int total = __shfl_sync(FULL, incl, tail) - __shfl_sync(FULL, excl, lead);
            if (mine) for (int k = 0; k < K; k++) V.who[first + k] = (unsigned short)(lane | (k << 5));
            __syncwarp();
            // ---------------- B: lane = item ----------------
            for (int t = lane; t < total; t += 32) {
                const int wk = V.who[t], o = wk & 31, k = wk >> 5;
                const int meta = V.meta[o], s0 = meta & 255, kt = (meta >> 8) & 255, n_in = s0 - kt;
                const double b2 = V.b2[o], v_nu = V.vnu[o];
                // shell of item k, mu R at its entry and exit (R: r_inner at s_bulk[shell], r_outer at s_bulk[S + shell])
                int shell; double s_e, s_x, R_e, R_x;
                if (k < n_in) { shell = s0 - k; R_x = s_bulk[shell]; s_x = -sqrt(R_x * R_x - b2); R_e = s_bulk[S + shell]; s_e = -sqrt(R_e * R_e - b2); }
                else if (k == n_in) { shell = kt; R_x = s_bulk[S + shell]; s_x = sqrt(R_x * R_x - b2); R_e = R_x; s_e = -s_x; }
                else { shell = kt + (k - n_in); R_x = s_bulk[S + shell]; s_x = sqrt(R_x * R_x - b2); R_e = s_bulk[shell]; s_e = sqrt(R_e * R_e - b2); }
                if (k == 0) { s_e = V.s0[o]; R_e = V.r0[o]; }
                const double d_b = s_x - s_e;
                double chi = s_bulk[2 * S + shell], nu_stop;
                if (FR) {
                    const double be = R_e * P.inv_ct, bx = R_x * P.inv_ct;
                    chi *= (1.0 - s_e * P.inv_ct) / sqrt(1.0 - be * be);  // x the Doppler factor at the entry (virtual_packet.py:112-114)
                    nu_stop = v_nu * (1.0 - s_x * P.inv_ct) / sqrt(1.0 - bx * bx);
                } else {
                    nu_stop = v_nu * (1.0 - s_x * P.inv_ct);
                }
                V.tau[t] = chi * d_b;
                int e = L;
                if (!(meta & (1 << 30))) {
                    e = (d_b * P.inv_ct > 1e-11) ? vp_first_break(nu_stop) : -1;
                    if (e < 0) atomicOr(&V.meta[o], (int)0x80000000);
                }
                V.e[t] = e;
            }
            __syncwarp();
            // ---------------- D: lane = item: tau of the lines crossed in shells 1.. of every path (shell 0 starts at the
            // packet's own next_line, which only its lane knows: E adds that one)
            for (int t = lane; t < total; t += 32) {
                const int wk = V.who[t], o = wk & 31, k = wk >> 5;
                const int meta = V.meta[o];
                if (meta < 0 || (meta & (1 << 30)) || k == 0) continue;
                const int s0 = meta & 255, kt = (meta >> 8) & 255, n_in = s0 - kt;
                const int shell = k < n_in ? s0 - k : kt + (k - n_in);
                const int en = V.e[t], stt = V.e[t - 1];
                if (en < stt) { atomicOr(&V.meta[o], (int)0x80000000); continue; }  // not monotone: the literal walk decides
                const double2 *prow = P.tau_prefix + (size_t)shell * (P.lpad + 1);
                V.tau[t] = V.tau[t] + dd_diff(prow[en], prow[stt]);
            }
            __syncwarp();
            // ---------------- E: lane = packet ----------------
            if (mine && active) {
                double energy = 0.0;
                bool walk = literal || V.meta[lane] < 0;
                if (!walk) {
                    double tau_total = 0.0, v_energy = st.v_energy;
                    int cur = p.next_line;
                    for (int k = 0; k < K; k++) {
                        const int t = first + k;
                        double tau_shell = V.tau[t];
                        if (cur < L) {
                            const int en = V.e[t];
                            if (k == 0) {
                                if (en < cur) { walk = true; break; }  // (before any draw of this virtual packet)
                                const double2 *prow = P.tau_prefix + (size_t)p.shell * (P.lpad + 1);
                                tau_shell = tau_shell + dd_diff(prow[en], prow[cur]);
                            }
                            n_vsteps += (unsigned long long)(en - cur + 1);
                            cur = en;
                        }
                        tau_total += tau_shell;
                        if (tau_total > P.tau_russian) {  // virtual_packet.py:214-231
                            const double event_random = rng.next_double();
                            if (event_random > P.survival_probability) { v_energy = 0.0; break; }
                            v_energy = v_energy / P.survival_probability * exp(-tau_total);
                            tau_total = 0.0;
                        }
                    }
                    energy = v_energy * exp(-tau_total);
                }
                if (walk) energy = trace_vpacket_literal<FR>(p.r, p.shell, p.next_line, st.v_mu, st.v_nu, st.v_energy, rng, n_vsteps);
                n_vp++;
                record_vpacket(st.v_nu, energy, st.v_mu, p.r, p.pid);
            }
            __syncwarp();
        }
    }
    n_vp_out += n_vp; n_vsteps_out += n_vsteps;
}


// ------------------------------------------------------------------------------------------
// Pieces of packet_propagation shared by both kernels
// ------------------------------------------------------------------------------------------

// The packet's record at its processing slot (StartRecord): three 16-byte loads
__device__ __forceinline__ int start_from_record(Lane &p, Rng &rng, long long slot) {
    const double2 *rec = reinterpret_cast<const double2 *>(cP.start + slot);
    const double2 rmu = rec[0], nue = rec[1];
    const int4 w = reinterpret_cast<const int4 *>(rec)[2];
    p.pid = w.w; p.r = rmu.x; p.mu = rmu.y; p.nu = nue.x; p.energy = nue.y; p.next_line = w.x;
    p.shell = 0; p.status = ST_IN_PROCESS; p.icount = 0; p.bbuf = -1; p.nev = 0; p.nsteps = 0; p.seg_open = 0;
    rng.start((unsigned)w.y, (unsigned)w.z, (unsigned)w.w);
    return w.w;
}

// make_r_packet (modes/montecarlo_transport.py:41-66) + set_packet_props_{partial,full}_relativity
// (modes/classic/packet_propagation.py:255-318) + RPacket.initialize_line_id (packets/radiative_packet.py:96-110) of
// packet pid: what the ordering pass writes into the packet's StartRecord
template <bool FR>
__device__ __forceinline__ StartRecord start_fields(long long pid, long long seed64) {
    const KParams &P = cP;
    StartRecord s;
    s.pid = (int)pid;
    s.r = P.in_r[pid]; s.mu = P.in_mu[pid]; s.nu = P.in_nu[pid]; s.energy = P.in_energy[pid];
    const uint2 sx = seed_expand(seed64);
    s.seed = sx.x; s.x397 = sx.y;
    double velocity = s.r / P.t_exp;
    double inv_doppler = inverse_doppler_factor<FR>(velocity, s.mu);
    if (FR) {
        double beta = (s.r / P.t_exp) / C_LIGHT;
        s.nu *= inv_doppler; s.energy *= inv_doppler;
        s.mu = (s.mu + beta) / (1 + beta * s.mu);
    } else {
        s.nu *= inv_doppler; s.energy *= inv_doppler;
    }
    // L - searchsorted(nu[::-1], comov_nu, 'left') == #lines with nu_line >= comov_nu
    double dop = doppler_factor<FR>(velocity, s.mu);
    int lo = first_line_below(s.nu * dop);
    if (lo == P.n_lines) lo -= 1;
    s.next_line = lo;
    return s;
}

// the prologue of packet_propagation (modes/classic/packet_propagation.py:99-122) for the packet at processing slot `slot`
// VP = true: the caller traces virtual packets per lane (classic scan kernel).  VP = false (continuum mode; the jump kernels,
// which run theirs warp-cooperatively or not at all): that code, and the registers the call to it would clobber, stay out
// of the kernel
template <bool FR, bool VP = true>
__device__ __noinline__ void start_packet_impl(Lane &p, Rng &rng, long long slot, Counters &c) {
    const KParams &P = cP;
    const int pid = start_from_record(p, rng, slot);
    if (P.last_type) {  // TrackerLastInteraction.__init__, tracker_last_interaction.py:55-82
        const double qnan = __longlong_as_double(0x7ff8000000000000ll);
        P.last_type[pid] = -1; P.last_event_id[pid] = 0; P.last_shell[pid] = -1;
        P.last_absorb[pid] = -1; P.last_emit[pid] = -1;
        P.last_radius[pid] = qnan; P.last_before_nu[pid] = qnan; P.last_before_mu[pid] = qnan;
        P.last_before_energy[pid] = qnan; P.last_after_nu[pid] = qnan; P.last_after_mu[pid] = qnan;
        P.last_after_energy[pid] = qnan;
    }
    if (VP && P.n_vpackets > 0) vpacket_volley<FR>(p, rng, c.vp, c.vsteps);  // packet_propagation.py:109-118
    log_boundary(p, -1, 0);                                             // :120-122
    c.boundary++;
}
template <bool FR, bool VP = true>
__device__ __forceinline__ void start_packet(Lane &p, Rng &rng, long long slot, Counters &c) {
    Lane lp; Rng lr = rng; Counters lc;
    start_packet_impl<FR, VP>(lp, lr, slot, lc);  // sets every field of lp
    p = lp; rng = lr; flush_rare(lc);
}


// J / nu_bar go to one of bulk_reps global replicas [J(S) | nu_bar(S)] (fp64 RED; reduce_bulk_kernel sums them).
// Shared-memory fp64 atomics are compare-and-swap loops that serialise the lanes of a warp sitting in the same shell.
__device__ __forceinline__ double *bulk_replica() {
    const KParams &P = cP;
    return P.bulk_rep + (size_t)((blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) & (P.bulk_reps - 1)) * P.rep_stride;
}

// move_r_packet, packets/movement.py:31-76 + update_estimators_bulk, radfield_estimator_calcs.py:25-53
template <bool FR, bool SMEM = false>
__device__ __forceinline__ void move_and_bulk(Lane &p, double distance, double *s_J, double *s_nubar) {
    const KParams &P = cP;
    if (++p.nsteps > MAX_EVENTS_PER_PACKET) atomicMax(P.error, ERR_STUCK);
    double velocity = p.r / P.t_exp;
    double dop = doppler_factor<FR>(velocity, p.mu);
    double r = p.r;
    if (distance > 0.0) {
        double new_r = sqrt(r * r + distance * distance + 2.0 * r * distance * p.mu);
        p.mu = (p.mu * r + distance) / new_r;
        p.r = new_r;
        double cnu = p.nu * dop;
        double cen = p.energy * dop;
        double dd = distance;
        if (FR) dd *= dop;
        if (SMEM) {  // scan kernel: per-CTA rows in shared memory
            atomicAdd(&s_J[p.shell], cen * dd);
            atomicAdd(&s_nubar[p.shell], cen * dd * cnu);
        } else {     // jump kernels: global replicas (bulk_replica)
            red_f64(&s_J[p.shell], cen * dd);
            red_f64(&s_nubar[p.shell], cen * dd * cnu);
        }
    }
}

// BOUNDARY branch of packet_propagation (:155-174) + move_packet_across_shell_boundary, movement.py:80-102
__device__ __forceinline__ void boundary_event(Lane &p, int delta_shell, Counters &c) {
    const KParams &P = cP;
    log_boundary(p, p.shell, p.shell + delta_shell);
    c.boundary++;
    int next_shell = p.shell + delta_shell;
    if (next_shell >= P.n_shells) p.status = ST_EMITTED;
    else if (next_shell < 0) p.status = ST_REABSORBED;
    else p.shell = next_shell;
}

// LINE / ESCATTERING branches of packet_propagation (:176-230)
template <bool FR, bool CONT, bool VP = !CONT>
__device__ __noinline__ void interaction_event_impl(Lane &p, Rng &rng, int itype, Counters &c) {
    const KParams &P = cP;
    if (itype == IT_LINE) {
        if (P.last_type || P.events) log_interaction_before(p, IT_LINE);
        // line_scatter_event, interaction_event_callers.py:187-239
        double velocity = p.r / P.t_exp;
        double old_dop = doppler_factor<FR>(velocity, p.mu);
        p.mu = 2.0 * rng.template next_double<CONT>() - 1.0;  // get_random_mu, utils.py:14-15
        double inv_new = inverse_doppler_factor<FR>(velocity, p.mu);
        double cen = p.energy * old_dop;
        p.energy = cen * inv_new;
        if (P.line_mode == 0) {
            line_emission<FR>(p, p.next_line);
        } else {
            double cnu = p.nu * old_dop;
            p.nu = cnu * inv_new;
            if (CONT) macro_atom_event_iip(p, rng, P.line2macro[p.next_line], c.jumps, c.scanned);
            else macro_atom_event<FR>(p, rng, P.macro_entry[p.next_line], c.jumps, c.scanned);
        }
        log_interaction_after(p, IT_LINE);
        c.line_ev++;
    } else {  // IT_ESCATTERING: thomson_scatter, interaction_events.py:184-217
        if (P.last_type || P.events) log_interaction_before(p, IT_ESCATTERING);
        double velocity = p.r / P.t_exp;
        double old_dop = doppler_factor<FR>(velocity, p.mu);
        double cnu = p.nu * old_dop;
        double cen = p.energy * old_dop;
        p.mu = 2.0 * rng.template next_double<CONT>() - 1.0;
        double inv_new = inverse_doppler_factor<FR>(velocity, p.mu);
        p.nu = cnu * inv_new;
        p.energy = cen * inv_new;
        if (FR) p.mu = aberration_cmf_to_lf(p.r, P.t_exp, p.mu);
        log_interaction_after(p, IT_ESCATTERING);
        c.escat_ev++;
    }
    if (VP && P.n_vpackets > 0) vpacket_volley<FR>(p, rng, c.vp, c.vsteps);  // (VP: see start_packet_impl)
}
template <bool FR, bool CONT, bool VP = !CONT>
__device__ __forceinline__ void interaction_event(Lane &p, Rng &rng, int itype, Counters &c) {
    Lane lp = p; Rng lr = rng; Counters lc;
    interaction_event_impl<FR, CONT, VP>(lp, lr, itype, lc);
    p = lp; rng = lr; flush_rare(lc);
}


// end of packet_propagation (:247-251) + set_packet_collection_output, modes/montecarlo_transport.py:70-90
__device__ __forceinline__ void finish_packet(Lane &p, const Rng &rng, Counters &c) {
    const KParams &P = cP;
    red_u64(&counter_replica()[CNT_RNG_DRAWS], (unsigned long long)(rng.n >> 1));  // counted where the packet ends: it may have changed lanes
    log_boundary(p, p.shell, p.shell + 1);
    c.boundary++;
    P.out_nu[p.pid] = p.nu;
    // ADIABATIC_COOLING leaves the -99 the collection was initialised with (modes/montecarlo_transport.py:85-90)
    P.out_energy[p.pid] = (p.status == ST_REABSORBED) ? -p.energy : ((p.status == ST_EMITTED) ? p.energy : -99.0);
    if (P.events && p.pid < P.n_tracked) P.event_counts[p.pid] = p.nev;
    // What the epilogue sums over the finished packets (SURVEY.md §8f rank 2).  Inline on purpose: this kernel family sits at
    // the 128-register limit and the trace loop's allocation is fragile -- the same block as an out-of-line call made the
    // kernel slower.
    if (p.status != ST_ADIABATIC_COOLING) {
        // Simulation.iterate's calculate_filtered_luminosity of the emitted / reabsorbed packets (simulation/base.py:455-466,
        // spectrum/luminosity.py:5-29; x 1 / time_of_simulation on the host): {emitted, emitted in window, reabsorbed, reabsorbed in window}
        double *lum = bulk_replica() + 2 * P.n_shells + (p.status == ST_EMITTED ? 0 : 2);
        red_f64(lum, p.energy);
        if (p.nu > P.lum_nu_start && p.nu < P.lum_nu_end) red_f64(lum + 1, p.energy);
    }
    if (P.spec_emitted && p.status != ST_ADIABATIC_COOLING) {
        // numpy.histogram(nu, bins=grid, weights=energy): bin i covers [grid[i], grid[i+1]), the last bin is closed
        const int nb = P.n_grid - 1;
        const double nu = p.nu;
        if (nb > 0 && nu >= P.grid0 && nu <= P.grid_last) {
            // uniform grid: arithmetic guess, then the edge comparisons decide (what numpy.histogram does too)
            int bin = (int)((nu - P.grid0) * P.inv_dgrid);
            bin = bin < 0 ? 0 : (bin > nb - 1 ? nb - 1 : bin);
            while (bin > 0 && nu < P.grid[bin]) bin--;
            while (bin < nb - 1 && nu >= P.grid[bin + 1]) bin++;
            red_f64((p.status == ST_EMITTED ? P.spec_emitted : P.spec_reabsorbed) + bin, p.energy);
        }
    }
}

__device__ __forceinline__ void flush_block(const Counters &c) {
    const KParams &P = cP;
    const int lane = threadIdx.x & 31;
    __syncthreads();
    unsigned long long vals[CNT_COUNT] = {c.line_steps, c.boundary, c.line_ev, c.escat_ev, c.draws,
                                         c.jumps, c.scanned, c.vp, c.vsteps, c.cont_ev, c.bf_upd, c.probes};
#pragma unroll
    for (int k = 0; k < CNT_COUNT; k++) {
        unsigned long long v = vals[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
        if (lane == 0 && v) atomicAdd(&P.counters[k], v);
    }
}

// ------------------------------------------------------------------------------------------
// The kernel
// ------------------------------------------------------------------------------------------
// Common: persistent warps, one RPacket per lane, packets pulled from a global counter in batches.
struct WarpFeed {
    bool exhausted = false;
    template <bool FR, bool ESCAPE = false, bool VP = true>
    __device__ __forceinline__ void refill(Lane &p, Rng &rng, bool &has, unsigned busy_mask, Counters &c) {
        bool done = false;
        refill<FR, ESCAPE, VP>(p, rng, has, busy_mask, c, done);
    }
    // returns with `has` set for lanes that received a packet
    // `done`: the lane still holds a packet that has left the grid and waits for finish_packet; such lanes count as
    // free, and they are finished here, together, right before the batch of new packets is started.
    // ESCAPE (scan kernel): call the out-of-line paths on the packet state itself.  That keeps Lane / Rng / Counters in
    // local memory for the whole kernel -- right for the scan kernel, whose registers belong to the cooperative line scan
    // (with the state in registers it spills 540 B at 3 CTAs/SM and loses 8 % of its bandwidth).
    template <bool FR, bool ESCAPE = false, bool VP = true>
    __device__ __forceinline__ void refill(Lane &p, Rng &rng, bool &has, unsigned busy_mask, Counters &c, bool &done) {
        const KParams &P = cP;
        const int lane = threadIdx.x & 31;
        const unsigned freemask = ~busy_mask;
        // Refill in batches: starting a packet (the record load, trackers, first virtual-packet volley) is a scalar
        // detour for the whole warp, so wait until refill_min lanes are free (or the warp is empty).
        if (!exhausted && !(__popc(freemask) >= P.refill_min || freemask == FULL)) return;
        if (done) { finish_packet(p, rng, c); done = false; }
        if (exhausted) return;
        const int nfree = __popc(freemask);
        unsigned long long base = 0;
        if (lane == 0) base = atomicAdd(P.next_packet, (unsigned long long)nfree);
        base = __shfl_sync(FULL, base, 0);
        if (base + (unsigned long long)nfree >= (unsigned long long)P.n_packets) exhausted = true;
        if (!has) {
            const unsigned long long slot = base + (unsigned long long)__popc(freemask & ((1u << lane) - 1u));
            if (slot < (unsigned long long)P.n_packets) {
                if (ESCAPE) start_packet_impl<FR, VP>(p, rng, (long long)slot, c); else start_packet<FR, VP>(p, rng, (long long)slot, c);
                has = true;
            }
        }
    }
};

// per-lane set-up of trace_packet (homologous_rad_packet_transport.py:76-98)
struct TraceSetup {
    double d_boundary, tau_event, comov_nu, chi;
    double chi_bf_tot, chi_ff, escat_prob, dop, boltz;  // continuum mode only
    int delta_shell;
    int cg, cn;                                         // continuum mode only: ContTrace {g, n_active}
};
// the continuum-mode fields as a classic-mode trace leaves them (trace_setup sets them in continuum mode)
__device__ __forceinline__ void clear_continuum_fields(TraceSetup &t) {
    t.chi_bf_tot = 0.0; t.chi_ff = 0.0; t.escat_prob = 1.0; t.dop = 1.0; t.boltz = 0.0; t.cg = -1; t.cn = 0;
}

// [4 S] shell table at the head of the jump kernels' dynamic shared memory {r_inner, r_outer, chi_e, 1 / chi_e} (see
// trace_setup).  The caller synchronises the CTA before reading it.
__device__ __forceinline__ void load_shell_table() {
    const KParams &P = cP;
    extern __shared__ double s_bulk[];
    for (int i = threadIdx.x; i < P.n_shells; i += blockDim.x) {
        const double chi_e = P.n_e[i] * P.sigma_thomson;
        s_bulk[i] = P.r_inner[i]; s_bulk[P.n_shells + i] = P.r_outer[i];
        s_bulk[2 * P.n_shells + i] = chi_e; s_bulk[3 * P.n_shells + i] = 1.0 / chi_e;
    }
}
// GEO (jump kernels): shell radii and the electron-scattering opacity come from the [4][S] table the kernel copied to
// the head of dynamic shared memory {r_inner, r_outer, chi_e, 1 / chi_e} -- they start the dependent chain of every
// trace, and the L1 (31 % hit rate under this access pattern) does not keep even 20-entry arrays resident.
template <bool FR, bool CONT, bool GEO>
__device__ __forceinline__ void trace_setup(const Lane &p, Rng &rng, TraceSetup &t) {
    const KParams &P = cP;
    extern __shared__ double s_bulk[];
    const double r_in = GEO ? s_bulk[p.shell] : P.r_inner[p.shell];
    const double r_out = GEO ? s_bulk[P.n_shells + p.shell] : P.r_outer[p.shell];
    t.d_boundary = distance_boundary(p.r, p.mu, r_in, r_out, t.delta_shell);
    const double velocity = p.r / P.t_exp;
    const double dop = doppler_factor<FR>(velocity, p.mu);
    t.comov_nu = p.nu * dop;
    t.chi = GEO ? s_bulk[2 * P.n_shells + p.shell] : P.n_e[p.shell] * P.sigma_thomson;  // chi_electron_calculator, opacities/opacities.py:50-67
    if (CONT) {
        // modes/iip/packet_propagation.py:118-149: chi_continuum = chi_e + chi_bf + chi_ff, escat_prob = chi_e / chi_continuum
        double chi_bf_tot, chi_ff;  // locals, so that `t` itself never has its address passed to a real call
        ContTrace ct;
        chi_continuum(t.comov_nu, p.shell, chi_bf_tot, chi_ff, ct);
        t.chi_bf_tot = chi_bf_tot; t.chi_ff = chi_ff; t.boltz = ct.boltz; t.cg = ct.g; t.cn = ct.n_active;
        const double chi_cont = t.chi + t.chi_bf_tot + t.chi_ff;
        t.escat_prob = t.chi / chi_cont;
        t.chi = chi_cont;
        t.dop = dop;
    }
    if (FR) t.chi *= dop;                       // packet_propagation.py:139-140
    t.tau_event = -log(rng.template next_double<CONT>());      // first draw of trace_packet (homologous_rad_packet_transport.py:84)
}

// update_estimators_bound_free of the trace that just ended (modes/iip/packet_propagation.py:157-168): comoving energy,
// path length and free-free opacity carry the Doppler factor of the trace start
__device__ __forceinline__ void trace_bf_estimators(const Lane &p, const TraceSetup &t, double distance, double *ffh, unsigned long long &n_updates) {
    ContTrace ct;
    ct.boltz = t.boltz; ct.g = t.cg; ct.n_active = t.cn;
    bf_estimators(t.comov_nu, p.energy * t.dop, p.shell, distance * t.dop, t.chi_ff * t.dop, ct, ffh, n_updates);
}

// A trace that stops on the continuous opacity is an electron scattering with probability escat_prob, else a continuum
// process (homologous_rad_packet_transport.py:126-135,160-167): one extra random number, drawn after tau_event.
template <bool CONT>
__device__ __forceinline__ int resolve_continuum_type(int itype, const TraceSetup &t, Rng &rng) {
    if (CONT && itype == IT_ESCATTERING) {
        const double zrand = rng.template next_double<CONT>();
        if (!(zrand < t.escat_prob)) return IT_CONTINUUM_PROCESS;
    }
    return itype;
}

// ------------------------------------------------------------------------------------------
// Kernel "scan": the line list is streamed, 32 lines per warp step.
// ------------------------------------------------------------------------------------------
template <bool FR, int MIN_CTAS, bool CONT>
__global__ void __launch_bounds__(256, MIN_CTAS) transport_scan_kernel() {
    const KParams &P = cP;
    extern __shared__ double s_bulk[];  // [2 S] per-CTA J and nu_bar rows (this kernel: 3 % faster than the global replicas)
    for (int i = threadIdx.x; i < 2 * P.n_shells; i += blockDim.x) s_bulk[i] = 0.0;
    __syncthreads();
    double *s_J = s_bulk, *s_nubar = s_bulk + P.n_shells;
    double *s_ffh = bulk_replica() + 2 * P.n_shells + 4;

    const int lane = threadIdx.x & 31;
    Rng rng;
    rng.start(0u, 0u, 0u);
    rng.ring = threadIdx.x & 31;
    Lane p = idle_lane();
    bool has = false;
    WarpFeed feed;
    Counters c;
    const int L = P.n_lines;

    while (true) {
        feed.refill<FR, true, !CONT>(p, rng, has, __ballot_sync(FULL, has), c);
        if (__ballot_sync(FULL, has) == 0u) break;
        // A physics error anywhere aborts the whole run, like the exception the reference raises
        // from inside its prange (utils.py:10, macro_atom.py:15): stop feeding and drain.
        if (*((volatile int *)P.error) != 0) break;

        TraceSetup t;
        t.d_boundary = 0.0; t.tau_event = 0.0; t.comov_nu = 0.0; t.chi = 1.0; t.delta_shell = 0;
        clear_continuum_fields(t);
        double distance = 0.0, tau_excl_res = 0.0;
        int itype = 0;
        bool need_scan = false;
        if (has) {
            trace_setup<FR, CONT, false>(p, rng, t);
            if (p.next_line >= L) {
                // ran off the end of the list, homologous_rad_packet_transport.py:157-172
                double d_cont = t.tau_event / t.chi;
                if (d_cont < t.d_boundary) { distance = d_cont; itype = IT_ESCATTERING; }
                else { distance = t.d_boundary; itype = IT_BOUNDARY; }
            } else {
                need_scan = true;
            }
        }

        // ================= cooperative line scan, one lane's packet at a time =================
        unsigned todo = __ballot_sync(FULL, need_scan);
        while (todo) {
            const int j = __ffs(todo) - 1;
            todo &= todo - 1u;
            const int start = __shfl_sync(FULL, p.next_line, j);
            const int shell = __shfl_sync(FULL, p.shell, j);
            const double b_comov = shfl_d(t.comov_nu, j);
            const double b_nu = shfl_d(p.nu, j);
            const double b_db = shfl_d(t.d_boundary, j);
            const double b_tau_event = shfl_d(t.tau_event, j);
            const double b_chi = shfl_d(t.chi, j);
            const double b_energy = shfl_d(p.energy, j);
            const double b_mu = shfl_d(p.mu, j);
            const double b_r = shfl_d(p.r, j);
            const double inv_nu = 1.0 / b_nu;
            const double d_scale = P.ct * inv_nu;
            const double inv_chi = 1.0 / b_chi;
            const double mur = b_mu * b_r;
            const double *tau_row = P.tau_t + (size_t)shell * P.lpad;
            double *jb_row = P.jblue_t + (size_t)shell * P.lpad;
            double *ed_row = P.edotlu_t + (size_t)shell * P.lpad;

            int base = start & ~31;
            double carry = 0.0;
            int res_line = start, res_type = 0;
            double res_excl = 0.0;
            // software prefetch of the first chunk
            double nu_l = P.nu_line[base + lane];
            double tau_l = tau_row[base + lane];
            while (true) {
                const int line = base + lane;
                const bool valid = (line >= start) && (line < L);
                // prefetch next chunk (speculative; rows are padded so the address is always mapped)
                const int nbase = (base + 32 < P.lpad) ? base + 32 : base;
                const double nu_next = P.nu_line[nbase + lane], tau_next = tau_row[nbase + lane];

                if (!valid) tau_l = 0.0;
                double d;
                const double nu_diff = b_comov - nu_l;
                if (line == L - 1) {
                    d = MISS_DISTANCE;
                } else if (fabs(nu_diff) * inv_nu < CLOSE_LINE_THRESHOLD) {
                    d = 0.0;
                } else {
                    if (valid && !(nu_diff >= 0)) atomicMax(P.error, ERR_NU_DIFF);
                    if (FR) d = distance_line_full_relativity(nu_l, b_nu, P.t_exp, b_r, b_mu);
                    else d = line_distance_partial(nu_diff, d_scale, b_nu, b_db);
                }
                // inclusive warp prefix sum of tau
                double incl = tau_l;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    double v = shfl_up_d(incl, o);
                    if (lane >= o) incl += v;
                }
                incl += carry;
                double excl = shfl_up_d(incl, 1);
                if (lane == 0) excl = carry;
                const double d_cont = (b_tau_event - excl) * inv_chi;
                const bool p1 = valid && (d != 0.0) && (fmin(b_db, d_cont) <= d);
                const bool p2 = valid && !p1 && !P.disable_line && (incl + b_chi * d > b_tau_event);
                const unsigned m = __ballot_sync(FULL, p1 || p2);
                const int f = m ? (__ffs(m) - 1) : 32;
                const bool upd = valid && (lane < f || (lane == f && p2));
                if (upd) {
                    // update_estimators_line, estimators/radfield_estimator_calcs.py:128-164
                    double e = FR ? b_energy : b_energy * (1.0 - (d + mur) * P.inv_ct);
                    red_f64(&jb_row[line], e * inv_nu);
                    red_f64(&ed_row[line], e);
                }
                const unsigned um = __ballot_sync(FULL, upd);
                if (lane == 0) c.line_steps += (unsigned long long)__popc(um);
                if (m) {
                    int my_type = p1 ? ((b_db <= d_cont) ? IT_BOUNDARY : IT_ESCATTERING) : IT_LINE;
                    res_type = __shfl_sync(FULL, my_type, f);
                    res_excl = shfl_d(excl, f);
                    res_line = base + f;
                    break;
                }
                carry = shfl_d(incl, 31);
                base += 32;
                if (base >= P.lpad) { res_type = IT_BOUNDARY; res_line = L - 1; break; }  // unreachable: line L-1 always breaks
                nu_l = nu_next; tau_l = tau_next;
            }
            if (lane == j) { p.next_line = res_line; itype = res_type; tau_excl_res = res_excl; }
        }

        // ================= per-lane event handling (packet_propagation.py:155-245) =================
        if (has) {
            if (need_scan) {
                if (itype == IT_BOUNDARY) distance = t.d_boundary;
                else if (itype == IT_ESCATTERING) distance = (t.tau_event - tau_excl_res) / t.chi;
                else distance = distance_line_literal<FR>(p.r, p.mu, p.nu, t.comov_nu, false, P.nu_line[p.next_line], P.t_exp, P.error);
            }
            itype = resolve_continuum_type<CONT>(itype, t, rng);
            if (CONT) trace_bf_estimators(p, t, distance, s_ffh, c.bf_upd);
            move_and_bulk<FR, true>(p, distance, s_J, s_nubar);
            if (itype == IT_BOUNDARY) boundary_event(p, t.delta_shell, c);
            else if (CONT && itype == IT_CONTINUUM_PROCESS) continuum_event_impl(p, rng, t.comov_nu, t.cg, t.chi_ff, c);
            else interaction_event_impl<FR, CONT>(p, rng, itype, c);  // (on the state itself: see WarpFeed::refill)
            if (p.status != ST_IN_PROCESS) { finish_packet(p, rng, c); has = false; }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < P.n_shells; i += blockDim.x) {
        if (s_J[i] != 0.0) red_f64(&P.J[i], s_J[i]);
        if (s_nubar[i] != 0.0) red_f64(&P.nubar[i], s_nubar[i]);
    }
    flush_block(c);
}

// ------------------------------------------------------------------------------------------
// Kernel "jump".  Two identities remove the O(lines) scan:
//  (1) all three stopping conditions of trace_packet are monotone in the line index, so the end of a trace is
//      found by search over the double-double tau prefix table;
//  (2) E * (1 - (d_i + mu r)/(c t)) == E * nu_i / nu exactly (d_i = (nu_cmf - nu_i)/nu * c t,
//      nu_cmf = nu (1 - mu r/(c t))), so the per-line estimator updates of one trace are two RANGE updates:
//      Edotlu[i] = nu_i * sum_t E_t/nu_t,  J_blue[i] = nu_i * sum_t E_t/nu_t^2  over the traces t passing line i,
//      accumulated in exact fixed-point difference arrays and finished by finalize_line_estimators_kernel.
// The event loop has two phases to keep lanes converged: the common case (trace ends at the shell boundary, found
// by the frequency-bucket guess and verified with two exact probes) is handled immediately; lanes whose trace
// needs a real search or ends in an interaction are PARKED and handled together once enough have accumulated.
// ------------------------------------------------------------------------------------------
struct Brk { bool b, p1; double excl, dcont; };

template <bool FR, bool CONT>
struct TraceProbe {
    const Lane &p; const TraceSetup &t; const double2 *prow; double2 p_start;
    double inv_nu, d_scale, inv_chi; int L; unsigned long long &n_probes;
    __device__ __forceinline__ TraceProbe(const Lane &p_, const TraceSetup &t_, unsigned long long &np) : p(p_), t(t_), n_probes(np) {
        const KParams &P = cP;
        L = P.n_lines;
        prow = P.tau_prefix + (size_t)p.shell * (P.lpad + 1);
        p_start = prow[p.next_line];
        inv_nu = 1.0 / p.nu; d_scale = P.ct * inv_nu;
        extern __shared__ double s_bulk[];
        inv_chi = (FR || CONT) ? 1.0 / t.chi : s_bulk[3 * P.n_shells + p.shell];  // the same quotient, computed once per CTA
    }
    // distance to line i as trace_packet sees it (homologous_rad_packet_transport.py:100-117).  In partial relativity
    // the product nu_diff * d_scale, or with EXACT the reference's (nu_diff / nu) * c * t (see line_distance_partial).
    template <bool EXACT = false>
    __device__ __forceinline__ double line_distance(int i, double nu_l) const {
        const double nu_diff = t.comov_nu - nu_l;
        if (i == L - 1) return MISS_DISTANCE;
        if (fabs(nu_diff) * inv_nu < CLOSE_LINE_THRESHOLD) return 0.0;
        if (FR) return distance_line_full_relativity(nu_l, p.nu, cP.t_exp, p.r, p.mu);
        return EXACT ? line_distance_partial_literal(nu_diff, p.nu) : nu_diff * d_scale;
    }
    // partial relativity: the product for line i lies within PR_TIE_MARGIN of d_boundary, where it may fall on the other
    // side of it than the reference's expression
    __device__ __forceinline__ bool near_boundary(int i) const {
        return fabs(line_distance(i, cP.nu_line[i]) - t.d_boundary) <= PR_TIE_MARGIN * t.d_boundary;
    }
    // stopping predicate of trace_packet at line i (homologous_rad_packet_transport.py:100-151)
    template <bool EXACT = false>
    __device__ __forceinline__ Brk probe(int i) const {
        const KParams &P = cP;
        n_probes++;
        const double nu_l = P.nu_line[i];
        const double excl = dd_diff(prow[i], p_start);
        const double incl = dd_diff(prow[i + 1], p_start);
        const double d = line_distance<EXACT>(i, nu_l);
        const double d_cont = (t.tau_event - excl) * inv_chi;
        const bool p1 = (d != 0.0) && (fmin(t.d_boundary, d_cont) <= d);
        const bool p2 = !p1 && !P.disable_line && (incl + t.chi * d > t.tau_event);
        Brk r; r.b = p1 || p2; r.p1 = p1; r.excl = excl; r.dcont = d_cont;
        return r;
    }
    __device__ __forceinline__ Brk operator()(int i) const { return probe<false>(i); }
};

// Lines [start, end) of the packet's shell get their estimator updates from the trace that just ended: +w at start and -w
// at end in the shell's difference row (w1 = E / nu, or E with full relativity; w2 = w1 / nu).  A packet that crosses into
// a neighbouring shell keeps its weight (neither the move nor the crossing changes the lab-frame E and nu) and its next
// range starts at the same column, so "-w at (s, end), +w at (s', end)" is ONE transfer: +w at xfer[s][end] for
// s' = s + 1, -w at xfer[s - 1][end] for s' = s - 1; fold_transfers_kernel later adds xfer[s - 1] - xfer[s] to diff[s].
// A range is opened at its start only when no transfer opened it (p.seg_open), and closed at its end only where the
// weight or the row really ends: an interaction, or the packet leaving the grid.  An empty range that nothing opened adds
// nothing; one that a transfer opened is transferred on or closed like any other (+w and -w at one cell cancel).  The
// words are integers added mod 2^64, so the folded diff equals that of a direct +w / -w pair per trace bit for bit.
// cross: +1 / -1 when the trace ends on an in-grid crossing into shell + cross, else 0.  end >= start.
template <bool FR>
__device__ __forceinline__ void trace_range_end(Lane &p, int start, int end, int cross, Counters &c) {
    const KParams &P = cP;
    if (end <= start && !p.seg_open) return;
    c.line_steps += (unsigned long long)(end - start);
    const double inv_nu = 1.0 / p.nu;
    const double w1 = FR ? p.energy : p.energy * inv_nu;
    const double w2 = w1 * inv_nu;
    const size_t row_words = (size_t)(P.lpad + 1) * 4;
    FixedTerm f;  // one term at a time, converted where it is added: the kernels sit at their register limit
    if (!p.seg_open) {
        unsigned long long *cell = P.diff + (size_t)p.shell * row_words + (size_t)start * 4;
        if (fixed_term(w1, P.scale1, f, P.error)) fixed_add(cell, f, false);
        if (fixed_term(w2, P.scale2, f, P.error)) fixed_add(cell + 2, f, false);
    }
    unsigned long long *cell = (cross != 0 ? P.xfer + (size_t)(p.shell - (cross < 0 ? 1 : 0)) * row_words
                                           : P.diff + (size_t)p.shell * row_words) + (size_t)end * 4;
    const bool negative = cross <= 0;
    if (fixed_term(w1, P.scale1, f, P.error)) fixed_add(cell, f, negative);
    if (fixed_term(w2, P.scale2, f, P.error)) fixed_add(cell + 2, f, negative);
    p.seg_open = cross != 0;
}

// cross argument of trace_range_end for a trace that ends on the boundary towards shell + delta_shell
__device__ __forceinline__ int grid_crossing(const Lane &p, int delta_shell) {
    return (unsigned)(p.shell + delta_shell) < (unsigned)cP.n_shells ? delta_shell : 0;
}

// What a trace that did not end in the common fast way leaves behind for phase B.
// state: 0: trace end known (f = g); 1: first true lies in [start, g-1]; 2: search upwards from g; 3: list exhausted
struct ParkState { TraceSetup t; Brk fb; int g, state; };

// A parked trace in shared memory, one column per field, slot s of `stride` slots (the lane-resident kernel: slot
// threadIdx.x of blockDim.x; the pooled kernel: a pool slot).  Doubles {d_boundary, tau_event, comov_nu, chi, fb.excl,
// fb.dcont} (+ continuum mode {chi_bf_tot, chi_ff, escat_prob, dop, boltz}), ints {g, word} (+ continuum mode {cg, cn})
// with word = state | fb.b << 2 | fb.p1 << 3 | (delta_shell + 1) << 4; bits 9.. of the word belong to the holder.
__host__ __device__ constexpr int trace_nd(bool cont) { return cont ? 11 : 6; }
__host__ __device__ constexpr int trace_ni(bool cont) { return cont ? 4 : 2; }
template <bool CONT>
struct TraceColumns {
    double *d; int *i; int stride;
    __device__ __forceinline__ int &word(int s) const { return i[stride + s]; }
    __device__ __forceinline__ void put(int s, const ParkState &ps, int high_bits) const {
        const int n = stride;
        d[s] = ps.t.d_boundary; d[n + s] = ps.t.tau_event; d[2 * n + s] = ps.t.comov_nu; d[3 * n + s] = ps.t.chi;
        d[4 * n + s] = ps.fb.excl; d[5 * n + s] = ps.fb.dcont;
        if (CONT) {
            d[6 * n + s] = ps.t.chi_bf_tot; d[7 * n + s] = ps.t.chi_ff; d[8 * n + s] = ps.t.escat_prob; d[9 * n + s] = ps.t.dop;
            d[10 * n + s] = ps.t.boltz; i[2 * n + s] = ps.t.cg; i[3 * n + s] = ps.t.cn;
        }
        i[s] = ps.g;
        word(s) = ps.state | (ps.fb.b ? 4 : 0) | (ps.fb.p1 ? 8 : 0) | ((ps.t.delta_shell + 1) << 4) | high_bits;
    }
    __device__ __forceinline__ void get(int s, ParkState &ps) const {
        const int n = stride;
        ps.t.d_boundary = d[s]; ps.t.tau_event = d[n + s]; ps.t.comov_nu = d[2 * n + s]; ps.t.chi = d[3 * n + s];
        ps.fb.excl = d[4 * n + s]; ps.fb.dcont = d[5 * n + s];
        ps.g = i[s];
        const int w = word(s);
        ps.state = w & 3; ps.fb.b = (w & 4) != 0; ps.fb.p1 = (w & 8) != 0; ps.t.delta_shell = ((w >> 4) & 3) - 1;
        if (CONT) {
            ps.t.chi_bf_tot = d[6 * n + s]; ps.t.chi_ff = d[7 * n + s]; ps.t.escat_prob = d[8 * n + s]; ps.t.dop = d[9 * n + s];
            ps.t.boltz = d[10 * n + s]; ps.t.cg = i[2 * n + s]; ps.t.cn = i[3 * n + s];
        } else {
            clear_continuum_fields(ps.t);
        }
    }
};

// Phase A of one packet: set the trace up, guess where it ends, verify.  Returns false when the trace ended at the
// shell boundary (the common case: the packet has been moved and the boundary handled; `has` drops if it left the
// grid), true when the packet must be parked (ps filled, no side effect on the packet or the estimators yet).
template <bool FR, bool CONT, bool DEFER>
__device__ __forceinline__ bool trace_phase_a(Lane &p, Rng &rng, Counters &c, double *s_J, double *s_nubar,
                                              double *s_ffh, ParkState &ps, bool &has) {
    const KParams &P = cP;
    const int L = P.n_lines;
    TraceSetup &t = ps.t;
    clear_continuum_fields(t);
    trace_setup<FR, CONT, true>(p, rng, t);
    const int start = p.next_line;
    ps.g = 0; ps.state = 0;
    ps.fb.b = false; ps.fb.p1 = false; ps.fb.excl = 0.0; ps.fb.dcont = 0.0;
    if (__builtin_expect(start >= L, 0)) {
        // ran off the end of the list, homologous_rad_packet_transport.py:157-172
        const double d_cont = t.tau_event / t.chi;
        if (d_cont < t.d_boundary) { ps.state = 3; return true; }
    } else {
        TraceProbe<FR, CONT> brk(p, t, c.probes);  // issues the load of the prefix entry at `start` early
        {   // MonteCarloException of calculate_distance_line: nu_diff is smallest at the first line
            const double nd0 = t.comov_nu - P.nu_line[start];
            if (__builtin_expect(start != L - 1 && !(fabs(nd0) * brk.inv_nu < CLOSE_LINE_THRESHOLD) && !(nd0 >= 0), 0)) atomicMax(P.error, ERR_NU_DIFF);
        }
        // Guess: most traces end at the shell boundary, i.e. at the first line with
        // nu_line <= nu_b = nu_cmf - d_boundary * nu / (c t).  The bucket table brackets that index; the guess
        // is then verified with the exact predicate, so a bad guess costs time, never correctness.
        // (with full relativity: the comoving frequency at the boundary point, nu * gamma' (1 - mu' beta'))
        double nu_b;
        if (FR) {
            const double r2 = p.r * p.r + t.d_boundary * t.d_boundary + 2.0 * p.r * t.d_boundary * p.mu;
            const double beta2 = r2 * P.inv_ct * P.inv_ct;
            nu_b = p.nu * (1.0 - (p.mu * p.r + t.d_boundary) * P.inv_ct) / sqrt(1.0 - beta2);
        } else {
            nu_b = t.comov_nu - t.d_boundary * p.nu * P.inv_ct;
        }
        int g = first_line_at_or_below(nu_b);
        g = g < start ? start : (g > L - 1 ? L - 1 : g);
        ps.g = g;
        const int gm = (g > start) ? g - 1 : g;
        // Verification of the common case (the trace ends at the shell boundary, right before line g) with ONE prefix
        // entry: E = tau summed over [start, g) is both excl(g) and incl(g-1).  The boundary stops the trace at g iff
        // d_g != 0, d_boundary <= d_g and d_boundary <= d_cont(g); line g-1 does not stop it earlier iff neither of its
        // two conditions holds, where fmin(d_boundary, d_cont(g-1)) == d_boundary because d_cont is non-increasing in
        // the line index (tau >= 0; rounding is monotone).  This is exactly `brk(g).p1 && boundary wins && !brk(g-1).b`.
        bool fast;
        if (!FR) {
            // With the plain products; a distance within PR_TIE_MARGIN of d_boundary, where the product may round to the
            // other side of it than the reference's expression, leaves the fast path and the exact probes below decide.
            c.probes += 1;
            const double nu_g = P.nu_line[g], nu_m = P.nu_line[gm];
            const double E = dd_diff(brk.prow[g], brk.p_start);
            const double d_g = brk.template line_distance<false>(g, nu_g);
            const double dcont_g = (t.tau_event - E) * brk.inv_chi;
            const double tie = PR_TIE_MARGIN * t.d_boundary;
            fast = (d_g != 0.0) && (t.d_boundary + tie < d_g) && (t.d_boundary <= dcont_g);
            if (g > start) {
                const double d_m = brk.template line_distance<false>(gm, nu_m);
                const bool p1m = (d_m != 0.0) && (t.d_boundary - tie <= d_m);
                const bool p2m = !p1m && !P.disable_line && (E + t.chi * d_m > t.tau_event);
                fast = fast && !p1m && !p2m;
            }
        } else {
            // Full relativity: the distance to a line (calculate_distances.py:198-219: a square root and three divisions) is the
            // path length at which the comoving frequency has fallen to nu_line -- strictly decreasing in nu_line -- and nu_b is
            // the comoving frequency at the boundary point, so  d_boundary <= d_line(nu_l)  <=>  nu_l <= nu_b.  The two formulas
            // round to within ~1e2 cm of c t ~ 3e16 cm, i.e. the floating-point comparison of the distances can only disagree
            // with the comparison of the frequencies when |nu_l - nu_b| < ~3e-15 nu_b.  Outside a window of 1e-12 nu_b the
            // frequencies decide (same outcome, no distance evaluated); inside it the literal distances do.
            c.probes += 1;
            const double nu_g = P.nu_line[g], nu_m = P.nu_line[gm];
            const double E = dd_diff(brk.prow[g], brk.p_start);
            const double dcont_g = (t.tau_event - E) * brk.inv_chi;
            const double nu_lo = nu_b * (1.0 - 1e-12), nu_hi = nu_b * (1.0 + 1e-12);
            const bool close_g = (g != L - 1) && (fabs(t.comov_nu - nu_g) * brk.inv_nu < CLOSE_LINE_THRESHOLD);
            bool ok_g;  // (d_g != 0) && (d_boundary <= d_g)
            if (g == L - 1) ok_g = true;                 // MISS_DISTANCE
            else if (close_g) ok_g = false;              // d_g == 0
            else if (nu_g <= nu_lo) ok_g = true;
            else if (nu_g >= nu_hi) ok_g = false;
            else ok_g = t.d_boundary <= brk.line_distance(g, nu_g);
            fast = ok_g && (t.d_boundary <= dcont_g);
            if (fast && g > start) {
                // line g-1 must not stop the trace: not p1 (its distance is 0 or shorter than d_boundary) and not p2
                // (tau through it + chi d_m <= tau_event).  With d_m <= d_boundary - 3e4 cm (the frequency margin) and
                // d_boundary <= (tau_event - E) / chi just established, E + chi d_m < tau_event by ~1e-12: p2 is false.
                const bool close_m = fabs(t.comov_nu - nu_m) * brk.inv_nu < CLOSE_LINE_THRESHOLD;  // (gm < L - 1)
                if (close_m) fast = P.disable_line || !(E > t.tau_event);                  // d_m == 0: p1 false, p2 = E > tau_event
                else if (nu_m >= nu_hi) fast = true;                                       // d_m < d_boundary by the margin
                else if (nu_m <= nu_lo) fast = false;                                      // d_boundary <= d_m: p1
                else {
                    const double d_m = brk.line_distance(gm, nu_m);
                    const bool p1m = (d_m != 0.0) && (t.d_boundary <= d_m);
                    const bool p2m = !p1m && !P.disable_line && (E + t.chi * d_m > t.tau_event);
                    fast = !p1m && !p2m;
                }
            }
        }
        if (__builtin_expect(!fast, 0)) {
            // anything else: the two full probes decide how phase B continues the search
            const Brk bm = brk(gm);
            ps.fb = brk(g);
            if (!ps.fb.b) { ps.state = 2; return true; }
            if ((g > start) && bm.b) { ps.fb = bm; ps.state = 1; return true; }
            ps.state = 0;  // an interaction right at the guessed line
            return true;
        }
        trace_range_end<FR>(p, start, g, grid_crossing(p, t.delta_shell), c);
        p.next_line = g;
    }
    // (start >= L: no range, and none is open -- transfers happen at columns <= L - 1 only, so seg_open implies start < L)
    if (CONT) trace_bf_estimators(p, t, t.d_boundary, s_ffh, c.bf_upd);
    move_and_bulk<FR>(p, t.d_boundary, s_J, s_nubar);
    boundary_event(p, t.delta_shell, c);
    // DEFER: the caller finishes the packet later, together with others (finish_packet on one lane would hold up the warp)
    if (p.status != ST_IN_PROCESS) { if (!DEFER) finish_packet(p, rng, c); has = false; }
    return false;
}

// Phase B of a parked packet: finish the search, apply the estimator range update, move and handle the event.
template <bool FR, bool CONT, bool DEFER, bool ESC>
__device__ __forceinline__ void event_phase_b(Lane &p, Rng &rng, Counters &c, double *s_J, double *s_nubar,
                                              double *s_ffh, const TraceSetup &t, Brk fb, int g, int pk_state, bool &has, int &ev_type) {
    const KParams &P = cP;
    const int L = P.n_lines;
    const int start = p.next_line;
    int itype, end = start;  // end of the estimator range (state 3, list exhausted: none)
    double distance;
    if (pk_state == 3) {
        itype = IT_ESCATTERING;
        distance = t.tau_event / t.chi;
    } else {
        TraceProbe<FR, CONT> brk(p, t, c.probes);
        int lo, hi;
        if (pk_state == 0) { lo = hi = g; }
        else if (pk_state == 1) {  // first true in [start, g-1]; g-1 is true (fb)
            lo = start; hi = g - 1;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                const Brk b = brk(mid);
                if (b.b) { hi = mid; fb = b; } else lo = mid + 1;
            }
        } else {  // gallop upwards from the guess
            int step = 1;
            lo = g + 1; hi = g;
            while (!fb.b && hi < L - 1) {  // line L-1 always breaks (MISS_DISTANCE); the bound guards NaN input
                lo = hi + 1;
                hi = (hi + step < L - 1) ? hi + step : L - 1;
                step <<= 1;
                fb = brk(hi);
            }
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                const Brk b = brk(mid);
                if (b.b) { hi = mid; fb = b; } else lo = mid + 1;
            }
        }
        int f = lo;
        // Partial relativity: the probes compare the product nu_diff * d_scale with d_boundary.  The reference's expression
        // decides differently only for a line whose product lies within PR_TIE_MARGIN of d_boundary, and as the distance
        // grows with the line index, such a line would be f or f - 1: search again with the reference's expression.
        if (!FR && __builtin_expect(brk.near_boundary(f) || (f > start && brk.near_boundary(f - 1)), 0)) {
            lo = start; hi = L - 1;  // line L-1 always stops a trace (MISS_DISTANCE)
            fb = brk.template probe<true>(hi);
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                const Brk b = brk.template probe<true>(mid);
                if (b.b) { hi = mid; fb = b; } else lo = mid + 1;
            }
            f = lo;
        }
        itype = fb.p1 ? ((t.d_boundary <= fb.dcont) ? IT_BOUNDARY : IT_ESCATTERING) : IT_LINE;
        end = fb.p1 ? f : f + 1;
        p.next_line = f;
        if (itype == IT_BOUNDARY) distance = t.d_boundary;
        else if (itype == IT_ESCATTERING) distance = (t.tau_event - fb.excl) / t.chi;
        else distance = distance_line_literal<FR>(p.r, p.mu, p.nu, t.comov_nu, false, P.nu_line[f], P.t_exp, P.error);
    }
    // closed before the interaction changes the weight; a boundary crossing transfers it
    trace_range_end<FR>(p, start, end, itype == IT_BOUNDARY ? grid_crossing(p, t.delta_shell) : 0, c);
    itype = resolve_continuum_type<CONT>(itype, t, rng);
    ev_type = itype;
    if (CONT) trace_bf_estimators(p, t, distance, s_ffh, c.bf_upd);
    move_and_bulk<FR>(p, distance, s_J, s_nubar);
    if (itype == IT_BOUNDARY) boundary_event(p, t.delta_shell, c);
    // (ESC -- continuum kernel, and the classic one when virtual packets are on: the handlers work on the packet state
    // itself, which keeps it in local memory -- see WarpFeed::refill; those kernels are bound by instruction supply)
    else if (CONT && itype == IT_CONTINUUM_PROCESS) {
        if (ESC) continuum_event_impl(p, rng, t.comov_nu, t.cg, t.chi_ff, c);
        else continuum_event(p, rng, t.comov_nu, t.cg, t.chi_ff, c);
    }
    else if (ESC) interaction_event_impl<FR, CONT, false>(p, rng, itype, c);
    else interaction_event<FR, CONT, false>(p, rng, itype, c);
    if (p.status != ST_IN_PROCESS) { if (!DEFER) finish_packet(p, rng, c); has = false; }
}

// Kernel "jump", lane-resident form (when the pools do not fit or with option pooled = 0; classic mode with virtual
// packets): one packet per lane; a parked packet keeps its lane idle until park_min lanes of the warp wait (its trace state waits
// in a per-thread shared-memory column).
// WVOL (classic mode with virtual packets): the volleys run warp-cooperatively (warp_volley).
template <bool FR, int MIN_CTAS, bool CONT, bool WVOL = false>
__global__ void __launch_bounds__(256, MIN_CTAS) transport_jump_kernel() {
    // ESC: the rare handlers work on the packet state itself (see WarpFeed::refill and event_phase_b)
    constexpr bool ESC = CONT || WVOL;
    const KParams &P = cP;
    extern __shared__ double s_bulk[];  // jump kernels: [4 S] shell table, then the parked-lane columns
    load_shell_table();
    __syncthreads();
    double *s_J = bulk_replica(), *s_nubar = s_J + P.n_shells;
    double *s_ffh = s_J + 2 * P.n_shells + 4;

    Rng rng;
    rng.start(0u, 0u, 0u);
    rng.ring = threadIdx.x & 31;
    Lane p = idle_lane();
    bool has = false, parked = false, vpend = false;
    WarpFeed feed;
    Counters c;
    // The state of a PARKED lane (its trace set-up and what the guess already established) waits in shared memory,
    // one column per thread, not in ~20 registers carried through phase A.
    const TraceColumns<CONT> park{s_bulk + P.park_off, reinterpret_cast<int *>(s_bulk + P.park_off + trace_nd(CONT) * blockDim.x),
                                  (int)blockDim.x};

    bool done = false;  // holds a packet that has left the grid; finish_packet runs batched, inside refill
    unsigned pass = 0;
    while (true) {
        const bool had_before = has;
        feed.refill<FR, ESC, false>(p, rng, has, __ballot_sync(FULL, has), c, done);
        if (__ballot_sync(FULL, has || done) == 0u) break;
        if (WVOL) {
            // A packet that owes a volley (at birth, packet_propagation.py:109-118; after a line interaction or an electron
            // scattering, :176-230) WAITS for it: the volleys are run for many packets at once, when vol_min lanes wait or
            // nothing else can run -- the geometry stage of warp_volley is one lane per packet, so it wants the warp full.
            if (has && !had_before) vpend = true;
            const unsigned vm = __ballot_sync(FULL, vpend);
            const unsigned others = __ballot_sync(FULL, has && !vpend);  // runnable or parked
            if (vm != 0u && (__popc(vm) >= P.vol_min || others == 0u)) {
                warp_volley<FR>(vpend, p, rng, c.vp, c.vsteps);
                vpend = false;
            }
        }
        // the error word is a global (uncached) load: look at it every 64th pass only -- an abort may be late, not missed
        if ((++pass & 63u) == 0u && *((volatile int *)P.error) != 0) break;
        const bool had = has;

        // ================= phase A: lanes that are not parked advance by one trace =================
        if (has && !parked && !(WVOL && vpend)) {
            ParkState ps;
            if (trace_phase_a<FR, CONT, true>(p, rng, c, s_J, s_nubar, s_ffh, ps, has)) {
                park.put(threadIdx.x, ps, 0);
                parked = true;
            }
        }

        // ================= phase B: parked lanes, once enough of them wait (or nothing else can run) =================
        const unsigned parked_mask = __ballot_sync(FULL, parked);
        const unsigned runnable = __ballot_sync(FULL, has && !parked && !(WVOL && vpend));
        if (parked_mask != 0u && (__popc(parked_mask) >= P.park_min || runnable == 0u)) {
            int ev_type = IT_BOUNDARY;
            if (parked) {
                ParkState ps;
                park.get(threadIdx.x, ps);
                // (inline on purpose: an out-of-line phase B with copied packet state measured 15 % slower)
                event_phase_b<FR, CONT, true, ESC>(p, rng, c, s_J, s_nubar, s_ffh, ps.t, ps.fb, ps.g, ps.state, has, ev_type);
                parked = false;
            }
            if (WVOL && ev_type != IT_BOUNDARY && has) vpend = true;  // owes a volley now (see above)
        }
        if (had && !has) done = true;
    }
    flush_block(c);
}

// ------------------------------------------------------------------------------------------
// Kernel "jump", pooled form (classic mode).  In the lane-resident form about half of a warp's lanes idle: parked
// lanes wait for company, finished lanes wait for a batched refill.  Here a warp owns 32 lanes PLUS a pool of
// packet contexts in shared memory.  A packet that must be parked is written to a pool slot and its lane goes on
// with another runnable packet at once (taken from the same slot when that held a stashed runnable packet); once
// park_min packets are parked the lanes swap their runnable packets against parked ones (which stashes the runnable
// ones in the very same slots), handle the events, and carry on tracing with the packets they just handled.
// A packet's trajectory does not depend on where it waits: its RNG state, ring id and seg_open bit travel with it.
// Pool slot = [POOL_ND doubles][POOL_NI ints], slot index fastest (conflict-free: lanes use distinct slots): the packet's
// 4 doubles, then its parked trace's doubles; the packet's ints {pid, next_line, shell, icount, bbuf, nev, nsteps, rng n,
// a, b}, the parked trace's ints (TraceColumns, whose word holds the slot's ring id in bits 9..), then seg_open.
// ------------------------------------------------------------------------------------------
__host__ __device__ constexpr int pool_nd(bool cont) { return 4 + trace_nd(cont); }
__host__ __device__ constexpr int pool_ni(bool cont) { return 10 + trace_ni(cont) + 1; }
__host__ __device__ constexpr int pool_bytes_per_slot(bool cont) { return pool_nd(cont) * 8 + pool_ni(cont) * 4 + 4; }  // + one int of the per-warp slot list

template <bool CONT>
struct PoolView {
    double *d; int *i; int *list; int ns;
    // the slot's parked trace (derived where it is used: the pooled kernels sit at their register limit)
    __device__ __forceinline__ TraceColumns<CONT> trace() const { return TraceColumns<CONT>{d + 4 * ns, i + 10 * ns, ns}; }
    // packet part of a slot (the ring id lives in bits 9.. of the trace word and always travels with the context)
    __device__ __forceinline__ void put_packet(int s, const Lane &q, const Rng &r) const {
        d[s] = q.r; d[ns + s] = q.mu; d[2 * ns + s] = q.nu; d[3 * ns + s] = q.energy;
        i[s] = q.pid; i[ns + s] = q.next_line; i[2 * ns + s] = q.shell; i[3 * ns + s] = q.icount; i[4 * ns + s] = q.bbuf;
        i[5 * ns + s] = q.nev; i[6 * ns + s] = q.nsteps; i[7 * ns + s] = (int)r.n; i[8 * ns + s] = (int)r.a; i[9 * ns + s] = (int)r.b;
        i[(10 + trace_ni(CONT)) * ns + s] = q.seg_open;
    }
    __device__ __forceinline__ void get_packet(int s, Lane &q, Rng &r) const {
        q.r = d[s]; q.mu = d[ns + s]; q.nu = d[2 * ns + s]; q.energy = d[3 * ns + s];
        q.pid = i[s]; q.next_line = i[ns + s]; q.shell = i[2 * ns + s]; q.icount = i[3 * ns + s]; q.bbuf = i[4 * ns + s];
        q.nev = i[5 * ns + s]; q.nsteps = i[6 * ns + s]; r.n = (unsigned)i[7 * ns + s]; r.a = (unsigned)i[8 * ns + s]; r.b = (unsigned)i[9 * ns + s];
        q.seg_open = i[(10 + trace_ni(CONT)) * ns + s];
        q.status = ST_IN_PROCESS; r.pid = (unsigned)q.pid;
    }
    __device__ __forceinline__ void put_trace(int s, const ParkState &ps, unsigned ring) const { trace().put(s, ps, (int)(ring << 9)); }
    __device__ __forceinline__ void put_ring(int s, unsigned ring) const { trace().word(s) = (int)(ring << 9); }
    __device__ __forceinline__ unsigned get_ring(int s) const { return (unsigned)trace().word(s) >> 9; }
    // list[k] = index of the k-th set bit of `first`, then of `second` (both uniform across the warp)
    __device__ __forceinline__ void rank_slots(unsigned long long first, unsigned long long second, int lane) const {
        const int nfirst = __popcll(first);
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int j = lane + 32 * h;
            const unsigned long long bit = 1ull << j, below = bit - 1ull;
            if (first & bit) list[__popcll(first & below)] = j;
            else if (second & bit) list[nfirst + __popcll(second & below)] = j;
        }
        __syncwarp();
    }
};

// OR over the warp of one slot bit per participating lane
__device__ __forceinline__ unsigned long long warp_or_slot(bool take, int s) {
    const unsigned lo = __reduce_or_sync(FULL, (take && s < 32) ? (1u << s) : 0u);
    const unsigned hi = __reduce_or_sync(FULL, (take && s >= 32) ? (1u << (s - 32)) : 0u);
    return ((unsigned long long)hi << 32) | lo;
}

template <bool FR, int MIN_CTAS, bool CONT = false>
__global__ void __launch_bounds__(256, MIN_CTAS) transport_pool_kernel() {
    const KParams &P = cP;
    extern __shared__ double s_bulk[];  // [4 S] shell table, then the per-warp pools
    load_shell_table();
    double *s_J = bulk_replica(), *s_nubar = s_J + P.n_shells;
    double *s_ffh = s_J + 2 * P.n_shells + 4;

    const int lane = threadIdx.x & 31;
    const int NS = P.pool_slots;  // 32 + park_min, even, <= 64
    PoolView<CONT> pool;
    {
        char *wbase = reinterpret_cast<char *>(s_bulk + P.park_off) + (size_t)(threadIdx.x >> 5) * NS * pool_bytes_per_slot(CONT);
        pool.d = reinterpret_cast<double *>(wbase);
        pool.i = reinterpret_cast<int *>(pool.d + pool_nd(CONT) * NS);
        pool.list = pool.i + pool_ni(CONT) * NS;
        pool.ns = NS;
    }
    for (int s = lane; s < NS; s += 32) pool.put_ring(s, 32u + (unsigned)s);
    __syncthreads();
    const unsigned long long all_slots = (NS >= 64) ? ~0ull : ((1ull << NS) - 1ull);
    unsigned long long parked = 0ull, stashed = 0ull;  // warp-uniform slot masks (the rest are empty)
    unsigned pass = 0;

    Rng rng;
    rng.start(0u, 0u, 0u);
    rng.ring = (unsigned)lane;
    Lane p = idle_lane();
    bool has = false;
    WarpFeed feed;
    Counters c;

    while (true) {
        // ---- free lanes take stashed runnable packets
        unsigned busy = __ballot_sync(FULL, has);
        if (stashed != 0ull && busy != FULL) {
            pool.rank_slots(stashed, 0ull, lane);
            const int ntake = min(__popc(~busy), __popcll(stashed));
            const int r = __popc(~busy & ((1u << lane) - 1u));
            const bool take = !has && r < ntake;
            int s = 0;
            if (take) {
                s = pool.list[r];
                const unsigned spare = rng.ring;
                rng.ring = pool.get_ring(s);
                pool.get_packet(s, p, rng);
                pool.put_ring(s, spare);
                has = true;
            }
            stashed &= ~warp_or_slot(take, s);
            __syncwarp();
            busy = __ballot_sync(FULL, has);
        }
        // ---- new packets only when nothing runnable is waiting in the pool
        if (stashed == 0ull) {
            // (VP = false: the pooled kernels never run with virtual packets.  The dead call alone costs registers around
            //  it and slows both the classic and the continuum kernels)
            feed.refill<FR, false, false>(p, rng, has, busy, c);
            busy = __ballot_sync(FULL, has);
        }
        if (busy == 0u && parked == 0ull) break;
        if ((++pass & 63u) == 0u && *((volatile int *)P.error) != 0) break;

        // ---- phase A: every lane that holds a packet advances it by one trace
        ParkState ps;
        bool want_park = false;
        // (finish_packet runs at once here: a per-warp queue of finished packets, flushed 16+ at a time, measured 6 % slower)
        if (has) want_park = trace_phase_a<FR, CONT, false>(p, rng, c, s_J, s_nubar, s_ffh, ps, has);

        // ---- park: into a slot that holds a stashed runnable packet (swap, the lane stays busy), else into an empty one
        const unsigned pm = __ballot_sync(FULL, want_park);
        if (pm != 0u) {
            const unsigned long long empty = all_slots & ~(parked | stashed);
            pool.rank_slots(stashed, empty, lane);
            const int nst = __popcll(stashed);
            int s = 0;
            if (want_park) {
                const int r = __popc(pm & ((1u << lane) - 1u));
                s = pool.list[r];
                if (r < nst) {
                    Lane q; Rng qr;
                    qr.ring = pool.get_ring(s);
                    pool.get_packet(s, q, qr);
                    pool.put_packet(s, p, rng);
                    pool.put_trace(s, ps, rng.ring);
                    p = q; rng = qr;
                } else {
                    const unsigned spare = pool.get_ring(s);
                    pool.put_packet(s, p, rng);
                    pool.put_trace(s, ps, rng.ring);
                    rng.ring = spare;
                    has = false;
                }
            }
            const unsigned long long used = warp_or_slot(want_park, s);
            parked |= used;
            stashed &= ~used;
            __syncwarp();
        }

        // ---- phase B: once enough packets are parked (or nothing else can run)
        busy = __ballot_sync(FULL, has);
        const int np = __popcll(parked);
        if (np > 0 && (np >= P.park_min || (busy == 0u && stashed == 0ull))) {
            pool.rank_slots(parked, 0ull, lane);
            const int nb = min(32, np);
            const bool take = lane < nb;
            const bool had = has;
            int s = 0;
            if (take) {
                s = pool.list[lane];
                Lane q; Rng qr; ParkState pk;
                qr.ring = pool.get_ring(s);
                pool.get_packet(s, q, qr);
                pool.trace().get(s, pk);
                if (had) { pool.put_packet(s, p, rng); pool.put_ring(s, rng.ring); }  // stash the runnable packet this lane held
                else pool.put_ring(s, rng.ring);
                p = q; rng = qr; has = true;
                int ev_type;
                event_phase_b<FR, CONT, false, false>(p, rng, c, s_J, s_nubar, s_ffh, pk.t, pk.fb, pk.g, pk.state, has, ev_type);
            }
            const unsigned long long used = warp_or_slot(take, s);
            parked &= ~used;
            stashed |= warp_or_slot(take && had, s);
            __syncwarp();
        }
    }
    flush_block(c);
}

// ------------------------------------------------------------------------------------------
// Table preparation kernels (run once per tb200_set_model)
// ------------------------------------------------------------------------------------------
// (line, shell) strided host layout -> shell-major [S][lpad], zero padded
__global__ void transpose_to_shell_major(const double *src, long long line_stride, long long shell_stride, int n_rows, int n_shells,
                                         int pad, double *dst) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    long long total = (long long)n_shells * pad;
    if (i >= total) return;
    int s = (int)(i / pad), l = (int)(i % pad);
    dst[i] = (l < n_rows) ? src[(long long)l * line_stride + (long long)s * shell_stride] : 0.0;
}

// shell-major [S][lpad] -> reference layout [L][S]
__global__ void transpose_to_line_major(const double *src, int n_rows, int n_shells, int pad, double *dst) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    long long total = (long long)n_rows * n_shells;
    if (i >= total) return;
    int l = (int)(i / n_shells), s = (int)(i % n_shells);
    dst[i] = src[(size_t)s * pad + l];
}

// one warp per shell: double-double exclusive prefix sums of tau along the line list
__global__ void tau_prefix_kernel(const double *tau_t, int n_lines, int lpad, double2 *prefix) {
    const int shell = blockIdx.x;
    const int lane = threadIdx.x;
    const double *row = tau_t + (size_t)shell * lpad;
    double2 *out = prefix + (size_t)shell * (lpad + 1);
    double ch = 0.0, cl = 0.0;  // running total (double-double)
    if (lane == 0) out[0] = make_double2(0.0, 0.0);
    for (int base = 0; base < lpad; base += 32) {
        double xh = (base + lane < n_lines) ? row[base + lane] : 0.0, xl = 0.0;
        // inclusive double-double scan
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            double th = __shfl_up_sync(FULL, xh, o), tl = __shfl_up_sync(FULL, xl, o);
            if (lane >= o) {
                double s = xh + th; double bb = s - xh; double e = (xh - (s - bb)) + (th - bb);
                e += xl + tl;
                xh = s + e; xl = e - (xh - s);
            }
        }
        // add carry
        {
            double s = xh + ch; double bb = s - xh; double e = (xh - (s - bb)) + (ch - bb);
            e += xl + cl;
            xh = s + e; xl = e - (xh - s);
        }
        out[base + lane + 1] = make_double2(xh, xl);
        ch = __shfl_sync(FULL, xh, 31); cl = __shfl_sync(FULL, xl, 31);
    }
}

// Packet processing order: counting sort of the packet indices by a COARSE frequency key of the initial nu (sign,
// exponent and `sort_bits` mantissa bits; original order inside a bucket), so that at any moment all warps of the
// GPU work in the same window of the line list and the per-shell windows of the prefix / difference / estimator
// tables stay L2-resident.  A fine sort is counter-productive at large N: the packets in flight then share their
// start lines and serialise on the same difference-array cells (it measured slower than no sort at all at 1e8 packets).
// Results per packet do not depend on the order.
// (per-block shared-memory counters when the keys fit: with ~90 coarse keys a global atomic per packet would serialise 1e8
//  adds on 90 addresses)
constexpr int ORDER_SMEM_KEYS = 2048, ORDER_ITEMS = 8;
__device__ __forceinline__ int order_key(double nu, int shift, long long key_min, int n_keys) {
    long long k = (__double_as_longlong(nu) >> shift) - key_min;
    return (int)(k < 0 ? 0 : (k >= n_keys ? n_keys - 1 : k));
}
__global__ void order_hist_kernel(const double *nu, long long n, int shift, long long key_min, int n_keys, unsigned *hist) {
    __shared__ unsigned sh[ORDER_SMEM_KEYS];
    const bool local = n_keys <= ORDER_SMEM_KEYS;
    if (local) { for (int k = threadIdx.x; k < n_keys; k += blockDim.x) sh[k] = 0u; __syncthreads(); }
    const long long base = (long long)blockIdx.x * blockDim.x * ORDER_ITEMS;
#pragma unroll
    for (int q = 0; q < ORDER_ITEMS; q++) {
        const long long i = base + (long long)q * blockDim.x + threadIdx.x;
        if (i < n) atomicAdd(local ? &sh[order_key(nu[i], shift, key_min, n_keys)] : &hist[order_key(nu[i], shift, key_min, n_keys)], 1u);
    }
    if (local) { __syncthreads(); for (int k = threadIdx.x; k < n_keys; k += blockDim.x) if (sh[k]) atomicAdd(&hist[k], sh[k]); }
}
// exclusive scan of hist in DESCENDING key order (high nu first = low line index first), single block
__global__ void order_scan_kernel(unsigned *hist, int n_keys) {
    __shared__ unsigned s_carry;
    __shared__ unsigned s_warp[32];
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    for (int base = 0; base < n_keys; base += blockDim.x) {
        const int j = base + threadIdx.x;           // position in descending order
        const int k = n_keys - 1 - j;               // key
        unsigned v = (j < n_keys) ? hist[k] : 0u;
        unsigned x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { unsigned t = __shfl_up_sync(FULL, x, o); if (lane >= o) x += t; }
        if (lane == 31) s_warp[warp] = x;
        __syncthreads();
        if (warp == 0) {
            unsigned w = (lane < nwarps) ? s_warp[lane] : 0u;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { unsigned t = __shfl_up_sync(FULL, w, o); if (lane >= o) w += t; }
            s_warp[lane] = w;
        }
        __syncthreads();
        const unsigned before = s_carry + (warp > 0 ? s_warp[warp - 1] : 0u) + (x - v);
        if (j < n_keys) hist[k] = before;
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) s_carry = before + v;
        __syncthreads();
    }
}
// The pass also writes each packet's StartRecord at its slot (START::at: start_fields of the transport mode), and the seed
// words by packet id for rng_replay_tier1.  Its reads of the packet arrays stay coalesced (i is sequential per thread); the
// transport kernel's refills then read consecutive records.
template <bool FR>
struct ClassicStart {
    __device__ __forceinline__ static StartRecord at(long long pid, long long seed64) { return start_fields<FR>(pid, seed64); }
};
template <class START>
__device__ __forceinline__ void write_start(long long i, long long slot, const long long *seeds64, unsigned *seed32, unsigned *x397,
                                            StartRecord *rec) {
    const StartRecord s = START::at(i, seeds64[i]);
    seed32[i] = s.seed; x397[i] = s.x397;
    rec[slot] = s;
}
// sort_packets = 0: packet i at slot i
template <class START>
__global__ void start_record_kernel(long long n, const long long *seeds64, unsigned *seed32, unsigned *x397, StartRecord *rec) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) write_start<START>(i, i, seeds64, seed32, x397, rec);
}
template <class START>
__global__ void order_scatter_kernel(const double *nu, long long n, int shift, long long key_min, int n_keys, unsigned *cursor,
                                     const long long *seeds64, unsigned *seed32, unsigned *x397, StartRecord *rec) {
    __shared__ unsigned sh[ORDER_SMEM_KEYS];  // count of the block per key, then the block's first slot of the key
    const long long base = (long long)blockIdx.x * blockDim.x * ORDER_ITEMS;
    if (n_keys > ORDER_SMEM_KEYS) {  // too many keys for the block's counters: one global atomic per packet
        for (int q = 0; q < ORDER_ITEMS; q++) {
            const long long i = base + (long long)q * blockDim.x + threadIdx.x;
            if (i < n) write_start<START>(i, atomicAdd(&cursor[order_key(nu[i], shift, key_min, n_keys)], 1u), seeds64, seed32, x397, rec);
        }
        return;
    }
    for (int k = threadIdx.x; k < n_keys; k += blockDim.x) sh[k] = 0u;
    __syncthreads();
    int key[ORDER_ITEMS]; unsigned rank[ORDER_ITEMS];
#pragma unroll
    for (int q = 0; q < ORDER_ITEMS; q++) {
        const long long i = base + (long long)q * blockDim.x + threadIdx.x;
        key[q] = -1; rank[q] = 0u;
        if (i < n) { key[q] = order_key(nu[i], shift, key_min, n_keys); rank[q] = atomicAdd(&sh[key[q]], 1u); }
    }
    __syncthreads();
    for (int k = threadIdx.x; k < n_keys; k += blockDim.x) { const unsigned cnt = sh[k]; sh[k] = cnt ? atomicAdd(&cursor[k], cnt) : 0u; }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < ORDER_ITEMS; q++) {
        const long long i = base + (long long)q * blockDim.x + threadIdx.x;
        if (key[q] >= 0) write_start<START>(i, sh[key[q]] + rank[q], seeds64, seed32, x397, rec);
    }
}

// in-place running sums of the transition probabilities inside each macro-atom block, per shell, in the
// reference's accumulation order (macro_atom.py:79-93)
__global__ void macro_cumsum_kernel(double *tp_t, const int *block_edge, int n_blocks, int n_shells, int tpad) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)n_blocks * n_shells) return;
    const int shell = (int)(i / n_blocks), block = (int)(i % n_blocks);
    double *row = tp_t + (size_t)shell * tpad;
    double acc = 0.0;
    for (int t = block_edge[block]; t < block_edge[block + 1]; t++) { acc += row[t]; row[t] = acc; }
}

// Guide table of the classic macro atom: guide[shell][b0 + k] = first transition of the block [b0, b1) whose running sum
// exceeds k / n (n = b1 - b0 entries, k = 0 .. n-1).  A draw xi then only has to be searched between the guide entries of
// the buckets around floor(xi * n) instead of over the whole block (macro_atom_event).
__global__ void macro_guide_kernel(const double *tp_t, const int *block_edge, int n_blocks, int n_shells, int tpad, int *guide) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)n_blocks * n_shells) return;
    const int shell = (int)(i / n_blocks), block = (int)(i % n_blocks);
    const double *cum = tp_t + (size_t)shell * tpad;
    int *g = guide + (size_t)shell * tpad;
    const int b0 = block_edge[block], b1 = block_edge[block + 1], n = b1 - b0;
    int tid = b0;
    for (int k = 0; k < n; k++) {
        const double thr = (double)k / (double)n;
        while (tid < b1 - 1 && !(cum[tid] > thr)) tid++;
        g[b0 + k] = tid;
    }
}

// macro_next / macro_entry (see MNEXT_EMIT): one thread per transition, then one per line
__device__ __forceinline__ int2 macro_block_of(int level, const int *block_edge, int n_blocks) {
    return (level < 0 || level >= n_blocks) ? make_int2(MNEXT_BAD_LEVEL, 0) : make_int2(block_edge[level], block_edge[level + 1]);
}
__global__ void macro_next_kernel(const int *block_edge, const int *ttype, const int *dest, const int *tline, const int *line2macro,
                                  int n_blocks, int n_transitions, int n_lines, int2 *next, int2 *entry) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_transitions) {
        const int type = ttype[i];
        next[i] = type >= 0 ? macro_block_of(dest[i], block_edge, n_blocks)
                            : (type == -1 ? make_int2(MNEXT_EMIT, tline[i]) : make_int2(MNEXT_BAD_TYPE, 0));
    }
    if (i < n_lines) entry[i] = macro_block_of(line2macro[i], block_edge, n_blocks);
}

// IIP macro atom: running sums of the absorbing-Markov-chain probabilities along the destination axis, in the
// reference's accumulation order (macro_atom.py:131-139)
__global__ void markov_cumsum_kernel(double *markov, long long n_rows, int n) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_rows) return;
    double *row = markov + i * n;
    double acc = 0.0;
    for (int k = 0; k < n; k++) { acc += row[k]; row[k] = acc; }
}

// continuum mode: {value at the left edge, slope} of chi_bf_tot and the number of active continua of every global bin
// (continuum_bins.cuh).  One thread per (shell, bin); chi_bf_t is shell-major [S][phot_pad].
__global__ void continuum_lin_kernel(const double *B, int n_phot, const double *phot_nus, const int *pos, const int *refs, int n_continua,
                                     const double *chi_bf_t, int phot_pad, int n_shells, double2 *chi_lin, int *nact) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)n_shells * (n_phot + 1)) return;
    const int shell = (int)(i / (n_phot + 1)), g = (int)(i % (n_phot + 1));
    double C, D;
    tbc::bin_chi_linear(g, B, n_phot, phot_nus, pos, refs, n_continua, chi_bf_t + (size_t)shell * phot_pad, &C, &D);
    chi_lin[i] = make_double2(C, D);
    if (shell == 0) {
        int n = 0;
        if (g >= 1 && g < n_phot)
            for (int k = 0; k < n_continua; k++) {
                const int cnt = refs[k + 1] - refs[k];
                const int idx = tbc::block_rank(pos, refs[k], cnt, g);
                if (idx >= 1 && idx <= cnt - 1 && phot_nus[refs[k] + idx] - phot_nus[refs[k] + idx - 1] > 0.0) n++;
            }
        nact[g] = n;
    }
}

// continuum mode epilogue: moments of the (shell, bin) cells + what the literal path accumulated -> the five
// [n_continua][S] estimator tables of the packed buffer (overwritten: the moments and cont_lit hold the whole accumulation).
__global__ void continuum_finalize_kernel(const double *mom, const double *lit, const double *B, int n_phot, const double *phot_nus,
                                          const double *x_sect, const int *pos, const int *refs, const double *bf_thr, int n_continua,
                                          int n_shells, int use_bins, double *est) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_continua * n_shells) return;
    const int k = i / n_shells, shell = i % n_shells;
    const size_t ncs = (size_t)n_continua * n_shells;
    double out[5];
#pragma unroll
    for (int q = 0; q < 5; q++) out[q] = lit[q * ncs + i];
    if (use_bins)
        tbc::continuum_estimators_from_moments(k, mom + (size_t)shell * (n_phot + 1) * tbc::N_MOMENTS, B, phot_nus, x_sect, pos, refs, bf_thr[k], out);
#pragma unroll
    for (int q = 0; q < 5; q++) est[q * ncs + i] = out[q];
}

// frequency-bucket table: key(nu) = top 28 bits of the binary64 pattern (sign, exponent, 16 mantissa bits)
// is monotone in nu > 0; first_le[k] = smallest line index whose key - key_min is <= k.
__global__ void nu_bucket_kernel(const double *nu_line, int n_lines, long long key_min, int n_keys, int *first_le) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_lines) return;
    long long k = (__double_as_longlong(nu_line[i]) >> NU_KEY_SHIFT) - key_min;
    long long prev = (i == 0) ? (long long)n_keys : (__double_as_longlong(nu_line[i - 1]) >> NU_KEY_SHIFT) - key_min;
    if (k < 0) k = 0;
    for (long long q = k; q < prev && q < n_keys; q++) first_le[q] = i;
}

// jump algorithm epilogue: exact 128-bit integer prefix sums of the fixed-point difference array along the line
// list, per (shell, quantity), then  estimator[i] = (FR ? 1 : nu_i) * sum_i / scale.
__device__ __forceinline__ __int128 shfl_up_i128(__int128 v, int d) {
    unsigned long long lo = (unsigned long long)v, hi = (unsigned long long)(v >> 64);
    lo = __shfl_up_sync(FULL, lo, d); hi = __shfl_up_sync(FULL, hi, d);
    return (__int128)(((unsigned __int128)hi << 64) | lo);
}
__device__ __forceinline__ double i128_to_double(__int128 v) {
    const bool neg = v < 0;
    unsigned __int128 u = neg ? (unsigned __int128)(-v) : (unsigned __int128)v;
    double d = (double)(unsigned long long)(u >> 64) * 18446744073709551616.0 + (double)(unsigned long long)u;
    return neg ? -d : d;
}
// One CTA of FIN_THREADS threads per (shell, quantity); the row is scanned in tiles of FIN_THREADS entries: warp scans by
// shuffle, a scan of the 32 warp totals in shared memory, a running carry.  (Integer adds: any grouping gives the same sums.
// One WARP per row was a visible share of a step.)
constexpr int FIN_THREADS = 1024;
__global__ void __launch_bounds__(FIN_THREADS) finalize_line_estimators_kernel(const unsigned long long *diff, const double *nu_line, int n_lines, int lpad,
                                                double inv_scale1, double inv_scale2, int full_rel, double *jblue_t, double *edotlu_t, int *error) {
    const int shell = blockIdx.x >> 1, q = blockIdx.x & 1;  // q = 0: w1 -> Edotlu, q = 1: w2 -> J_blue
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned long long *row = diff + (size_t)shell * (lpad + 1) * 4 + q * 2;
    double *out = (q == 0 ? edotlu_t : jblue_t) + (size_t)shell * lpad;
    const double inv_scale = q == 0 ? inv_scale1 : inv_scale2;
    __shared__ unsigned long long tot_lo[32], tot_hi[32];  // inclusive scan of the warp totals of the current tile
    __int128 carry = 0;
    bool negative = false;  // a finished prefix below zero (see the end of the kernel)
    for (int base = 0; base < lpad; base += FIN_THREADS) {
        const int i = base + threadIdx.x;
        __int128 x = 0;
        if (i <= n_lines) {
            const long long hi = (long long)row[(size_t)i * 4], lo = (long long)row[(size_t)i * 4 + 1];
            x = (__int128)hi * (__int128)536870912ll + (__int128)lo;  // FIXED_SPLIT
        }
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            __int128 t = shfl_up_i128(x, o);
            if (lane >= o) x += t;
        }
        if (lane == 31) { tot_lo[warp] = (unsigned long long)x; tot_hi[warp] = (unsigned long long)(x >> 64); }
        __syncthreads();
        if (warp == 0) {
            __int128 t = (__int128)(((unsigned __int128)tot_hi[lane] << 64) | tot_lo[lane]);
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                __int128 u = shfl_up_i128(t, o);
                if (lane >= o) t += u;
            }
            tot_lo[lane] = (unsigned long long)t; tot_hi[lane] = (unsigned long long)(t >> 64);
        }
        __syncthreads();
        if (warp > 0) x += (__int128)(((unsigned __int128)tot_hi[warp - 1] << 64) | tot_lo[warp - 1]);
        x += carry;
        if (i < n_lines) {
            negative |= x < 0;
            double v = i128_to_double(x) * inv_scale;
            out[i] = full_rel ? v : v * nu_line[i];
        } else if (i < lpad) {
            out[i] = 0.0;
        }
        carry += (__int128)(((unsigned __int128)tot_hi[31] << 64) | tot_lo[31]);
        __syncthreads();  // the totals are overwritten by the next tile
    }
    // every range update is a +w / -w pair inside this row: a non-zero total means a 64-bit word wrapped (fixed_add).
    // The total alone misses a wrap that the closing cell mirrors: a true sum of 2^63 + k at a range's first cell reads as
    // -2^63 + k, the -2^63 - k behind its last line as 2^63 - k, and the row still sums to zero (sums over the members of
    // a collective can get there).  But a prefix is a sum of the non-negative weights of the traces that cover the line,
    // so a finished prefix below zero is a wrapped word too.
    // Unless an error already stopped the launch: the packets it was carrying keep the ranges that transfers opened
    // (trace_range_end) unclosed, so the sums say nothing and the error that stopped it is the one to report.
    if (negative || (threadIdx.x == 0 && carry != 0)) atomicCAS(error, 0, ERR_FIXED_POINT);
}

// diff[s] += xfer[s - 1] - xfer[s] element-wise mod 2^64 (the transfers of trace_range_end; xfer has rows 0 .. S - 2).
// One thread per 16 bytes of a row walks down the shells, so every transfer word is read once.
__global__ void fold_transfers_kernel(unsigned long long *diff, const unsigned long long *xfer, int n_shells, size_t row_words) {
    const size_t k = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 2;
    if (k >= row_words) return;
    ulonglong2 below = make_ulonglong2(0ull, 0ull);  // xfer[s - 1]
#pragma unroll 4
    for (int s = 0; s < n_shells; s++) {
        const ulonglong2 above = (s + 1 < n_shells) ? *reinterpret_cast<const ulonglong2 *>(xfer + (size_t)s * row_words + k)
                                                    : make_ulonglong2(0ull, 0ull);
        ulonglong2 *d = reinterpret_cast<ulonglong2 *>(diff + (size_t)s * row_words + k);
        ulonglong2 v = *d;
        v.x += below.x - above.x; v.y += below.y - above.y;
        *d = v;
        below = above;
    }
}

// replicas {J | nu_bar | luminosity sums | ff_heating} -> packed estimator buffer (adds, then clears the replicas)
__global__ void reduce_bulk_kernel(double *rep, int reps, int n_shells, int rep_stride, double *J, double *nubar, double *lum, double *ffh,
                                   unsigned long long *cnt_rep, unsigned long long *counters) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < CNT_COUNT) {
        unsigned long long acc = 0ull;
        for (int r = 0; r < reps; r++) { acc += cnt_rep[(size_t)r * CNT_COUNT + i]; cnt_rep[(size_t)r * CNT_COUNT + i] = 0ull; }
        counters[i] += acc;
    }
    if (i >= rep_stride) return;
    double acc = 0.0;
    for (int r = 0; r < reps; r++) { acc += rep[(size_t)r * rep_stride + i]; rep[(size_t)r * rep_stride + i] = 0.0; }
    if (i < n_shells) J[i] += acc;
    else if (i < 2 * n_shells) nubar[i - n_shells] += acc;
    else if (i < 2 * n_shells + 4) lum[i - 2 * n_shells] += acc;
    else if (ffh) ffh[i - 2 * n_shells - 4] += acc;
}

}  // namespace tb
