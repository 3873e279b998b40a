// engine.cu -- host side of libtardis_b200.so: device memory, table upload, launches, and the C-ABI
// declared in include/tardis_b200.h.  No torch types, no CPU compute path: every entry point that
// does work needs a CUDA device and fails with TB200_ERR_CUDA otherwise.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include <algorithm>

#include "../../include/tardis_b200.h"
#include "device_buffer.cuh"
#include "continuum_bins.cuh"
#include "continuum_macro_build.cuh"
#include "transport_kernel.cuh"
#include "source_function.cuh"
#include "packet_source.cuh"
#include "radfield.cuh"
#include "opacity_build.cuh"
#include "formal_integral.cuh"
#include "markov_build.cuh"
#include "nonhomologous.cuh"
#include "plasma.cuh"

namespace {

#define CK(call)                                                                                     \
    do {                                                                                             \
        cudaError_t err__ = (call);                                                                  \
        if (err__ != cudaSuccess)                                                                    \
            return fail(TB200_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(err__));      \
    } while (0)

inline int round_up(int x, int m) { return (x + m - 1) / m * m; }

}  // namespace

struct tb200_engine {
    int device = 0;
    int sm_count = 132;
    size_t smem_optin = 227 * 1024;  // largest dynamic + static shared memory one CTA may opt in to (H100: 227 KiB)
    // declared before every buffer, so that the buffers are freed first
    Stream stream, h2d_stream, d2h_stream;
    Event ev_start, ev_stop, ev_fin;
    bool have_model = false;
    bool timing_valid = false;
    int64_t launches = 0;
    // options
    int ctas_per_sm = 0, threads_per_cta = 256;  // 0 = the measured best for the kernel that will run (launch_range)
    int refill_min = 0;             // 0 = the measured best for the kernel that will run: pooled classic 12, others 8
    int sort_packets = 1;           // process packets in order of initial frequency (L2 locality); results unchanged
    int sort_bits = 5;              // mantissa bits of the ordering key (coarse buckets)
    int park_min = 0;     // 0 = measured best: 32 for the pooled kernel, 16 with one packet per lane
    int algorithm = 1;  // 0 = scan (stream the line list), 1 = jump (prefix-table search + range updates; default)
    int vol_min = 24;     // warp-cooperative volleys start when this many lanes of a warp wait for one
    int pooled = 1;     // jump, classic mode: packet pool per warp (transport_pool_kernel); 0 = one packet per lane
    int pipeline_chunks = 8;        // tb200_run splits the packets so that H2D / kernel / D2H overlap
    int pipeline_edges = 1;         // short first and last range (their copies are the exposed ones)
    double nu_typ = 1.0;
    double chunk_kernel_ms = 0.0;   // sum over the chunks of the last pipelined tb200_run
    bool chunked_timing = false;

    // model
    int S = 0, L = 0, lpad = 0, T = 0, tpad = 0, n_blocks = 0, n_grid = 0;
    tb200_config cfg{};
    double t_exp = 0;
    DBuf<double> r_inner, r_outer, n_e, nu_line, tau_t, tp_t, grid, staging;
    DBuf<double2> prefix;
    DBuf<int> first_le;
    long long key_min = 0; int n_keys = 0;
    DBuf<int> macro_guide;             // [S][tpad] (classic macro atom)
    DBuf<int2> macro_next, macro_entry;  // [T], [L] (classic macro atom)
    DBuf<unsigned long long> cnt_rep;  // [BULK_REPS][CNT_COUNT] rare-path counter replicas
    DBuf<double> bulk_rep;          // jump algorithm: [BULK_REPS][2 S] J / nu_bar replicas (zero between launches)
    double grid0 = 0, grid_last = 0, inv_dgrid = 0;
    int bulk_reps_used = 256;
    bool have_macro_guide = false;
    DBuf<unsigned long long> diff;  // jump algorithm: [S][lpad+1][4] fixed-point difference arrays
    DBuf<unsigned long long> xfer;  // jump algorithm: [S-1][lpad+1][4] shell-crossing transfers, folded into diff per call
    double e_typ = 0.0;             // typical packet energy (sets the fixed-point scale)
    double e_typ_group = 0.0;       // > 0: imposed by an engine group for the call in progress (the whole set's e_typ)
    double diff_scale1 = 0.0, diff_scale2 = 0.0;  // scales of what the difference arrays hold (0 = they are empty)
    double finalize_ms = 0.0;
    bool est_unreduced = false;     // a transport filled the estimators since the last engine-group collective
    DBuf<int> line2macro, block_edge, ttype, dest, tline;
    // nonhomologous mode (nonhomologous.cuh): NumbaRadial1DGeometry's v_inner / v_outer / velocity_gradient [S]
    int nonhomologous = 0;
    DBuf<double> v_inner, v_outer, dvdr;
    // continuum (IIP mode)
    int continuum = 0, n_continua = 0, n_phot = 0, phot_pad = 0, n_activation = 0, n_markov = 0;
    long long k_packet_idx = -1;
    DBuf<double> t_e, bf_thr, pi_min, pi_max, x_sect, phot_nus, ff_factor, chi_bf_t, emiss_t, markov_cum;
    DBuf<int> pi_refs, pi_act;
    // continuum macro atom built on the device (markov_build.cuh)
    bool markov_pending = false;    // tb200_set_model got no absorbing_markov_probabilities / transition_probabilities
    DBuf<double> mk_p_t, mk_q, mk_r, mk_c, mk_keep;  // normalised input [S][tpad]; q [S][n]; pivot row / column; kept X
    DBuf<int> mk_type, mk_dest, mk_err;
    int mk_keep_n = 0;              // n of the kept X (0: none)
    bool mk_resident = false;       // mk_p_t holds the normalised table of a tb200_build_opacity since the last tb200_set_model
    // continuum macro atom's rows built on the device (continuum_macro_build.cuh): the row map of tb200_set_atomic_data
    // (table offset + key * S of every row, -1: none; energy), the per-iteration tables and shell arrays, the kept table
    int ct_T = -1;                  // T of the row map (-1: none)
    long long ct_base[tbcm::N_TABLES + 1] = {};  // start of each table in ct_tab, in units of S doubles
    DBuf<long long> ct_off;
    DBuf<double> ct_energy, ct_tab, ct_shell, op_cont_tp_t;
    bool op_cont_valid = false;     // op_cont_tp_t holds the kept normalised table of the last continuum tb200_build_opacity
    // global frequency bins of the bound-free opacity / estimators (continuum_bins.cuh)
    int cont_bins = 0, cb_n_gkeys = 0;
    long long cb_gkey_min = 0;
    DBuf<double> cb_B, cb_mom, cont_lit;
    DBuf<int> cb_guide, cb_nact, cb_pos, cb_act_start, cb_act;
    DBuf<double2> cb_chi_lin;
    size_t off_ffheat = 0, off_cont = 0, off_spec = 0, off_lum = 0;  // packed estimator buffer: ff_heating(S) and 5 x (n_continua * S)
    // packed estimators: [J(S) | nubar(S) | vhist(G) | pad | jblue(S*lpad) | edotlu(S*lpad)]
    DBuf<double> est;
    size_t off_J = 0, off_nubar = 0, off_vhist = 0, off_jblue = 0, off_edotlu = 0, est_count = 0;
    // packets
    int64_t N = 0;
    DBuf<double> in_r, in_nu, in_mu, in_energy, out_nu, out_energy;
    DBuf<long long> seeds64;
    DBuf<double> ps_l_array;                 // device-side packet source: l_array, rejected raw draws, {count, overflow}
    DBuf<unsigned long long> ps_rejected;
    DBuf<unsigned> ps_count;
    DBuf<unsigned long long> ps_minmax;      // weighted source: {min, max} of the Carter-Cashwell nus (as bit patterns)
    DBuf<double> ps_leaf_sums;               // weighted source: the pairwise-sum leaves that start in this engine's range
    DBuf<unsigned> seed32, x397, order_hist;
    DBuf<tb::StartRecord> start_rec;         // by processing slot (tb::StartRecord), written by the ordering pass
    // radiation-field solve (radfield.cuh): resident results + scratch for host-supplied estimators
    DBuf<double> rf_shell;   // [5 S]: t_rad, w, norm, j, nu_bar (the last two only with host-supplied estimators)
    DBuf<double> rf_volume, rf_jblues_t, rf_in_t;  // [S]; [S][lpad] normalised J_blue (shell-major); [S][lpad] uploaded estimator
    DBuf<double> rf_dvdr;                          // [S] the caller's velocity_gradient (nonhomologous mode)
    // opacity build (opacity_build.cuh)
    bool opacity_pending = false;   // tb200_set_model got no tau_sobolev / transition_probabilities: tb200_build_opacity must run first
    bool have_macro = false;        // macro-atom metadata uploaded (line_interaction_type != scatter or continuum)
    bool have_atomic = false, rf_valid = false;
    bool sf_valid = false;          // att_S_ul / Jred_lu / Jblue_lu of tb200_solve_source_function are resident (for this model)
    int keep_opacity_tables = 0;
    // source function (source_function.cuh): CSR lists built by tb200_solve_source_function, per-shell work vectors
    DBuf<int> sf_lvl_ptr, sf_lvl_lines, sf_in_ptr, sf_in_rows, sf_in_src, sf_em_row, sf_upper;
    DBuf<double> sf_wave, sf_norm, sf_e, sf_c0, sf_c1, sf_att_t, sf_jred_t, sf_jblue_t, sf_in_t, sf_in2_t, sf_delta;
    int64_t n_levels = 0;
    // formal integral (formal_integral.cuh): cells of the integrator's shells, per-shell set-up, results
    DBuf<double> fi_cells;           // [S2][L + 2] x 4 doubles
    DBuf<double> fi_shells;          // r_inner, r_outer, kappa of the integrator's shells [3 S2]
    DBuf<double> fi_weights;         // tbfi::ShellWeights [S2] (as raw storage)
    DBuf<double> fi_freq, fi_I, fi_L, fi_att_t, fi_jred_t, fi_jblue_t;
    double fi_cells_ms = 0.0, fi_rays_ms = 0.0;
    tbo::Constants op_const{};
    DBuf<int> at_lower, at_upper;
    DBuf<unsigned char> at_meta, at_nlte;
    DBuf<double> at_g, at_wfl, at_flu, at_ful, at_elo, at_eup, op_lnd, op_beta_t, op_stim_t, op_tp_norm_t;
    DBuf<double> op_dvdr;  // [S] the caller's velocity_gradient of tb200_build_opacity (nonhomologous mode)
    // classic plasma (plasma.cuh): the tables of tb200_set_plasma_data, per-iteration work arrays.  The level populations
    // of tb200_solve_plasma lie in op_lnd, where tb200_build_opacity reads them.
    bool pl_set = false;            // tb200_set_plasma_data has been given (for pl_S shells and pl_n_levels levels)
    bool pl_valid = false;          // op_lnd holds the populations of a tb200_solve_plasma since the last tb200_set_model
    int pl_S = 0, pl_n_ions = 0, pl_n_elements = 0;
    int64_t pl_n_levels = 0;
    double pl_chi_0 = 0.0;
    tbp::Constants pl_const{};
    double pl_c = 0.0;
    std::vector<double> pl_zeta_t;  // zeta temperature grid (the interpolation weights are set up on the host)
    DBuf<double> pl_energy, pl_charge, pl_chi, pl_nd, pl_zeta, pl_z, pl_phi, pl_pop, pl_ne, pl_new, pl_fixed_ne;
    DBuf<int> pl_level_ion, pl_ion_first, pl_element_first, pl_status;
    DBuf<tbp::Shell> pl_shell;
    // control
    DBuf<unsigned> rng_buf;
    DBuf<unsigned long long> ctrl;  // [0] next_packet, [1] vlog_count, [2..] counters
    DBuf<int> error;
    // tracking
    DBuf<long long> last_i;  // 5 * N
    DBuf<double> last_d;     // 7 * N
    DBuf<tb::Event> events;
    DBuf<long long> event_counts;
    int64_t n_tracked = 0, max_events = 0;
    bool track_last = false;
    DBuf<double> vlog_d;  // 4 * cap
    DBuf<long long> vlog_pid;
    int64_t vlog_capacity = 0;
};

extern "C" {

const char *tb200_last_error(void) { return g_last_error.c_str(); }
const char *tb200_version(void) { return "tardis_b200 0.1 (sm_90a)"; }

int tb200_create(int device_id, tb200_engine **engine) {
    if (!engine) return fail(TB200_ERR_INVALID, "engine is NULL");
    *engine = nullptr;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
        return fail(TB200_ERR_CUDA, std::string("no CUDA device: ") + (e != cudaSuccess ? cudaGetErrorString(e) : "count is 0") +
                                        " (tardis_b200 has no CPU path)");
    if (device_id < 0 || device_id >= count) return fail(TB200_ERR_INVALID, "bad device id");
    CK(cudaSetDevice(device_id));
    tb200_engine *en = new tb200_engine();
    en->device = device_id;
    cudaDeviceProp prop;
    cudaError_t ce = cudaGetDeviceProperties(&prop, device_id);
    if (ce == cudaSuccess) ce = cudaStreamCreateWithFlags(&en->stream.h, cudaStreamNonBlocking);
    if (ce == cudaSuccess) ce = cudaStreamCreateWithFlags(&en->h2d_stream.h, cudaStreamNonBlocking);
    if (ce == cudaSuccess) ce = cudaStreamCreateWithFlags(&en->d2h_stream.h, cudaStreamNonBlocking);
    if (ce == cudaSuccess) ce = cudaEventCreate(&en->ev_start.h);
    if (ce == cudaSuccess) ce = cudaEventCreate(&en->ev_stop.h);
    if (ce == cudaSuccess) ce = cudaEventCreate(&en->ev_fin.h);
    if (ce != cudaSuccess) {  // nothing half-built is handed out or left behind
        delete en;
        return fail(TB200_ERR_CUDA, std::string("tb200_create: ") + cudaGetErrorString(ce));
    }
    en->sm_count = prop.multiProcessorCount;
    en->smem_optin = prop.sharedMemPerBlockOptin;
    *engine = en;
    return TB200_OK;
}

void tb200_destroy(tb200_engine *en) {
    if (!en) return;
    cudaSetDevice(en->device);
    cudaStreamSynchronize(en->stream);
    delete en;  // the buffers, then the events and streams (tb200_engine's owners)
}

int tb200_set_option(tb200_engine *en, const char *name, int64_t value) {
    if (!en || !name) return fail(TB200_ERR_INVALID, "bad argument");
    std::string k(name);
    if (k == "ctas_per_sm") { if (value < 0 || value > 16) return fail(TB200_ERR_INVALID, "ctas_per_sm out of range"); en->ctas_per_sm = (int)value; }
    else if (k == "threads_per_cta") { if (value != 128 && value != 256) return fail(TB200_ERR_INVALID, "threads_per_cta must be 128 or 256"); en->threads_per_cta = (int)value; }
    else if (k == "refill_min") { if (value < 0 || value > 32) return fail(TB200_ERR_INVALID, "refill_min must be in [0, 32]"); en->refill_min = (int)value; }
    else if (k == "pipeline_edges") { en->pipeline_edges = value ? 1 : 0; }
    else if (k == "pipeline_chunks") { if (value < 1 || value > 64) return fail(TB200_ERR_INVALID, "pipeline_chunks must be in [1, 64]"); en->pipeline_chunks = (int)value; }
    else if (k == "sort_packets") { en->sort_packets = value ? 1 : 0; }
    else if (k == "sort_bits") { if (value < 0 || value > 16) return fail(TB200_ERR_INVALID, "sort_bits must be in [0, 16]"); en->sort_bits = (int)value; }
    else if (k == "park_min") { if (value < 0 || value > 32) return fail(TB200_ERR_INVALID, "park_min must be in [1, 32]"); en->park_min = (int)value; }
    else if (k == "pooled") { en->pooled = value ? 1 : 0; }
    else if (k == "keep_opacity_tables") { en->keep_opacity_tables = value ? 1 : 0; }
    else if (k == "vol_min") { if (value < 1 || value > 32) return fail(TB200_ERR_INVALID, "vol_min must be in [1, 32]"); en->vol_min = (int)value; }
    else if (k == "algorithm") { if (value < 0 || value > 1) return fail(TB200_ERR_INVALID, "algorithm must be 0 (scan) or 1 (jump)"); en->algorithm = (int)value; }
    else return fail(TB200_ERR_INVALID, "unknown option " + k);
    return TB200_OK;
}

// Slack past the last row of the line-list tables (nu_line, tau, and every table upload_strided_table makes): kept until
// every reader of them is known not to read past shells * pad.
constexpr size_t TABLE_SLACK = 128;

static int upload_strided_table(tb200_engine *en, const double *src, int64_t rows, int64_t shells, int64_t row_stride,
                                int64_t shell_stride, int pad, DBuf<double> &dst) {
    // Stage the host view as it lies in memory: the smallest contiguous span covering it.
    int r;
    if ((r = dst.ensure((size_t)shells * pad + TABLE_SLACK))) return r;
    if (rows == 0 || shells == 0) { CK(cudaMemsetAsync(dst.p, 0, (size_t)shells * pad * sizeof(double), en->stream)); return TB200_OK; }
    if (row_stride < 0 || shell_stride < 0) return fail(TB200_ERR_INVALID, "negative strides are not supported");
    size_t span = (size_t)(rows - 1) * row_stride + (size_t)(shells - 1) * shell_stride + 1;
    if ((r = en->staging.ensure(span))) return r;
    CK(cudaMemcpyAsync(en->staging.p, src, span * sizeof(double), cudaMemcpyHostToDevice, en->stream));
    long long total = (long long)shells * pad;
    tb::transpose_to_shell_major<<<(unsigned)((total + 255) / 256), 256, 0, en->stream>>>(en->staging.p, row_stride, shell_stride,
                                                                                        (int)rows, (int)shells, pad, dst.p);
    en->launches++;
    CK(cudaGetLastError());
    return TB200_OK;
}

// The way back: rows x S of a shell-major [S][pad] table to the host as [rows][S] (line-major), through staging.  Only
// queued on en->stream: the caller synchronises before it reads dst.
static int download_line_major(tb200_engine *en, const double *src_t, int rows, int pad, double *dst) {
    const long long cells = (long long)rows * en->S;
    int r;
    if ((r = en->staging.ensure((size_t)cells))) return r;
    tb::transpose_to_line_major<<<(unsigned)((cells + 255) / 256), 256, 0, en->stream>>>(src_t, rows, en->S, pad, en->staging.p);
    en->launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(dst, en->staging.p, (size_t)cells * sizeof(double), cudaMemcpyDeviceToHost, en->stream));
    return TB200_OK;
}

static int upload_i64_as_i32(tb200_engine *en, const int64_t *src, int64_t n, DBuf<int> &dst) {
    int r;
    if ((r = dst.ensure((size_t)(n > 0 ? n : 1)))) return r;
    std::vector<int> tmp((size_t)(n > 0 ? n : 1), 0);
    for (int64_t i = 0; i < n; i++) {
        int64_t v = src[i];
        if (v > 2147483647LL || v < -2147483648LL) return fail(TB200_ERR_INVALID, "index table value does not fit in 32 bits");
        tmp[(size_t)i] = (int)v;
    }
    CK(cudaMemcpyAsync(dst.p, tmp.data(), tmp.size() * sizeof(int), cudaMemcpyHostToDevice, en->stream));
    CK(cudaStreamSynchronize(en->stream));  // tmp goes out of scope
    return TB200_OK;
}

// What the kernels read besides the opacity tables themselves: running sums + guide table of the macro atom, double-double
// prefix sums of tau.  Runs at the end of tb200_set_model (host tables) or of tb200_build_opacity (device-built tables).
static int finish_opacity_tables(tb200_engine *en) {
    int r;
    const int S = en->S;
    if (en->have_macro) {
        const long long total = (long long)en->n_blocks * S;
        tb::macro_cumsum_kernel<<<(unsigned)((total + 127) / 128), 128, 0, en->stream>>>(en->tp_t.p, en->block_edge.p, en->n_blocks, S, en->tpad);
        en->launches++;
        CK(cudaGetLastError());
        if ((r = en->macro_guide.ensure((size_t)S * en->tpad))) return r;
        tb::macro_guide_kernel<<<(unsigned)((total + 127) / 128), 128, 0, en->stream>>>(en->tp_t.p, en->block_edge.p, en->n_blocks, S, en->tpad, en->macro_guide.p);
        en->launches++;
        CK(cudaGetLastError());
        if ((r = en->macro_next.ensure((size_t)std::max(en->T, 1))) || (r = en->macro_entry.ensure((size_t)en->L))) return r;
        const int n_items = std::max(en->T, en->L);
        tb::macro_next_kernel<<<(unsigned)((n_items + 255) / 256), 256, 0, en->stream>>>(en->block_edge.p, en->ttype.p, en->dest.p, en->tline.p,
            en->line2macro.p, en->n_blocks, en->T, en->L, en->macro_next.p, en->macro_entry.p);
        en->launches++;
        CK(cudaGetLastError());
        en->have_macro_guide = true;
    }
    tb::tau_prefix_kernel<<<S, 32, 0, en->stream>>>(en->tau_t.p, en->L, en->lpad, en->prefix.p);
    en->launches++;
    CK(cudaGetLastError());
    return TB200_OK;
}

int tb200_set_model(tb200_engine *en, const tb200_model *m, const tb200_config *c) {
    if (!en || !m || !c) return fail(TB200_ERR_INVALID, "bad argument");
    CK(cudaSetDevice(en->device));
    if (m->n_shells < 1 || m->n_lines < 1) return fail(TB200_ERR_INVALID, "need at least one shell and one line");
    if (m->n_lines > 2000000000LL || m->n_transitions > 2000000000LL) return fail(TB200_ERR_INVALID, "table too large for 32-bit indices");
    if (c->n_grid < 2 && c->number_of_vpackets > 0) return fail(TB200_ERR_INVALID, "virtual packets need a spectrum grid");
    if (c->line_interaction_type < 0 || c->line_interaction_type > 2) return fail(TB200_ERR_INVALID, "line_interaction_type must be 0, 1 or 2");
    for (int64_t i = 1; i < m->n_lines; i++)
        if (m->line_list_nu[i] > m->line_list_nu[i - 1]) return fail(TB200_ERR_INVALID, "line_list_nu must be sorted in descending order");
    if (c->nonhomologous) {  // modes/nonhomologous: partial relativity and lines + electron scattering only
        if (c->enable_full_relativity) return fail(TB200_ERR_INVALID, "Full relativity not supported for non-homology.");
        if (c->continuum_processes_enabled) return fail(TB200_ERR_INVALID, "continuum processes are not supported in the nonhomologous mode");
        if (!m->v_inner || !m->v_outer) return fail(TB200_ERR_INVALID, "the nonhomologous mode needs the model's v_inner and v_outer");
    }
    en->have_model = false;
    en->sf_valid = false;
    en->pl_valid = false;
    en->diff_scale1 = en->diff_scale2 = 0.0;  // the difference arrays are zeroed below
    en->S = (int)m->n_shells; en->L = (int)m->n_lines; en->lpad = round_up(en->L, 32) + 32;
    en->T = (int)m->n_transitions; en->tpad = round_up(en->T > 0 ? en->T : 1, 32); en->n_blocks = (int)m->n_blocks;
    en->n_grid = (int)c->n_grid;
    en->cfg = *c;
    en->cfg.spectrum_frequency_grid = nullptr;
    en->t_exp = m->time_explosion;
    en->nu_typ = sqrt(fabs(m->line_list_nu[0] * m->line_list_nu[m->n_lines - 1]));
    if (!(en->nu_typ > 0)) en->nu_typ = 1.0;
    int r;
    const int S = en->S, L = en->L;
    if ((r = en->r_inner.ensure(S)) || (r = en->r_outer.ensure(S)) || (r = en->n_e.ensure(S)) || (r = en->nu_line.ensure(en->lpad + TABLE_SLACK))) return r;
    CK(cudaMemcpyAsync(en->r_inner.p, m->r_inner, S * sizeof(double), cudaMemcpyHostToDevice, en->stream));
    CK(cudaMemcpyAsync(en->r_outer.p, m->r_outer, S * sizeof(double), cudaMemcpyHostToDevice, en->stream));
    CK(cudaMemcpyAsync(en->n_e.p, m->electron_density, S * sizeof(double), cudaMemcpyHostToDevice, en->stream));
    en->nonhomologous = c->nonhomologous ? 1 : 0;
    if (en->nonhomologous) {
        // NumbaRadial1DGeometry.__init__ (model/geometry/radial1d.py:342-357): velocity_gradient by the reference's expression
        std::vector<double> g((size_t)S);
        for (int s = 0; s < S; s++) g[s] = nh::velocity_gradient(m->r_inner[s], m->r_outer[s], m->v_inner[s], m->v_outer[s]);
        if ((r = en->v_inner.ensure(S)) || (r = en->v_outer.ensure(S)) || (r = en->dvdr.ensure(S))) return r;
        CK(cudaMemcpyAsync(en->v_inner.p, m->v_inner, S * sizeof(double), cudaMemcpyHostToDevice, en->stream));
        CK(cudaMemcpyAsync(en->v_outer.p, m->v_outer, S * sizeof(double), cudaMemcpyHostToDevice, en->stream));
        CK(cudaMemcpyAsync(en->dvdr.p, g.data(), S * sizeof(double), cudaMemcpyHostToDevice, en->stream));
        CK(cudaStreamSynchronize(en->stream));  // g goes out of scope
    }
    CK(cudaMemsetAsync(en->nu_line.p, 0, (en->lpad + TABLE_SLACK) * sizeof(double), en->stream));
    CK(cudaMemcpyAsync(en->nu_line.p, m->line_list_nu, L * sizeof(double), cudaMemcpyHostToDevice, en->stream));
    en->opacity_pending = false;
    en->markov_pending = false;
    en->mk_keep_n = 0;
    en->mk_resident = false;
    en->op_cont_valid = false;
    en->ct_T = -1;  // the row map holds offsets for this model's S and was checked against its types: give it again
    if (m->tau_sobolev) {
        if ((r = upload_strided_table(en, m->tau_sobolev, L, S, m->tau_line_stride, m->tau_shell_stride, en->lpad, en->tau_t))) return r;
    } else {  // built on the device by tb200_build_opacity
        if ((r = en->tau_t.ensure((size_t)S * en->lpad + TABLE_SLACK))) return r;
        CK(cudaMemsetAsync(en->tau_t.p, 0, ((size_t)S * en->lpad + TABLE_SLACK) * sizeof(double), en->stream));
        en->opacity_pending = true;
    }
    if (c->n_grid > 0) {
        if ((r = en->grid.ensure((size_t)c->n_grid))) return r;
        CK(cudaMemcpyAsync(en->grid.p, c->spectrum_frequency_grid, c->n_grid * sizeof(double), cudaMemcpyHostToDevice, en->stream));
        en->grid0 = c->spectrum_frequency_grid[0]; en->grid_last = c->spectrum_frequency_grid[c->n_grid - 1];
        en->inv_dgrid = c->n_grid > 1 ? 1.0 / (c->spectrum_frequency_grid[1] - c->spectrum_frequency_grid[0]) : 0.0;
    }
    // macro atom tables (only read when line_interaction_type != scatter)
    en->have_macro_guide = false;
    en->have_macro = false;
    if (c->line_interaction_type != 0 || c->continuum_processes_enabled) {
        if (!m->macro_block_edge_index) return fail(TB200_ERR_INVALID, "macro atom tables missing");
        if (m->transition_probabilities) {
            if ((r = upload_strided_table(en, m->transition_probabilities, en->T, S, m->tp_transition_stride, m->tp_shell_stride, en->tpad, en->tp_t))) return r;
        } else {
            if ((r = en->tp_t.ensure((size_t)S * en->tpad))) return r;
            CK(cudaMemsetAsync(en->tp_t.p, 0, (size_t)S * en->tpad * sizeof(double), en->stream));
            // continuum mode: tb200_build_absorbing_markov writes the deactivation table; otherwise tb200_build_opacity
            if (c->continuum_processes_enabled) en->markov_pending = true;
            else en->opacity_pending = true;
        }
        en->have_macro = true;
        if ((r = upload_i64_as_i32(en, m->line2macro_level_upper, L, en->line2macro))) return r;
        if ((r = upload_i64_as_i32(en, m->macro_block_edge_index, m->n_blocks + 1, en->block_edge))) return r;
        if ((r = upload_i64_as_i32(en, m->transition_type, en->T, en->ttype))) return r;
        if ((r = upload_i64_as_i32(en, m->destination_level_id, en->T, en->dest))) return r;
        if ((r = upload_i64_as_i32(en, m->transition_line_id, en->T, en->tline))) return r;
        for (int64_t b = 0; b < m->n_blocks; b++)
            if (m->macro_block_edge_index[b] > m->macro_block_edge_index[b + 1] || m->macro_block_edge_index[b] < 0 ||
                m->macro_block_edge_index[b + 1] > m->n_transitions)
                return fail(TB200_ERR_INVALID, "macro_block_edge_index must be non-decreasing and within [0, n_transitions]");
    }
    // continuum (IIP mode) tables
    en->continuum = c->continuum_processes_enabled ? 1 : 0;
    if (en->continuum) {
        if (!m->t_electrons || !m->phot_nus || !m->chi_bf || !m->x_sect || !m->emissivities || !m->photo_ion_block_references ||
            !m->photo_ion_nu_threshold_mins || !m->photo_ion_nu_threshold_maxs || !m->bf_threshold_list_nu || !m->ff_opacity_factor ||
            !m->photo_ion_activation_idx)
            return fail(TB200_ERR_INVALID, "continuum tables missing");
        if (m->n_continua < 0 || m->n_phot < 2 || (m->absorbing_markov_probabilities && m->n_markov < 1))
            return fail(TB200_ERR_INVALID, "bad continuum sizes");
        en->n_continua = (int)m->n_continua; en->n_phot = (int)m->n_phot; en->phot_pad = round_up(en->n_phot, 32);
        en->n_activation = (int)m->n_activation; en->n_markov = (int)m->n_markov; en->k_packet_idx = m->k_packet_idx;
        for (int64_t k = 0; k < m->n_continua; k++)
            if (m->photo_ion_block_references[k + 1] - m->photo_ion_block_references[k] < 2 || m->photo_ion_block_references[k] < 0 ||
                m->photo_ion_block_references[k + 1] > m->n_phot)
                return fail(TB200_ERR_INVALID, "photo_ion_block_references: every continuum needs >= 2 cross-section points inside [0, n_phot]");
        const int nc = en->n_continua > 0 ? en->n_continua : 1;
        if ((r = en->t_e.ensure(S)) || (r = en->ff_factor.ensure(S)) || (r = en->bf_thr.ensure(nc)) || (r = en->pi_min.ensure(nc)) ||
            (r = en->pi_max.ensure(nc)) || (r = en->x_sect.ensure(en->n_phot)) || (r = en->phot_nus.ensure(en->n_phot)))
            return r;
        CK(cudaMemcpyAsync(en->t_e.p, m->t_electrons, S * sizeof(double), cudaMemcpyHostToDevice, en->stream));
        CK(cudaMemcpyAsync(en->ff_factor.p, m->ff_opacity_factor, S * sizeof(double), cudaMemcpyHostToDevice, en->stream));
        if (en->n_continua > 0) {
            CK(cudaMemcpyAsync(en->bf_thr.p, m->bf_threshold_list_nu, en->n_continua * sizeof(double), cudaMemcpyHostToDevice, en->stream));
            CK(cudaMemcpyAsync(en->pi_min.p, m->photo_ion_nu_threshold_mins, en->n_continua * sizeof(double), cudaMemcpyHostToDevice, en->stream));
            CK(cudaMemcpyAsync(en->pi_max.p, m->photo_ion_nu_threshold_maxs, en->n_continua * sizeof(double), cudaMemcpyHostToDevice, en->stream));
        }
        CK(cudaMemcpyAsync(en->x_sect.p, m->x_sect, en->n_phot * sizeof(double), cudaMemcpyHostToDevice, en->stream));
        CK(cudaMemcpyAsync(en->phot_nus.p, m->phot_nus, en->n_phot * sizeof(double), cudaMemcpyHostToDevice, en->stream));
        if ((r = upload_strided_table(en, m->chi_bf, en->n_phot, S, S, 1, en->phot_pad, en->chi_bf_t))) return r;
        if ((r = upload_strided_table(en, m->emissivities, en->n_phot, S, S, 1, en->phot_pad, en->emiss_t))) return r;
        if ((r = upload_i64_as_i32(en, m->photo_ion_block_references, m->n_continua + 1, en->pi_refs))) return r;
        if ((r = upload_i64_as_i32(en, m->photo_ion_activation_idx, m->n_activation, en->pi_act))) return r;
        if (m->absorbing_markov_probabilities) {
            const size_t nm = (size_t)S * en->n_markov * en->n_markov;
            if ((r = en->markov_cum.ensure(nm))) return r;
            CK(cudaMemcpyAsync(en->markov_cum.p, m->absorbing_markov_probabilities, nm * sizeof(double), cudaMemcpyHostToDevice, en->stream));
            const long long rows = (long long)S * en->n_markov;
            tb::markov_cumsum_kernel<<<(unsigned)((rows + 127) / 128), 128, 0, en->stream>>>(en->markov_cum.p, rows, en->n_markov);
            en->launches++;
            CK(cudaGetLastError());
        } else {  // built on the device by tb200_build_absorbing_markov
            en->n_markov = 0;
            en->markov_pending = true;
        }
        // global frequency bins (continuum_bins.cuh): sorted union of the blocks, guide table, per-(shell, bin) linear chi_bf_tot
        {
            const tbc::HostBins hb = tbc::build_bins(m->phot_nus, en->n_phot, (const long long *)m->photo_ion_block_references, en->n_continua,
                                                     m->photo_ion_nu_threshold_mins, m->photo_ion_nu_threshold_maxs);
            en->cont_bins = hb.usable ? 1 : 0;
            const size_t nb = (size_t)en->n_phot + 1, ncs = (size_t)(en->n_continua > 0 ? en->n_continua : 1) * S;
            if ((r = en->cb_mom.ensure((size_t)S * nb * tbc::N_MOMENTS)) || (r = en->cont_lit.ensure(5 * ncs))) return r;
            CK(cudaMemsetAsync(en->cb_mom.p, 0, (size_t)S * nb * tbc::N_MOMENTS * sizeof(double), en->stream));
            CK(cudaMemsetAsync(en->cont_lit.p, 0, 5 * ncs * sizeof(double), en->stream));
            if ((r = en->cb_pos.ensure(nb))) return r;  // (also read, unused, by the finalize kernel when the bins are off)
            if (hb.usable) {
                en->cb_gkey_min = hb.gkey_min; en->cb_n_gkeys = hb.n_gkeys;
                if ((r = en->cb_B.ensure(nb)) || (r = en->cb_guide.ensure(hb.guide.size())) || (r = en->cb_nact.ensure(nb)) ||
                    (r = en->cb_chi_lin.ensure((size_t)S * nb)) || (r = en->cb_act_start.ensure(hb.act_start.size())) ||
                    (r = en->cb_act.ensure(hb.act.size())))
                    return r;
                CK(cudaMemcpyAsync(en->cb_B.p, hb.B.data(), hb.B.size() * sizeof(double), cudaMemcpyHostToDevice, en->stream));
                CK(cudaMemcpyAsync(en->cb_pos.p, hb.pos.data(), hb.pos.size() * sizeof(int), cudaMemcpyHostToDevice, en->stream));
                CK(cudaMemcpyAsync(en->cb_guide.p, hb.guide.data(), hb.guide.size() * sizeof(int), cudaMemcpyHostToDevice, en->stream));
                CK(cudaMemcpyAsync(en->cb_act_start.p, hb.act_start.data(), hb.act_start.size() * sizeof(int), cudaMemcpyHostToDevice, en->stream));
                if (!hb.act.empty()) CK(cudaMemcpyAsync(en->cb_act.p, hb.act.data(), hb.act.size() * sizeof(int), cudaMemcpyHostToDevice, en->stream));
                const long long total = (long long)S * nb;
                tb::continuum_lin_kernel<<<(unsigned)((total + 127) / 128), 128, 0, en->stream>>>(en->cb_B.p, en->n_phot, en->phot_nus.p, en->cb_pos.p,
                    en->pi_refs.p, en->n_continua, en->chi_bf_t.p, en->phot_pad, S, en->cb_chi_lin.p, en->cb_nact.p);
                en->launches++;
                CK(cudaGetLastError());
                CK(cudaStreamSynchronize(en->stream));  // hb goes out of scope
            }
        }
        if (c->line_interaction_type == 0) {
            // `scatter` lines with continuum: the macro atom is still needed for continuum events
            if (!m->macro_block_edge_index) return fail(TB200_ERR_INVALID, "macro atom tables missing");
        }
    }
    // double-double prefix sums of tau along the line list, per shell (jump traces and virtual packets)
    {
        size_t cnt = (size_t)S * (en->lpad + 1);
        if ((r = en->prefix.ensure(cnt))) return r;
        if (!en->opacity_pending && en->have_macro && en->keep_opacity_tables) {  // the normalised rows themselves (tp_t becomes running sums)
            if ((r = en->op_tp_norm_t.ensure((size_t)S * en->tpad))) return r;
            CK(cudaMemcpyAsync(en->op_tp_norm_t.p, en->tp_t.p, (size_t)S * en->tpad * sizeof(double), cudaMemcpyDeviceToDevice, en->stream));
        }
        if (!en->opacity_pending && (r = finish_opacity_tables(en))) return r;
        if ((r = en->diff.ensure(cnt * 4))) return r;
        CK(cudaMemsetAsync(en->diff.p, 0, cnt * 4 * sizeof(unsigned long long), en->stream));
        // frequency-bucket table (guess of the boundary-crossing line)
        long long kmax, kmin;
        {
            double a = m->line_list_nu[0], b = m->line_list_nu[L - 1];
            if (!(b > 0.0)) return fail(TB200_ERR_INVALID, "line frequencies must be positive");
            memcpy(&kmax, &a, 8); memcpy(&kmin, &b, 8);
            kmax >>= tb::NU_KEY_SHIFT; kmin >>= tb::NU_KEY_SHIFT;
        }
        if (kmax - kmin + 1 > 64LL * 1024 * 1024) return fail(TB200_ERR_INVALID, "line list spans too many octaves for the bucket table");
        en->key_min = kmin; en->n_keys = (int)(kmax - kmin + 1);
        if ((r = en->first_le.ensure((size_t)en->n_keys))) return r;
        {
            std::vector<int> init((size_t)en->n_keys, L);
            CK(cudaMemcpyAsync(en->first_le.p, init.data(), init.size() * sizeof(int), cudaMemcpyHostToDevice, en->stream));
            CK(cudaStreamSynchronize(en->stream));
        }
        tb::nu_bucket_kernel<<<(L + 255) / 256, 256, 0, en->stream>>>(en->nu_line.p, L, en->key_min, en->n_keys, en->first_le.p);
        en->launches++;
        CK(cudaGetLastError());
    }
    // packed estimator buffer
    size_t off = 0;
    en->off_J = off; off += S;
    en->off_nubar = off; off += S;
    en->off_vhist = off; off += (size_t)(en->n_grid > 0 ? en->n_grid : 1);
    en->off_spec = off; off += (size_t)2 * (en->n_grid > 1 ? en->n_grid - 1 : 0);
    en->off_lum = off; off += 4;
    en->off_ffheat = off; if (en->continuum) off += S;
    en->off_cont = off; if (en->continuum) off += (size_t)5 * en->n_continua * S;
    off = (off + 31) / 32 * 32;  // 256-byte alignment of the line tables
    en->off_jblue = off; off += (size_t)S * en->lpad;
    en->off_edotlu = off; off += (size_t)S * en->lpad;
    en->est_count = off;
    if ((r = en->est.ensure(off))) return r;
    CK(cudaMemsetAsync(en->est.p, 0, off * sizeof(double), en->stream));
    // control words
    if ((r = en->ctrl.ensure(2 + tb::CNT_COUNT)) || (r = en->error.ensure(1))) return r;
    CK(cudaMemsetAsync(en->ctrl.p, 0, (2 + tb::CNT_COUNT) * sizeof(unsigned long long), en->stream));
    CK(cudaMemsetAsync(en->error.p, 0, sizeof(int), en->stream));
    CK(cudaStreamSynchronize(en->stream));
    en->have_model = true;
    return TB200_OK;
}

static int prepare_tracking(tb200_engine *en, const tb200_outputs *o) {
    int r;
    en->track_last = o && o->last_interaction_type != nullptr;
    if (en->track_last) {
        if ((r = en->last_i.ensure((size_t)5 * en->N)) || (r = en->last_d.ensure((size_t)7 * en->N))) return r;
    }
    en->n_tracked = 0; en->max_events = 0;
    if (o && o->events && o->n_tracked_packets > 0 && o->max_events_per_packet > 0) {
        en->n_tracked = o->n_tracked_packets < en->N ? o->n_tracked_packets : en->N;
        en->max_events = o->max_events_per_packet;
        if ((r = en->events.ensure((size_t)en->n_tracked * en->max_events)) || (r = en->event_counts.ensure((size_t)en->n_tracked))) return r;
        CK(cudaMemsetAsync(en->event_counts.p, 0, en->n_tracked * sizeof(long long), en->stream));
    }
    en->vlog_capacity = 0;
    if (o && o->vlog_nus && o->vlog_capacity > 0) {
        en->vlog_capacity = o->vlog_capacity;
        if ((r = en->vlog_d.ensure((size_t)4 * en->vlog_capacity)) || (r = en->vlog_pid.ensure((size_t)en->vlog_capacity))) return r;
    }
    return TB200_OK;
}

// Typical packet energy: mean |energy| over a strided sample of at most 65536 packets.
static double typical_energy(const double *energies, int64_t n) {
    const int64_t m = n < 65536 ? n : 65536;
    double acc = 0.0;
    for (int64_t i = 0; i < m; i++) acc += fabs(energies[i * (n / m)]);
    return acc / (double)m;
}

static void set_typical_energy(tb200_engine *en, const tb200_packets *pk) {
    if (en->e_typ_group > 0) en->e_typ = en->e_typ_group;
    else if (pk->n_packets > 0) en->e_typ = typical_energy(pk->initial_energies, pk->n_packets);
}

// The per-packet arrays of the transport, for n packets.
static int ensure_packet_arrays(tb200_engine *en, int64_t n) {
    int r;
    if ((r = en->in_r.ensure(n)) || (r = en->in_nu.ensure(n)) || (r = en->in_mu.ensure(n)) || (r = en->in_energy.ensure(n)) ||
        (r = en->out_nu.ensure(n)) || (r = en->out_energy.ensure(n)) || (r = en->seeds64.ensure(n)) || (r = en->seed32.ensure(n)) ||
        (r = en->x397.ensure(n)))
        return r;
    return TB200_OK;
}

int tb200_upload_packets(tb200_engine *en, const tb200_packets *pk) {
    if (!en || !pk) return fail(TB200_ERR_INVALID, "bad argument");
    if (pk->n_packets < 0 || pk->n_packets > 2000000000LL) return fail(TB200_ERR_INVALID, "n_packets out of range");
    CK(cudaSetDevice(en->device));
    const int64_t n = pk->n_packets;
    en->N = n;
    int r;
    if ((r = ensure_packet_arrays(en, n))) return r;
    set_typical_energy(en, pk);
    if (n == 0) return TB200_OK;
    CK(cudaMemcpyAsync(en->in_r.p, pk->initial_radii, n * sizeof(double), cudaMemcpyHostToDevice, en->stream));
    CK(cudaMemcpyAsync(en->in_nu.p, pk->initial_nus, n * sizeof(double), cudaMemcpyHostToDevice, en->stream));
    CK(cudaMemcpyAsync(en->in_mu.p, pk->initial_mus, n * sizeof(double), cudaMemcpyHostToDevice, en->stream));
    CK(cudaMemcpyAsync(en->in_energy.p, pk->initial_energies, n * sizeof(double), cudaMemcpyHostToDevice, en->stream));
    CK(cudaMemcpyAsync(en->seeds64.p, pk->packet_seeds, n * sizeof(long long), cudaMemcpyHostToDevice, en->stream));
    // (the processing order, with each packet's start record and RNG seed expansion, is part of every tb200_transport: an
    //  MC iteration has new packets every time, so a timed step pays for it)
    return TB200_OK;
}

// ---- device-side packet source (packet_source.cuh) -----------------------------------------------------------------
namespace {
constexpr int PS_CHUNK = 256;        // packets (or raw draws) per thread: amortises the seven O(log k) jump-aheads
constexpr int PS_MAX_REJECTED = 4096;

__global__ void packet_source_scan_kernel(tbps::Pcg64 origin, unsigned long long n_raw, unsigned rng_excl, unsigned threshold,
                                          unsigned long long *rejected, unsigned *count) {
    const unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long k0 = t * PS_CHUNK;
    if (k0 >= n_raw) return;
    const unsigned long long k1 = (k0 + PS_CHUNK < n_raw) ? k0 + PS_CHUNK : n_raw;
    uint64_t found[8];
    const int c = tbps::scan_chunk(origin, k0, k1, rng_excl, threshold, found, 8);
    if (c > 0) {
        const unsigned base = atomicAdd(count, (unsigned)c);
        for (int j = 0; j < c && j < 8; j++) if (base + j < (unsigned)PS_MAX_REJECTED) rejected[base + j] = found[j];
        if (c > 8) atomicAdd(count + 1, 1u);  // more rejections in one chunk than this path lists
    }
}

// Packets [lo, hi) of the P.n the source creates; the arrays hold that range only (element i - lo is packet i).
__global__ void packet_source_fill_kernel(tbps::SourceParams P, unsigned long long lo, unsigned long long hi, double *r, double *nu,
                                          double *mu, double *e, long long *seeds) {
    const unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long i0 = lo + t * PS_CHUNK;
    if (i0 >= hi) return;
    const unsigned long long i1 = (i0 + PS_CHUNK < hi) ? i0 + PS_CHUNK : hi;
    tbps::fill_chunk(P, i0, i1, r, nu, mu, e, seeds, lo);
}

// Weighted source, pass 1: min and max of the Carter-Cashwell nus of packets [lo, hi).  nu > 0, so the order of the
// bit patterns is the order of the values and the reduction is exact in any order.
__global__ void packet_source_minmax_kernel(tbps::SourceParams P, unsigned long long lo, unsigned long long hi, unsigned long long *mm) {
    const unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long i0 = lo + t * PS_CHUNK;
    double mn = __longlong_as_double(0x7FF0000000000000LL), mx = 0.0;
    if (i0 < hi) tbps::blackbody_nu_minmax(P, i0, (i0 + PS_CHUNK < hi) ? i0 + PS_CHUNK : hi, mn, mx);
    for (int o = 16; o > 0; o >>= 1) {
        mn = fmin(mn, __shfl_xor_sync(0xFFFFFFFFu, mn, o));
        mx = fmax(mx, __shfl_xor_sync(0xFFFFFFFFu, mx, o));
    }
    if ((threadIdx.x & 31) == 0 && mx > 0.0) {
        atomicMin(mm, (unsigned long long)__double_as_longlong(mn));
        atomicMax(mm + 1, (unsigned long long)__double_as_longlong(mx));
    }
}

// Weighted source, pass 2: thread t takes the pairwise-sum leaves that start in [lo + t PS_CHUNK, ...) (thread 0 also the
// leaf holding packet lo), stores its packets with I(nu) as their energy and each leaf's sum at its slot.
__global__ void packet_source_weighted_fill_kernel(tbps::SourceParams P, tbps::WeightedParams W, unsigned long long lo, unsigned long long hi,
                                                   double *r, double *nu, double *mu, double *e, long long *seeds, double *slots) {
    const unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long a = lo + t * PS_CHUNK;
    if (a >= hi) return;
    const unsigned long long b = (a + PS_CHUNK < hi) ? a + PS_CHUNK : hi;
    tbps::weighted_fill_leaves(P, W, a, b, lo, hi, r, nu, mu, e, seeds, slots, tbps::pw_slot(lo));
}

// Weighted source, pass 3: energy = I / sum, a division as numpy's `intensity / intensity.sum()`.
__global__ void packet_source_normalize_kernel(double *e, long long n, double sum) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += stride) e[k] = e[k] / sum;
}
}  // namespace

// Everything create_packets_range needs before its kernels: argument checks, the engine's arrays, the rejected draws of
// the seed segment and the generator parameters.  *ready = false: nothing to generate (no packets, or none in [lo, hi)).
static int packet_source_setup(tb200_engine *en, const tb200_packet_source *src, int64_t lo, int64_t hi, tbps::SourceParams &P, bool *ready) {
    *ready = false;
    if (!en || !src) return fail(TB200_ERR_INVALID, "bad argument");
    if (src->n_packets < 0 || src->n_packets > 2000000000LL) return fail(TB200_ERR_INVALID, "n_packets out of range");
    if (!src->l_array || src->n_l < 1 || src->n_l > (1 << 24)) return fail(TB200_ERR_INVALID, "l_array missing");
    if (!(src->temperature > 0) || !(src->radius > 0)) return fail(TB200_ERR_INVALID, "temperature and radius must be positive");
    if (src->weighted && src->relativistic) return fail(TB200_ERR_INVALID, "the weighted source has no relativistic variant");
    if (src->weighted && src->n_packets == 0)
        return fail(TB200_ERR_INVALID, "the weighted source needs at least one packet (the min / max of zero frequencies is undefined)");
    CK(cudaSetDevice(en->device));
    const int64_t n = src->n_packets, count = hi - lo;
    en->N = count;
    int r;
    if ((r = ensure_packet_arrays(en, count)) || (r = en->ps_l_array.ensure((size_t)src->n_l)) || (r = en->ps_rejected.ensure(PS_MAX_REJECTED)) ||
        (r = en->ps_count.ensure(2)))
        return r;
    if (n == 0) return TB200_OK;
    en->e_typ = 1.0 / (double)n;
    CK(cudaMemcpyAsync(en->ps_l_array.p, src->l_array, (size_t)src->n_l * sizeof(double), cudaMemcpyHostToDevice, en->stream));

    P.origin = tbps::pcg64_from_seed(src->seed);
    P.n = (uint64_t)n;
    const uint32_t pop = src->max_seed_val ? src->max_seed_val : 0xFFFFFFFFu;  // rng.choice(pop, N): integers in [0, pop)
    if (pop < 2u) return fail(TB200_ERR_INVALID, "max_seed_val must be at least 2");
    const uint32_t rng = pop - 1u;  // numpy: rng = high - 1 - low
    P.rng_excl = rng + 1u; P.threshold = tbps::lemire_threshold(rng);
    // rejected raw draws of the seed segment: fixed point of "rejections among the first n + R raw draws" (R is 0 for
    // the reference's population 2**32 - 1 unless a raw draw is exactly 0: probability 2^-32 per packet)
    std::vector<unsigned long long> rejected;
    for (int it = 0;; it++) {
        if (it == 16) return fail(TB200_ERR_INVALID, "packet source: rejection count did not settle");
        const unsigned long long n_raw = (unsigned long long)n + rejected.size();
        CK(cudaMemsetAsync(en->ps_count.p, 0, 2 * sizeof(unsigned), en->stream));
        const unsigned long long threads = (n_raw + PS_CHUNK - 1) / PS_CHUNK;
        packet_source_scan_kernel<<<(unsigned)((threads + 127) / 128), 128, 0, en->stream>>>(P.origin, n_raw, P.rng_excl, P.threshold,
                                                                                             en->ps_rejected.p, en->ps_count.p);
        en->launches++;
        CK(cudaGetLastError());
        unsigned h[2] = {0, 0};
        CK(cudaMemcpyAsync(h, en->ps_count.p, sizeof(h), cudaMemcpyDeviceToHost, en->stream));
        CK(cudaStreamSynchronize(en->stream));
        if (h[1] != 0 || h[0] > (unsigned)PS_MAX_REJECTED)
            return fail(TB200_ERR_INVALID, "packet source: this population size rejects too many draws for the device path");
        const bool settled = (h[0] == rejected.size());
        rejected.resize(h[0]);
        if (h[0]) CK(cudaMemcpy(rejected.data(), en->ps_rejected.p, h[0] * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
        if (settled) break;
    }
    std::sort(rejected.begin(), rejected.end());
    if (!rejected.empty()) CK(cudaMemcpyAsync(en->ps_rejected.p, rejected.data(), rejected.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice, en->stream));
    P.rejected = reinterpret_cast<const uint64_t *>(en->ps_rejected.p); P.n_rej = (int)rejected.size();
    P.dbl_start = ((uint64_t)n + rejected.size() + 1) / 2;
    P.l_array = en->ps_l_array.p; P.n_l = (int)src->n_l;
    P.l_coef = pow(M_PI, 4.0) / 90.0;  // np.pi**4 / 90.0: CPython's float ** is libm pow() too
    P.k_b_t = tb::K_BOLTZMANN * src->temperature; P.h_planck = tb::H_PLANCK;
    P.radius = src->radius; P.energy = 1.0 / (double)n;
    P.relativistic = src->relativistic ? 1 : 0; P.beta = src->beta;
    if (P.relativistic) {  // create_packet_energies, black_body_relativistic.py:160-177: energies * static_inner_boundary2cmf_factor / gamma
        if (!(src->beta >= 0.0 && src->beta < 1.0)) return fail(TB200_ERR_INVALID, "beta must be in [0, 1)");
        const double gamma = 1.0 / sqrt(1 - src->beta * src->beta);
        const double factor = (2 * src->beta + 1) / (1 - src->beta * src->beta);
        P.energy = 1.0 / (double)n * factor / gamma;
    }
    en->e_typ = P.energy;
    *ready = count > 0;
    return TB200_OK;
}

// Packets [lo, hi) of the source's n_packets become the engine's resident packets 0 .. hi - lo - 1, bit for bit what
// the whole set holds there (an engine group generates each member's range in place).  Not the weighted source, whose
// energies need sums over the whole set: create_weighted_packets.
static int create_packets_range(tb200_engine *en, const tb200_packet_source *src, int64_t lo, int64_t hi) {
    tbps::SourceParams P;
    bool ready;
    const int r = packet_source_setup(en, src, lo, hi, P, &ready);
    if (r || !ready) return r;
    const unsigned long long threads = ((unsigned long long)(hi - lo) + PS_CHUNK - 1) / PS_CHUNK;
    packet_source_fill_kernel<<<(unsigned)((threads + 127) / 128), 128, 0, en->stream>>>(P, (unsigned long long)lo, (unsigned long long)hi,
                                                                                         en->in_r.p, en->in_nu.p, en->in_mu.p, en->in_energy.p,
                                                                                         en->seeds64.p);
    en->launches++;
    CK(cudaGetLastError());
    return TB200_OK;
}

// The weighted source on members m[0 .. G) holding packets [b[i], b[i + 1]) (one engine: G = 1).  each(f) runs f(i) for
// every member and returns the first error.  Three passes, with the host between them:
//   1. every member: min / max of the Carter-Cashwell nus of its range; the host takes the min / max over members;
//   2. every member: its packets with I(nu) as energy, and the sums of the pairwise-sum leaves that START in its range (a
//      leaf that runs past the range's end is generated to its end, its packets there not stored); the host combines
//      all leaf sums along numpy's tree, so the sum does not depend on the number of members;
//   3. every member: energy = I / sum.
// Every member's e_typ is the whole set's mean energy, 1 / N.
extern "C++" {  // a template, inside the C-ABI block
template <class Each>
static int create_weighted_packets(const tb200_packet_source *src, tb200_engine *const *m, const int64_t *b, int G, Each each) {
    std::vector<tbps::SourceParams> P((size_t)G);
    std::vector<char> ready((size_t)G, 0);
    std::vector<double> mn((size_t)G, 0.0), mx((size_t)G, 0.0);
    int r = each([&](int i) -> int {
        tb200_engine *en = m[i];
        bool rd;
        int rr = packet_source_setup(en, src, b[i], b[i + 1], P[(size_t)i], &rd);
        if (rr || !rd) return rr;
        ready[(size_t)i] = 1;
        en->e_typ = 1.0 / (double)src->n_packets;
        if ((rr = en->ps_minmax.ensure(2))) return rr;
        const unsigned long long init[2] = {~0ull, 0ull}, count = (unsigned long long)(b[i + 1] - b[i]);
        unsigned long long h[2];
        CK(cudaMemcpyAsync(en->ps_minmax.p, init, sizeof(init), cudaMemcpyHostToDevice, en->stream));
        const unsigned long long threads = (count + PS_CHUNK - 1) / PS_CHUNK;
        packet_source_minmax_kernel<<<(unsigned)((threads + 127) / 128), 128, 0, en->stream>>>(P[(size_t)i], (unsigned long long)b[i],
                                                                                               (unsigned long long)b[i + 1], en->ps_minmax.p);
        en->launches++;
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(h, en->ps_minmax.p, sizeof(h), cudaMemcpyDeviceToHost, en->stream));
        CK(cudaStreamSynchronize(en->stream));
        memcpy(&mn[(size_t)i], &h[0], sizeof(double));
        memcpy(&mx[(size_t)i], &h[1], sizeof(double));
        return TB200_OK;
    });
    if (r) return r;
    tbps::WeightedParams W;
    bool first = true;
    double lo_nu = 0.0, hi_nu = 0.0;
    for (int i = 0; i < G; i++) {
        if (!ready[(size_t)i]) continue;
        lo_nu = first || mn[(size_t)i] < lo_nu ? mn[(size_t)i] : lo_nu;
        hi_nu = first || mx[(size_t)i] > hi_nu ? mx[(size_t)i] : hi_nu;
        first = false;
    }
    W.nu_lo = lo_nu;
    W.nu_range = hi_nu - lo_nu;
    if (!std::isfinite(W.nu_range)) return fail(TB200_ERR_INVALID, "weighted source: the frequency range is not finite");
    W.h_planck = tb::H_PLANCK;
    W.beta_rad = 1 / (tb::K_BOLTZMANN * src->temperature);  // util/base.py:297-298
    W.coefficient = 2 * tb::H_PLANCK / (tb::C_LIGHT * tb::C_LIGHT);

    std::vector<std::vector<double>> slots((size_t)G);
    r = each([&](int i) -> int {
        if (!ready[(size_t)i]) return TB200_OK;
        tb200_engine *en = m[i];
        const uint64_t lo = (uint64_t)b[i], hi = (uint64_t)b[i + 1];
        const size_t n_slots = (size_t)(tbps::pw_slot(hi) - tbps::pw_slot(lo) + 1);
        int rr;
        if ((rr = en->ps_leaf_sums.ensure(n_slots))) return rr;
        const unsigned long long threads = (hi - lo + PS_CHUNK - 1) / PS_CHUNK;
        packet_source_weighted_fill_kernel<<<(unsigned)((threads + 127) / 128), 128, 0, en->stream>>>(
            P[(size_t)i], W, lo, hi, en->in_r.p, en->in_nu.p, en->in_mu.p, en->in_energy.p, en->seeds64.p, en->ps_leaf_sums.p);
        en->launches++;
        CK(cudaGetLastError());
        slots[(size_t)i].resize(n_slots);
        CK(cudaMemcpyAsync(slots[(size_t)i].data(), en->ps_leaf_sums.p, n_slots * sizeof(double), cudaMemcpyDeviceToHost, en->stream));
        CK(cudaStreamSynchronize(en->stream));
        return TB200_OK;
    });
    if (r) return r;
    // leaves are visited in ascending order of their start, so the member holding each one is found by walking forward
    int owner = 0;
    const double sum = tbps::pw_combine(0, (uint64_t)src->n_packets, [&](uint64_t s) {
        while ((int64_t)s >= b[owner + 1]) owner++;
        return slots[(size_t)owner][tbps::pw_slot(s) - tbps::pw_slot((uint64_t)b[owner])];
    });
    return each([&](int i) -> int {
        if (!ready[(size_t)i]) return TB200_OK;
        tb200_engine *en = m[i];
        const long long count = b[i + 1] - b[i];
        const long long blocks = std::min<long long>((count + 255) / 256, 4096);
        packet_source_normalize_kernel<<<(unsigned)blocks, 256, 0, en->stream>>>(en->in_energy.p, count, sum);
        en->launches++;
        CK(cudaGetLastError());
        return tb200_sync(en);
    });
}
}  // extern "C++"

int tb200_create_packets(tb200_engine *en, const tb200_packet_source *src) {
    if (src && src->weighted) {
        if (!en) return fail(TB200_ERR_INVALID, "bad argument");
        const int64_t b[2] = {0, src->n_packets};
        return create_weighted_packets(src, &en, b, 1, [](auto f) { return f(0); });
    }
    return create_packets_range(en, src, 0, src ? src->n_packets : 0);
}

int tb200_download_packets(tb200_engine *en, double *radii, double *nus, double *mus, double *energies, int64_t *seeds) {
    if (!en) return fail(TB200_ERR_INVALID, "bad argument");
    CK(cudaSetDevice(en->device));
    const size_t n = (size_t)en->N;
    if (n == 0) return TB200_OK;
    if (radii) CK(cudaMemcpyAsync(radii, en->in_r.p, n * sizeof(double), cudaMemcpyDeviceToHost, en->stream));
    if (nus) CK(cudaMemcpyAsync(nus, en->in_nu.p, n * sizeof(double), cudaMemcpyDeviceToHost, en->stream));
    if (mus) CK(cudaMemcpyAsync(mus, en->in_mu.p, n * sizeof(double), cudaMemcpyDeviceToHost, en->stream));
    if (energies) CK(cudaMemcpyAsync(energies, en->in_energy.p, n * sizeof(double), cudaMemcpyDeviceToHost, en->stream));
    if (seeds) CK(cudaMemcpyAsync(seeds, en->seeds64.p, n * sizeof(long long), cudaMemcpyDeviceToHost, en->stream));
    CK(cudaStreamSynchronize(en->stream));
    return TB200_OK;
}

// Launch the transport kernel over packets [off, off + n) of the device-resident arrays.
//   first: zero the work counters / error word (and the estimators when zero_estimators)
//   last : run the jump epilogue (difference arrays -> J_blue / Edotlu)
static int launch_range(tb200_engine *en, int64_t off, int64_t n, bool first, bool last, int zero_estimators, cudaEvent_t ev_a, cudaEvent_t ev_b) {
    if (!en->have_model) return fail(TB200_ERR_NO_MODEL, "tb200_set_model has not been called");
    if (en->opacity_pending) return fail(TB200_ERR_NO_MODEL, "the opacity tables are pending: tb200_set_model got no tau_sobolev, call tb200_build_opacity");
    if (en->markov_pending)
        return fail(TB200_ERR_NO_MODEL, "the continuum macro atom is pending: tb200_set_model got no absorbing_markov_probabilities / "
                                        "transition_probabilities, call tb200_build_absorbing_markov");
    CK(cudaSetDevice(en->device));
    const int S = en->S;
    const size_t row_words = (size_t)(en->lpad + 1) * 4;  // one shell's row of the difference arrays
    // the nonhomologous kernel accumulates J_blue / Edotlu straight into the estimator buffer, as the scan kernel does:
    // none of the jump algorithm's difference arrays, fixed-point scales or finalisation
    const bool jump = en->algorithm == 1 && !en->nonhomologous;
    if (first) {
        if (jump) {  // the transfers of one call start from zero whatever happens to diff
            const size_t xfer_words = (size_t)(S > 1 ? S - 1 : 1) * row_words;
            int rx = en->xfer.ensure(xfer_words);
            if (rx) return rx;
            CK(cudaMemsetAsync(en->xfer.p, 0, xfer_words * sizeof(unsigned long long), en->stream));
        }
        if (zero_estimators) {
            CK(cudaMemsetAsync(en->est.p, 0, en->est_count * sizeof(double), en->stream));
            if (jump) CK(cudaMemsetAsync(en->diff.p, 0, (size_t)S * row_words * sizeof(unsigned long long), en->stream));
            if (en->continuum) {
                CK(cudaMemsetAsync(en->cb_mom.p, 0, (size_t)S * (en->n_phot + 1) * tbc::N_MOMENTS * sizeof(double), en->stream));
                CK(cudaMemsetAsync(en->cont_lit.p, 0, (size_t)5 * (en->n_continua > 0 ? en->n_continua : 1) * S * sizeof(double), en->stream));
            }
        }
        CK(cudaMemsetAsync(en->ctrl.p, 0, (2 + tb::CNT_COUNT) * sizeof(unsigned long long), en->stream));
        CK(cudaMemsetAsync(en->error.p, 0, sizeof(int), en->stream));
        en->timing_valid = false;
        en->est_unreduced = true;
    } else {
        CK(cudaMemsetAsync(en->ctrl.p, 0, sizeof(unsigned long long), en->stream));  // next_packet only
    }
    const int threads = en->threads_per_cta;
    const bool vpackets = !en->continuum && en->cfg.number_of_vpackets > 0;
    const bool want_pool = jump && en->pooled && !vpackets;
    const bool warp_volley = jump && vpackets;
    // resident CTAs per SM (x 256 threads), measured with scripts/perf_probe.py on the bench model on an H100 SXM at a 400 W power
    // limit: the pooled classic kernel (2e7 packets) is fastest at 2 of 1-4, the pooled continuum kernel (4e6 packets, 50 shells)
    // at 2 rather than 3, and the warp-volley kernel of virtual packets (1e8 packets x 10) at 2 rather than 3 (3.73 vs 3.90 s;
    // at 3 or 4 CTAs it is held to 80 / 64 registers and spills, at 2 it has 128 and none).  The lane-resident jump kernel
    // (option pooled = 0; 3 with continuum) and the scan kernel (3) are not re-measured on the H100.  Each kernel is compiled
    // for its own count (__launch_bounds__, the dispatch below); the option ctas_per_sm only sizes the grid, at most to what fits.
    const int ctas_per_sm = en->ctas_per_sm > 0 ? en->ctas_per_sm
                                                : (en->nonhomologous ? 2 : (en->algorithm == 1 ? (en->continuum ? (want_pool ? 2 : 3) : 2) : 3));
    const int grid = en->sm_count * ctas_per_sm;
    const size_t n_warps = (size_t)grid * (threads / 32);
    int r;
    const int park_min = en->park_min < 1 ? (want_pool ? 32 : 16) : (en->park_min > 32 ? 32 : en->park_min);
    const int pool_slots = (32 + park_min + 1) & ~1;  // a trace step can park 32 packets on top of park_min - 1 waiting ones
    // the pools need shared memory next to the per-CTA J / nu_bar rows; with very many shells fall back to one packet per lane
    const bool pooled = want_pool &&
                        (size_t)4 * S * sizeof(double) + (size_t)(threads / 32) * pool_slots * tb::pool_bytes_per_slot(en->continuum != 0) <= 110 * 1024;
    const int rng_units = pooled ? 32 + pool_slots : 32;
    if ((r = en->rng_buf.ensure(n_warps * tb::MT_N * rng_units))) return r;

    tb::KParams P{};
    P.n_shells = S; P.n_lines = en->L; P.lpad = en->lpad;
    P.r_inner = en->r_inner.p; P.r_outer = en->r_outer.p; P.n_e = en->n_e.p; P.nu_line = en->nu_line.p; P.tau_t = en->tau_t.p;
    P.tau_prefix = en->prefix.p;
    P.nu_first_le = en->first_le.p; P.nu_key_min = en->key_min; P.n_keys = en->n_keys;
    P.t_exp = en->t_exp; P.ct = tb::C_LIGHT * en->t_exp; P.inv_ct = 1.0 / P.ct; P.sigma_thomson = en->cfg.sigma_thomson;
    P.n_transitions = en->T; P.tpad = en->tpad; P.n_blocks = en->n_blocks;
    P.tp_t = en->tp_t.p; P.line2macro = en->line2macro.p; P.block_edge = en->block_edge.p; P.ttype = en->ttype.p;
    P.dest = en->dest.p; P.tline = en->tline.p;
    P.continuum = en->continuum;
    if (en->continuum) {
        P.n_continua = en->n_continua; P.n_phot = en->n_phot; P.phot_pad = en->phot_pad; P.n_activation = en->n_activation;
        P.k_packet_idx = (int)en->k_packet_idx; P.n_markov = en->n_markov;
        P.t_e = en->t_e.p; P.bf_thr = en->bf_thr.p; P.pi_min = en->pi_min.p; P.pi_max = en->pi_max.p; P.x_sect = en->x_sect.p;
        P.phot_nus = en->phot_nus.p; P.ff_factor = en->ff_factor.p; P.pi_refs = en->pi_refs.p; P.pi_act = en->pi_act.p;
        P.chi_bf_t = en->chi_bf_t.p; P.emiss_t = en->emiss_t.p; P.markov_cum = en->markov_cum.p;
        // FF_OPAC_CONST, opacities/opacities.py:25-27 (CODATA-2010 cgs)
        const double m_el = 9.10938291e-28, k_b = 1.3806488e-16, e_esu = 4.80320425e-10, h_pl = 6.62606957e-27;
        P.ff_opac_const = pow(2 * M_PI / (3 * m_el * k_b), 0.5) * 4 * pow(e_esu, 6) / (3 * m_el * h_pl * tb::C_LIGHT);
        P.cont_bins = en->cont_bins; P.cb_n_gkeys = en->cb_n_gkeys; P.cb_gkey_min = en->cb_gkey_min;
        P.cb_B = en->cb_B.p; P.cb_guide = en->cb_guide.p; P.cb_nact = en->cb_nact.p; P.cb_chi_lin = en->cb_chi_lin.p;
        P.cb_act_start = en->cb_act_start.p; P.cb_act = reinterpret_cast<const int2 *>(en->cb_act.p);
        P.cb_mom = en->cb_mom.p; P.cont_lit = en->cont_lit.p;
    }
    P.full_rel = (en->cfg.enable_full_relativity || en->continuum) ? 1 : 0; P.line_mode = en->cfg.line_interaction_type;
    P.disable_line = en->cfg.disable_line_scattering; P.n_vpackets = en->continuum ? 0 : (int)en->cfg.number_of_vpackets;
    P.survival_probability = en->cfg.survival_probability; P.tau_russian = en->cfg.vpacket_tau_russian;
    P.spawn_start = en->cfg.vpacket_spawn_start_frequency; P.spawn_end = en->cfg.vpacket_spawn_end_frequency;
    P.lum_nu_start = en->cfg.luminosity_nu_start;
    P.lum_nu_end = en->cfg.luminosity_nu_end > 0.0 ? en->cfg.luminosity_nu_end : INFINITY;  // an all-zero config means "no window"
    P.grid = en->grid.p; P.n_grid = en->n_grid; P.grid0 = en->grid0; P.grid_last = en->grid_last; P.inv_dgrid = en->inv_dgrid;
    constexpr int BULK_REPS = 256;
    {
        const int rep_stride = 2 * S + 4 + (en->continuum ? S : 0);  // {J | nu_bar | luminosity sums | ff_heating}
        P.rep_stride = rep_stride;
        if ((r = en->bulk_rep.ensure((size_t)BULK_REPS * rep_stride)) || (r = en->cnt_rep.ensure((size_t)BULK_REPS * tb::CNT_COUNT))) return r;
        if (first) {
            CK(cudaMemsetAsync(en->bulk_rep.p, 0, (size_t)BULK_REPS * rep_stride * sizeof(double), en->stream));
            CK(cudaMemsetAsync(en->cnt_rep.p, 0, (size_t)BULK_REPS * tb::CNT_COUNT * sizeof(unsigned long long), en->stream));
        }
        P.cnt_rep = en->cnt_rep.p;
        P.macro_guide = (en->have_macro_guide && !en->continuum) ? en->macro_guide.p : nullptr;
        P.macro_next = (en->have_macro_guide && !en->continuum) ? en->macro_next.p : nullptr;
        P.macro_entry = (en->have_macro_guide && !en->continuum) ? en->macro_entry.p : nullptr;
        P.bulk_rep = en->bulk_rep.p; P.bulk_reps = BULK_REPS;
    }
    if (en->nonhomologous) { P.v_inner = en->v_inner.p; P.v_outer = en->v_outer.p; P.dvdr = en->dvdr.p; }
    P.vol_min = en->vol_min;
    P.refill_min = en->refill_min > 0 ? en->refill_min : (pooled && !en->continuum ? 12 : 8); P.park_min = park_min; P.pool_slots = pool_slots; P.rng_units = rng_units;
    P.J = en->est.p + en->off_J; P.nubar = en->est.p + en->off_nubar; P.vhist = en->est.p + en->off_vhist;
    P.jblue_t = en->est.p + en->off_jblue; P.edotlu_t = en->est.p + en->off_edotlu;
    if (en->n_grid > 1) { P.spec_emitted = en->est.p + en->off_spec; P.spec_reabsorbed = P.spec_emitted + (en->n_grid - 1); }
    P.rng_buf = en->rng_buf.p;
    P.next_packet = en->ctrl.p; P.vlog_count = en->ctrl.p + 1; P.counters = en->ctrl.p + 2;
    P.error = en->error.p;
    // fixed-point scales of the jump algorithm: typical term -> 2^58 (see fixed_add)
    {
        const double e_typ = en->e_typ > 0 ? en->e_typ : 1.0;
        const double w1 = P.full_rel ? e_typ : e_typ / en->nu_typ;
        const double w2 = w1 / en->nu_typ;
        P.scale1 = ldexp(1.0, tb::FIXED_TYPICAL_LOG2 - ilogb(w1));
        P.scale2 = ldexp(1.0, tb::FIXED_TYPICAL_LOG2 - ilogb(w2));
        P.diff = en->diff.p; P.xfer = en->xfer.p;
        if (jump) {
            // accumulating (zero_estimators == 0) into difference arrays that were filled at another scale would mix units
            if (first && zero_estimators) { en->diff_scale1 = 0.0; en->diff_scale2 = 0.0; }
            if (en->diff_scale1 != 0.0 && (en->diff_scale1 != P.scale1 || en->diff_scale2 != P.scale2))
                return fail(TB200_ERR_INVALID, "zero_estimators = 0 with packets whose typical energy differs from the accumulated run's "
                                               "(the fixed-point line estimators would mix scales): start a fresh accumulation");
            en->diff_scale1 = P.scale1; en->diff_scale2 = P.scale2;
        }
    }

    if (n > 0) {
        if ((r = en->start_rec.ensure((size_t)en->N))) return r;
        P.n_packets = n;
        P.in_r = en->in_r.p + off; P.in_nu = en->in_nu.p + off; P.in_mu = en->in_mu.p + off; P.in_energy = en->in_energy.p + off;
        P.seed = en->seed32.p + off; P.seed_x397 = en->x397.p + off;
        P.start = en->start_rec.p + off;
        P.out_nu = en->out_nu.p + off; P.out_energy = en->out_energy.p + off;
        if (en->track_last) {
            long long *li = en->last_i.p + off; double *ld = en->last_d.p + off; const int64_t N = en->N;
            P.last_type = li; P.last_event_id = li + N; P.last_shell = li + 2 * N; P.last_absorb = li + 3 * N; P.last_emit = li + 4 * N;
            P.last_radius = ld; P.last_before_nu = ld + N; P.last_before_mu = ld + 2 * N; P.last_before_energy = ld + 3 * N;
            P.last_after_nu = ld + 4 * N; P.last_after_mu = ld + 5 * N; P.last_after_energy = ld + 6 * N;
        }
        if (en->n_tracked > 0 && off == 0) { P.events = en->events.p; P.event_counts = en->event_counts.p; P.n_tracked = en->n_tracked; P.max_events = en->max_events; }
        if (en->vlog_capacity > 0) {
            double *v = en->vlog_d.p; const int64_t cap = en->vlog_capacity;
            P.vlog_nu = v; P.vlog_energy = v + cap; P.vlog_mu = v + 2 * cap; P.vlog_r = v + 3 * cap; P.vlog_pid = en->vlog_pid.p; P.vlog_capacity = cap;
        }
        size_t smem = (size_t)(en->algorithm == 1 ? 4 : 2) * S * sizeof(double);  // jump: [4 S] shell table; scan: J, nu_bar rows
        if (en->nonhomologous) smem = 0;  // (its bulk estimators go to the global replicas)
        if (smem > 200 * 1024) return fail(TB200_ERR_INVALID, "too many shells for the shared-memory bulk estimators");
        if (pooled) {  // packet pools of the warps
            P.park_off = (int)(smem / sizeof(double));
            smem += (size_t)(threads / 32) * pool_slots * tb::pool_bytes_per_slot(en->continuum != 0);
        } else if (jump) {
            // parked-lane columns (tb::TraceColumns), one per thread
            const bool cont = en->continuum != 0;
            P.park_off = (int)(smem / sizeof(double));
            smem += (size_t)(tb::trace_nd(cont) * sizeof(double) + tb::trace_ni(cont) * sizeof(int)) * threads;
            if (warp_volley) {  // item slots of the warp-cooperative virtual-packet volleys
                P.vol_off = (int)(smem / sizeof(double));
                smem += (size_t)(threads / 32) * tb::vol_doubles_per_warp(P.full_rel != 0) * sizeof(double);
            }
        }
#define TB_LAUNCH(KERNEL)                                                                                                  \
    do {                                                                                                                   \
        /* refused here rather than by cudaFuncSetAttribute, whose error would stay pending and fail the next launch */   \
        cudaFuncAttributes fa__;                                                                                           \
        CK(cudaFuncGetAttributes(&fa__, KERNEL));                                                                          \
        if (smem + fa__.sharedSizeBytes > en->smem_optin)                                                                  \
            return fail(TB200_ERR_INVALID, "too many shells for the transport kernel's shared memory with this configuration"); \
        if (smem > 48 * 1024) CK(cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));    \
        int fit = 0;                                                                                                       \
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&fit, KERNEL, threads, smem));                                    \
        if (fit < 1) return fail(TB200_ERR_INVALID, "transport kernel does not fit on an SM with this configuration");     \
        const int resident_grid = en->sm_count * (fit < ctas_per_sm ? fit : ctas_per_sm);  /* persistent CTAs only */ \
        KERNEL<<<resident_grid, threads, smem, en->stream>>>();                                                            \
    } while (0)
        CK(cudaMemcpyToSymbolAsync(tb::cP, &P, sizeof(P), 0, cudaMemcpyHostToDevice, en->stream));
        // The processing order by initial frequency, inside this range (indices are relative to the range), recomputed on every
        // launch (every iteration brings new packets).  It writes each packet's start record at its slot, computed from the
        // range's packets and the model in cP, and the seed words by packet id (tb::order_scatter_kernel).
        {
            const long long *seeds64 = en->seeds64.p + off;
            unsigned *seed32 = en->seed32.p + off, *x397 = en->x397.p + off;
            tb::StartRecord *rec = en->start_rec.p + off;
            if (en->sort_packets) {
                const int shift = 52 - en->sort_bits;
                const long long okey_min = (en->key_min << tb::NU_KEY_SHIFT) >> shift;
                const long long okey_max = (((en->key_min + en->n_keys - 1) << tb::NU_KEY_SHIFT) >> shift);
                const int n_okeys = (int)(okey_max - okey_min + 1);
                if ((r = en->order_hist.ensure((size_t)n_okeys))) return r;
                const unsigned nblk = (unsigned)((n + 256 * tb::ORDER_ITEMS - 1) / (256 * tb::ORDER_ITEMS));
                CK(cudaMemsetAsync(en->order_hist.p, 0, (size_t)n_okeys * sizeof(unsigned), en->stream));
                tb::order_hist_kernel<<<nblk, 256, 0, en->stream>>>(en->in_nu.p + off, n, shift, okey_min, n_okeys, en->order_hist.p);
                tb::order_scan_kernel<<<1, 1024, 0, en->stream>>>(en->order_hist.p, n_okeys);
#define TB_SCATTER(START) \
    tb::order_scatter_kernel<START><<<nblk, 256, 0, en->stream>>>(en->in_nu.p + off, n, shift, okey_min, n_okeys, en->order_hist.p, seeds64, seed32, x397, rec)
                if (en->nonhomologous) TB_SCATTER(nh::NhStart);
                else if (P.full_rel) TB_SCATTER(tb::ClassicStart<true>);
                else TB_SCATTER(tb::ClassicStart<false>);
#undef TB_SCATTER
                en->launches += 3;
            } else {
                const unsigned nblk = (unsigned)((n + 255) / 256);
                if (en->nonhomologous) tb::start_record_kernel<nh::NhStart><<<nblk, 256, 0, en->stream>>>(n, seeds64, seed32, x397, rec);
                else if (P.full_rel) tb::start_record_kernel<tb::ClassicStart<true>><<<nblk, 256, 0, en->stream>>>(n, seeds64, seed32, x397, rec);
                else tb::start_record_kernel<tb::ClassicStart<false>><<<nblk, 256, 0, en->stream>>>(n, seeds64, seed32, x397, rec);
                en->launches++;
            }
            CK(cudaGetLastError());
        }
        if (ev_a) CK(cudaEventRecord(ev_a, en->stream));
        // one kernel per mode, compiled for the CTAs per SM its default runs at (see ctas_per_sm above)
        if (en->nonhomologous) {  // whatever the algorithm / pooled options say
            TB_LAUNCH(nh::transport_nonhomologous_kernel);
        } else if (en->continuum) {  // IIP mode: full relativity always (modes/iip/packet_propagation.py:104,123)
            if (pooled) TB_LAUNCH((tb::transport_pool_kernel<true, 2, true>));
            else if (en->algorithm == 1) TB_LAUNCH((tb::transport_jump_kernel<true, 3, true>));
            else TB_LAUNCH((tb::transport_scan_kernel<true, 2, true>));
        } else if (en->algorithm == 0) {
            if (P.full_rel) TB_LAUNCH((tb::transport_scan_kernel<true, 3, false>)); else TB_LAUNCH((tb::transport_scan_kernel<false, 3, false>));
        } else if (pooled) {
            if (P.full_rel) TB_LAUNCH((tb::transport_pool_kernel<true, 2>)); else TB_LAUNCH((tb::transport_pool_kernel<false, 2>));
        } else if (warp_volley) {  // virtual packets: warp-cooperative volleys
            if (P.full_rel) TB_LAUNCH((tb::transport_jump_kernel<true, 2, false, true>)); else TB_LAUNCH((tb::transport_jump_kernel<false, 2, false, true>));
        } else {  // option pooled = 0, or the pools do not fit
            if (P.full_rel) TB_LAUNCH((tb::transport_jump_kernel<true, 2, false>)); else TB_LAUNCH((tb::transport_jump_kernel<false, 2, false>));
        }
#undef TB_LAUNCH
        en->launches++;
        CK(cudaGetLastError());
        if (ev_b) CK(cudaEventRecord(ev_b, en->stream));
    }
    if (last) {
        const int rep_stride = 2 * S + 4 + (en->continuum ? S : 0);
        const int nred = rep_stride > tb::CNT_COUNT ? rep_stride : tb::CNT_COUNT;
        tb::reduce_bulk_kernel<<<(nred + 127) / 128, 128, 0, en->stream>>>(en->bulk_rep.p, en->bulk_reps_used, S, rep_stride, en->est.p + en->off_J,
                                                                         en->est.p + en->off_nubar, en->est.p + en->off_lum,
                                                                         en->continuum ? en->est.p + en->off_ffheat : nullptr, en->cnt_rep.p, en->ctrl.p + 2);
        en->launches++;
        CK(cudaGetLastError());
        if (en->continuum && en->n_continua > 0) {
            const int ncs = en->n_continua * S;
            tb::continuum_finalize_kernel<<<(ncs + 127) / 128, 128, 0, en->stream>>>(en->cb_mom.p, en->cont_lit.p, en->cb_B.p, en->n_phot, en->phot_nus.p,
                en->x_sect.p, en->cb_pos.p, en->pi_refs.p, en->bf_thr.p, en->n_continua, S, en->cont_bins, en->est.p + en->off_cont);
            en->launches++;
            CK(cudaGetLastError());
        }
    }
    if (last && jump) {
        // diff[s] += xfer[s - 1] - xfer[s]: from here on diff holds every trace's +w / -w pair (trace_range_end)
        tb::fold_transfers_kernel<<<(unsigned)((row_words / 2 + 255) / 256), 256, 0, en->stream>>>(en->diff.p, en->xfer.p, S, row_words);
        en->launches++;
        CK(cudaGetLastError());
        tb::finalize_line_estimators_kernel<<<2 * S, tb::FIN_THREADS, 0, en->stream>>>(en->diff.p, en->nu_line.p, en->L, en->lpad, 1.0 / P.scale1,
                                                                         1.0 / P.scale2, P.full_rel, P.jblue_t, P.edotlu_t, en->error.p);
        en->launches++;
        CK(cudaGetLastError());
    }
    return TB200_OK;
}

static int launch_transport(tb200_engine *en, int zero_estimators) {
    int r = launch_range(en, 0, en->N, true, true, zero_estimators, en->ev_start, en->ev_stop);
    if (r) return r;
    CK(cudaEventRecord(en->ev_fin, en->stream));
    en->timing_valid = en->N > 0;
    en->chunked_timing = false;
    return TB200_OK;
}

int tb200_transport(tb200_engine *en, int zero_estimators) {
    if (!en) return fail(TB200_ERR_INVALID, "bad argument");
    int r;
    if ((r = prepare_tracking(en, nullptr))) return r;
    return launch_transport(en, zero_estimators);
}

int tb200_sync(tb200_engine *en) {
    if (!en) return fail(TB200_ERR_INVALID, "bad argument");
    CK(cudaSetDevice(en->device));
    CK(cudaStreamSynchronize(en->stream));
    if (!en->error.p) return TB200_OK;
    int err = 0;
    CK(cudaMemcpy(&err, en->error.p, sizeof(int), cudaMemcpyDeviceToHost));
    if (err == tb::ERR_NU_DIFF) return fail(TB200_ERR_NU_DIFF, "nu difference is less than 0.0");
    if (err == tb::ERR_MACRO_ATOM) return fail(TB200_ERR_MACRO_ATOM, "MacroAtom ran out of the block / unknown transition type");
    if (err == tb::ERR_VPACKET_LOOP) return fail(TB200_ERR_VPACKET_LOOP, "virtual packet did not leave the grid");
    if (err == tb::ERR_CONTINUUM) return fail(TB200_ERR_CONTINUUM, "continuum tables inconsistent (frequency outside a cross-section block or index out of range)");
    if (err == tb::ERR_STUCK) return fail(TB200_ERR_INVALID, "a packet exceeded the event watchdog (4e6 events): inconsistent tables or an engine bug");
    if (err == tb::ERR_FIXED_POINT) return fail(TB200_ERR_INVALID, "fixed-point line-estimator accumulator out of range (packet energy / frequency far from the typical values, or more than ~2^28 traces through one (line, shell) cell)");
    return TB200_OK;
}

int tb200_get_counters(tb200_engine *en, tb200_counters *c) {
    if (!en || !c) return fail(TB200_ERR_INVALID, "bad argument");
    CK(cudaSetDevice(en->device));
    unsigned long long h[2 + tb::CNT_COUNT] = {0};
    if (en->ctrl.p) {
        CK(cudaStreamSynchronize(en->stream));
        CK(cudaMemcpy(h, en->ctrl.p, sizeof(h), cudaMemcpyDeviceToHost));
    }
    const unsigned long long *k = h + 2;
    c->n_line_steps = (int64_t)k[tb::CNT_LINE_STEPS]; c->n_boundary_events = (int64_t)k[tb::CNT_BOUNDARY];
    c->n_line_events = (int64_t)k[tb::CNT_LINE_EVENTS]; c->n_escat_events = (int64_t)k[tb::CNT_ESCAT_EVENTS];
    c->n_rng_draws = (int64_t)k[tb::CNT_RNG_DRAWS]; c->n_macro_jumps = (int64_t)k[tb::CNT_MACRO_JUMPS];
    c->n_macro_scanned = (int64_t)k[tb::CNT_MACRO_SCANNED]; c->n_vpackets = (int64_t)k[tb::CNT_VPACKETS];
    c->n_vpacket_line_steps = (int64_t)k[tb::CNT_VPACKET_LINE_STEPS];
    c->n_continuum_events = (int64_t)k[tb::CNT_CONT_EVENTS]; c->n_bf_estimator_updates = (int64_t)k[tb::CNT_BF_UPDATES];
    c->n_search_probes = (int64_t)k[tb::CNT_PROBES];
    return TB200_OK;
}

int tb200_download(tb200_engine *en, tb200_outputs *o) {
    if (!en || !o) return fail(TB200_ERR_INVALID, "bad argument");
    if (!en->have_model) return fail(TB200_ERR_NO_MODEL, "tb200_set_model has not been called");
    CK(cudaSetDevice(en->device));
    const int S = en->S, L = en->L;
    const int64_t N = en->N;
    cudaStream_t st = en->stream;
    // what was not recorded cannot be downloaded: tb200_transport runs without tracking, only tb200_run arms it
    if (o->last_interaction_type && !en->track_last)
        return fail(TB200_ERR_INVALID, "last-interaction columns requested, but the last transport ran without tracking (use tb200_run)");
    if (o->events && o->n_tracked_packets > 0 && en->n_tracked == 0)
        return fail(TB200_ERR_INVALID, "event log requested, but the last transport ran without it (use tb200_run)");
    if (o->vlog_nus && o->vlog_capacity > 0 && en->vlog_capacity == 0)
        return fail(TB200_ERR_INVALID, "virtual-packet log requested, but the last transport ran without it (use tb200_run)");
    if (o->output_nus && N) CK(cudaMemcpyAsync(o->output_nus, en->out_nu.p, N * sizeof(double), cudaMemcpyDeviceToHost, st));
    if (o->output_energies && N) CK(cudaMemcpyAsync(o->output_energies, en->out_energy.p, N * sizeof(double), cudaMemcpyDeviceToHost, st));
    if (o->j) CK(cudaMemcpyAsync(o->j, en->est.p + en->off_J, S * sizeof(double), cudaMemcpyDeviceToHost, st));
    if (o->nu_bar) CK(cudaMemcpyAsync(o->nu_bar, en->est.p + en->off_nubar, S * sizeof(double), cudaMemcpyDeviceToHost, st));
    if (o->vhist && en->n_grid > 0) CK(cudaMemcpyAsync(o->vhist, en->est.p + en->off_vhist, en->n_grid * sizeof(double), cudaMemcpyDeviceToHost, st));
    if (en->n_grid > 1) {
        const size_t nb = (size_t)en->n_grid - 1;
        if (o->spectrum_emitted) CK(cudaMemcpyAsync(o->spectrum_emitted, en->est.p + en->off_spec, nb * sizeof(double), cudaMemcpyDeviceToHost, st));
        if (o->spectrum_reabsorbed) CK(cudaMemcpyAsync(o->spectrum_reabsorbed, en->est.p + en->off_spec + nb, nb * sizeof(double), cudaMemcpyDeviceToHost, st));
    }
    if (o->luminosity_sums) CK(cudaMemcpyAsync(o->luminosity_sums, en->est.p + en->off_lum, 4 * sizeof(double), cudaMemcpyDeviceToHost, st));
    std::vector<double> stats_tmp;
    if (en->continuum && en->n_continua > 0) {
        const size_t ncs = (size_t)en->n_continua * S;
        const double *cb = en->est.p + en->off_cont;
        if (o->ff_heating_estimator) CK(cudaMemcpyAsync(o->ff_heating_estimator, en->est.p + en->off_ffheat, S * sizeof(double), cudaMemcpyDeviceToHost, st));
        double *dst[4] = {o->photo_ion_estimator, o->stim_recomb_estimator, o->bf_heating_estimator, o->stim_recomb_cooling_estimator};
        for (int k = 0; k < 4; k++) if (dst[k]) CK(cudaMemcpyAsync(dst[k], cb + k * ncs, ncs * sizeof(double), cudaMemcpyDeviceToHost, st));
        if (o->photo_ion_estimator_statistics) {
            stats_tmp.resize(ncs);
            CK(cudaMemcpyAsync(stats_tmp.data(), cb + 4 * ncs, ncs * sizeof(double), cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            for (size_t i = 0; i < ncs; i++) o->photo_ion_estimator_statistics[i] = (int64_t)llround(stats_tmp[i]);
        }
    } else if (en->continuum && o->ff_heating_estimator) {
        CK(cudaMemcpyAsync(o->ff_heating_estimator, en->est.p + en->off_ffheat, S * sizeof(double), cudaMemcpyDeviceToHost, st));
    }
    int r;
    if (o->j_blue && (r = download_line_major(en, en->est.p + en->off_jblue, L, en->lpad, o->j_blue))) return r;
    if (o->edotlu && (r = download_line_major(en, en->est.p + en->off_edotlu, L, en->lpad, o->edotlu))) return r;
    if (o->last_interaction_type && en->track_last && N) {
        long long *li = en->last_i.p; double *ld = en->last_d.p;
        int64_t *di[5] = {o->last_interaction_type, o->last_event_id, o->last_shell_id, o->last_line_absorb_id, o->last_line_emit_id};
        double *dd[7] = {o->last_radius, o->last_before_nu, o->last_before_mu, o->last_before_energy, o->last_after_nu, o->last_after_mu, o->last_after_energy};
        for (int k = 0; k < 5; k++) if (di[k]) CK(cudaMemcpyAsync(di[k], li + (size_t)k * N, N * sizeof(long long), cudaMemcpyDeviceToHost, st));
        for (int k = 0; k < 7; k++) if (dd[k]) CK(cudaMemcpyAsync(dd[k], ld + (size_t)k * N, N * sizeof(double), cudaMemcpyDeviceToHost, st));
    }
    if (o->events && en->n_tracked > 0) {
        CK(cudaMemcpyAsync(o->events, en->events.p, (size_t)en->n_tracked * en->max_events * sizeof(tb::Event), cudaMemcpyDeviceToHost, st));
        if (o->event_counts) CK(cudaMemcpyAsync(o->event_counts, en->event_counts.p, en->n_tracked * sizeof(long long), cudaMemcpyDeviceToHost, st));
    }
    o->vlog_count = 0;
    if (o->vlog_nus && en->vlog_capacity > 0) {
        unsigned long long cnt = 0;
        CK(cudaStreamSynchronize(st));
        CK(cudaMemcpy(&cnt, en->ctrl.p + 1, sizeof(cnt), cudaMemcpyDeviceToHost));
        o->vlog_count = (int64_t)cnt;
        size_t m = (size_t)(cnt < (unsigned long long)en->vlog_capacity ? cnt : (unsigned long long)en->vlog_capacity);
        const int64_t cap = en->vlog_capacity;
        if (m) {
            CK(cudaMemcpyAsync(o->vlog_nus, en->vlog_d.p, m * sizeof(double), cudaMemcpyDeviceToHost, st));
            if (o->vlog_energies) CK(cudaMemcpyAsync(o->vlog_energies, en->vlog_d.p + cap, m * sizeof(double), cudaMemcpyDeviceToHost, st));
            if (o->vlog_initial_mus) CK(cudaMemcpyAsync(o->vlog_initial_mus, en->vlog_d.p + 2 * cap, m * sizeof(double), cudaMemcpyDeviceToHost, st));
            if (o->vlog_initial_rs) CK(cudaMemcpyAsync(o->vlog_initial_rs, en->vlog_d.p + 3 * cap, m * sizeof(double), cudaMemcpyDeviceToHost, st));
            if (o->vlog_packet_index) CK(cudaMemcpyAsync(o->vlog_packet_index, en->vlog_pid.p, m * sizeof(long long), cudaMemcpyDeviceToHost, st));
        }
    }
    CK(cudaStreamSynchronize(st));
    return tb200_get_counters(en, &o->counters);
}

// Host packets in, host results out.  With enough packets and no per-packet tracking requested, the packets are
// processed in `pipeline_chunks` ranges so that the H2D copy of range c+1, the kernels of range c and the D2H copy
// of the outputs of range c-1 overlap (three streams; true overlap needs page-locked host buffers).
// (pk == nullptr: the packets already lie in HBM -- uploaded earlier or generated by tb200_create_packets -- and only the
//  per-packet outputs of range c-1 travel while range c computes)
// log_on_device: the virtual-packet log stays in the engine's device buffer and only its count comes back (an engine group
// copies the rows of all members straight into the caller's arrays afterwards).
static int run_pipelined(tb200_engine *en, const tb200_packets *pk, tb200_outputs *o, bool log_on_device = false) {
    int r;
    const int64_t n = pk ? pk->n_packets : en->N;
    const bool tracking = o->last_interaction_type || (o->events && o->n_tracked_packets > 0) || (o->vlog_nus && o->vlog_capacity > 0);
    int chunks = en->pipeline_chunks;
    if (tracking || n < 4000000 || chunks <= 1) {
        if (pk && (r = tb200_upload_packets(en, pk))) return r;
        if ((r = prepare_tracking(en, o))) return r;
        if ((r = launch_transport(en, 1))) return r;
        if ((r = tb200_sync(en))) return r;
        if (!log_on_device) return tb200_download(en, o);
        tb200_outputs q = *o;
        q.vlog_nus = nullptr;
        if ((r = tb200_download(en, &q))) return r;
        o->counters = q.counters;
        unsigned long long cnt = 0;
        if (en->vlog_capacity > 0) CK(cudaMemcpy(&cnt, en->ctrl.p + 1, sizeof(cnt), cudaMemcpyDeviceToHost));
        o->vlog_count = (int64_t)cnt;
        return TB200_OK;
    }
    if (!en->have_model) return fail(TB200_ERR_NO_MODEL, "tb200_set_model has not been called");
    if (n > 2000000000LL) return fail(TB200_ERR_INVALID, "n_packets out of range");
    CK(cudaSetDevice(en->device));
    if (pk) {
        en->N = n;
        if ((r = ensure_packet_arrays(en, n))) return r;
    }
    if ((r = prepare_tracking(en, nullptr))) return r;
    if (pk) set_typical_energy(en, pk);
    std::vector<Event> ev_up(chunks), ev_k0(chunks), ev_k1(chunks);
    for (int c = 0; c < chunks; c++) { CK(cudaEventCreateWithFlags(&ev_up[c].h, cudaEventDisableTiming)); CK(cudaEventCreate(&ev_k0[c].h)); CK(cudaEventCreate(&ev_k1[c].h)); }
    int rc = TB200_OK;
    // Range boundaries: the first and the last range are a quarter of the others -- the H2D copy of the first range and the
    // D2H copy of the last one are the only transfers nothing hides (option pipeline_edges = 0: all ranges equal)
    std::vector<int64_t> edge((size_t)chunks + 1);
    {
        const int64_t small = (en->pipeline_edges && chunks >= 4) ? n / (4 * (int64_t)chunks) : 0;
        if (small > 0) {
            const int64_t rest = n - 2 * small;
            edge[0] = 0; edge[(size_t)chunks] = n;
            for (int c = 1; c < chunks; c++) edge[(size_t)c] = small + rest * (c - 1) / (chunks - 2);
        } else {
            for (int c = 0; c <= chunks; c++) edge[(size_t)c] = n * c / chunks;
        }
    }
    for (int c = 0; c < chunks && rc == TB200_OK; c++) {
        const int64_t lo = edge[(size_t)c], hi = edge[(size_t)c + 1], m = hi - lo;
        cudaStream_t hs = en->h2d_stream;
        auto chk = [&](cudaError_t e) { if (e != cudaSuccess && rc == TB200_OK) rc = fail(TB200_ERR_CUDA, cudaGetErrorString(e)); };
        if (pk) {
            chk(cudaMemcpyAsync(en->in_r.p + lo, pk->initial_radii + lo, m * sizeof(double), cudaMemcpyHostToDevice, hs));
            chk(cudaMemcpyAsync(en->in_nu.p + lo, pk->initial_nus + lo, m * sizeof(double), cudaMemcpyHostToDevice, hs));
            chk(cudaMemcpyAsync(en->in_mu.p + lo, pk->initial_mus + lo, m * sizeof(double), cudaMemcpyHostToDevice, hs));
            chk(cudaMemcpyAsync(en->in_energy.p + lo, pk->initial_energies + lo, m * sizeof(double), cudaMemcpyHostToDevice, hs));
            chk(cudaMemcpyAsync(en->seeds64.p + lo, pk->packet_seeds + lo, m * sizeof(long long), cudaMemcpyHostToDevice, hs));
            chk(cudaEventRecord(ev_up[c], hs));
            chk(cudaStreamWaitEvent(en->stream, ev_up[c], 0));
        }
        if (rc) break;
        if ((rc = launch_range(en, lo, m, c == 0, c == chunks - 1, 1, ev_k0[c], ev_k1[c]))) break;
        // outputs of this range go back while the next range computes
        chk(cudaStreamWaitEvent(en->d2h_stream, ev_k1[c], 0));
        if (o->output_nus) chk(cudaMemcpyAsync(o->output_nus + lo, en->out_nu.p + lo, m * sizeof(double), cudaMemcpyDeviceToHost, en->d2h_stream));
        if (o->output_energies) chk(cudaMemcpyAsync(o->output_energies + lo, en->out_energy.p + lo, m * sizeof(double), cudaMemcpyDeviceToHost, en->d2h_stream));
    }
    if (rc == TB200_OK) {
        if (cudaEventRecord(en->ev_fin, en->stream) != cudaSuccess) rc = fail(TB200_ERR_CUDA, "cudaEventRecord");
    }
    if (rc == TB200_OK) rc = tb200_sync(en);
    cudaStreamSynchronize(en->d2h_stream);
    cudaStreamSynchronize(en->h2d_stream);
    double total_ms = 0.0;
    for (int c = 0; c < chunks; c++) {
        float f = 0.0f;
        if (rc == TB200_OK && cudaEventElapsedTime(&f, ev_k0[c], ev_k1[c]) == cudaSuccess) total_ms += f;
    }
    if (rc) return rc;
    en->chunk_kernel_ms = total_ms; en->chunked_timing = true; en->timing_valid = true;
    // estimators (and anything else but the per-packet outputs, which are already on their way)
    tb200_outputs rest = *o;
    rest.output_nus = nullptr; rest.output_energies = nullptr;
    r = tb200_download(en, &rest);
    o->counters = rest.counters; o->vlog_count = rest.vlog_count;
    return r;
}

int tb200_run(tb200_engine *en, const tb200_packets *pk, tb200_outputs *o) {
    if (!en || !pk || !o) return fail(TB200_ERR_INVALID, "bad argument");
    return run_pipelined(en, pk, o);
}

int tb200_run_resident(tb200_engine *en, tb200_outputs *o) {
    if (!en || !o) return fail(TB200_ERR_INVALID, "bad argument");
    if (!en->have_model) return fail(TB200_ERR_NO_MODEL, "tb200_set_model has not been called");
    if (en->N <= 0 || !en->in_nu.p) return fail(TB200_ERR_INVALID, "no packets are resident: call tb200_upload_packets or tb200_create_packets first");
    return run_pipelined(en, nullptr, o);
}

static int check_line_accumulators(const tb200_engine *en) {
    if (!en->have_model) return fail(TB200_ERR_NO_MODEL, "tb200_set_model has not been called");
    if (en->algorithm != 1 || en->nonhomologous || !en->diff.p)
        return fail(TB200_ERR_INVALID, "the line accumulators exist only with algorithm = 1 (jump), outside the nonhomologous mode");
    return TB200_OK;
}

int tb200_line_accumulators(tb200_engine *en, void **device_ptr, int64_t *n_words, double *scale_j_blue, double *scale_edotlu) {
    if (!en || !device_ptr || !n_words || !scale_j_blue || !scale_edotlu) return fail(TB200_ERR_INVALID, "bad argument");
    int r;
    if ((r = check_line_accumulators(en))) return r;
    *device_ptr = en->diff.p;
    *n_words = (int64_t)en->S * (en->lpad + 1) * 4;
    *scale_j_blue = en->diff_scale2; *scale_edotlu = en->diff_scale1;  // scale1: w1 -> Edotlu, scale2: w2 -> J_blue
    return TB200_OK;
}

int tb200_finalize_line_estimators(tb200_engine *en) {
    if (!en) return fail(TB200_ERR_INVALID, "bad argument");
    int r;
    if ((r = check_line_accumulators(en))) return r;
    if (en->diff_scale1 == 0.0 || en->diff_scale2 == 0.0) return fail(TB200_ERR_INVALID, "no transport has filled the line accumulators yet");
    CK(cudaSetDevice(en->device));
    const int full_rel = (en->cfg.enable_full_relativity || en->continuum) ? 1 : 0;
    tb::finalize_line_estimators_kernel<<<2 * en->S, tb::FIN_THREADS, 0, en->stream>>>(en->diff.p, en->nu_line.p, en->L, en->lpad, 1.0 / en->diff_scale1,
        1.0 / en->diff_scale2, full_rel, en->est.p + en->off_jblue, en->est.p + en->off_edotlu, en->error.p);
    en->launches++;
    CK(cudaGetLastError());
    return TB200_OK;
}

int tb200_estimator_buffer(tb200_engine *en, void **device_ptr, int64_t *n_doubles) {
    if (!en || !device_ptr || !n_doubles) return fail(TB200_ERR_INVALID, "bad argument");
    if (!en->have_model) return fail(TB200_ERR_NO_MODEL, "tb200_set_model has not been called");
    *device_ptr = en->est.p;
    *n_doubles = (int64_t)en->est_count;
    return TB200_OK;
}

namespace {
__global__ void radfield_shell_kernel(tbr::Constants K, const double *j, const double *nu_bar, const double *volume, double time_explosion,
                                      double time_of_simulation, int n_shells, double *out /* [3 S]: t_rad, w, norm */,
                                      const double *dvdr /* [S] nonhomologous mode, or null */) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_shells) return;
    double t, w;
    tbr::dilute_planck(K, j[s], nu_bar[s], time_of_simulation, volume[s], &t, &w);
    out[s] = t; out[n_shells + s] = w;
    if (dvdr)  // modes/nonhomologous/mc_rad_field_solver.py:120-124
        out[2 * n_shells + s] = (K.c / dvdr[s]) / (4 * M_PI * time_of_simulation * volume[s]);
    else
        out[2 * n_shells + s] = K.c * time_explosion / (4 * M_PI * time_of_simulation * volume[s]);  // j_blues_norm_factor
}
__global__ void radfield_jblue_kernel(tbr::Constants K, const double *est_t, const double *nu_line, const double *shell, int n_lines, int lpad,
                                      int n_shells, double w_epsilon, int window, double *out_t) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)n_shells * lpad) return;
    const int s = (int)(i / lpad), l = (int)(i % lpad);
    out_t[i] = (l < n_lines) ? tbr::j_blue_cell(K, est_t[i], shell[2 * n_shells + s], nu_line[l], shell[s], shell[n_shells + s], w_epsilon, window != 0) : 0.0;
}
}  // namespace

int tb200_solve_radiation_field(tb200_engine *en, const tb200_radfield_params *p, double *t_radiative, double *dilution_factor, double *j_blues) {
    if (!en || !p || !p->volume) return fail(TB200_ERR_INVALID, "bad argument");
    if (!en->have_model) return fail(TB200_ERR_NO_MODEL, "tb200_set_model has not been called");
    if ((p->j == nullptr) != (p->nu_bar == nullptr) || (p->j == nullptr) != (p->j_blue == nullptr))
        return fail(TB200_ERR_INVALID, "j, nu_bar and j_blue must be given together (or all NULL for the resident estimators)");
    // a nonhomologous model carries no usable time_explosion: its J_blue normalisation needs the velocity gradient
    if (en->nonhomologous && !p->velocity_gradient)
        return fail(TB200_ERR_INVALID, "the nonhomologous mode normalises J_blue by c / velocity_gradient: pass velocity_gradient");
    if (!en->nonhomologous && p->velocity_gradient)
        return fail(TB200_ERR_INVALID, "velocity_gradient is the nonhomologous mode's normalisation; this model is homologous");
    if (p->velocity_gradient && p->detailed_optical_window)
        return fail(TB200_ERR_INVALID, "the nonhomologous radiation-field solver has no optical window");
    CK(cudaSetDevice(en->device));
    const int S = en->S, L = en->L, lpad = en->lpad;
    int r;
    if ((r = en->rf_shell.ensure((size_t)5 * S)) || (r = en->rf_volume.ensure(S)) || (r = en->rf_jblues_t.ensure((size_t)S * lpad))) return r;
    cudaStream_t st = en->stream;
    CK(cudaMemcpyAsync(en->rf_volume.p, p->volume, S * sizeof(double), cudaMemcpyHostToDevice, st));
    const double *d_j = en->est.p + en->off_J, *d_nubar = en->est.p + en->off_nubar, *d_est_t = en->est.p + en->off_jblue;
    if (p->j) {
        CK(cudaMemcpyAsync(en->rf_shell.p + 3 * S, p->j, S * sizeof(double), cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(en->rf_shell.p + 4 * S, p->nu_bar, S * sizeof(double), cudaMemcpyHostToDevice, st));
        if ((r = upload_strided_table(en, p->j_blue, L, S, S, 1, lpad, en->rf_in_t))) return r;
        d_j = en->rf_shell.p + 3 * S; d_nubar = en->rf_shell.p + 4 * S; d_est_t = en->rf_in_t.p;
    }
    tbr::Constants K;
    K.t_radiative_estimator_constant = p->t_radiative_estimator_constant; K.sigma_sb = p->sigma_sb; K.c = p->c; K.h = p->h; K.k_b = p->k_b;
    if (p->velocity_gradient) {
        if ((r = en->rf_dvdr.ensure(S))) return r;
        CK(cudaMemcpyAsync(en->rf_dvdr.p, p->velocity_gradient, S * sizeof(double), cudaMemcpyHostToDevice, st));
    }
    radfield_shell_kernel<<<(S + 127) / 128, 128, 0, st>>>(K, d_j, d_nubar, en->rf_volume.p, p->time_explosion, p->time_of_simulation, S, en->rf_shell.p,
                                                           p->velocity_gradient ? en->rf_dvdr.p : nullptr);
    const long long total = (long long)S * lpad;
    radfield_jblue_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(K, d_est_t, en->nu_line.p, en->rf_shell.p, L, lpad, S, p->w_epsilon,
                                                                          p->detailed_optical_window, en->rf_jblues_t.p);
    en->launches += 2;
    CK(cudaGetLastError());
    if (t_radiative) CK(cudaMemcpyAsync(t_radiative, en->rf_shell.p, S * sizeof(double), cudaMemcpyDeviceToHost, st));
    if (dilution_factor) CK(cudaMemcpyAsync(dilution_factor, en->rf_shell.p + S, S * sizeof(double), cudaMemcpyDeviceToHost, st));
    if (j_blues && (r = download_line_major(en, en->rf_jblues_t.p, L, lpad, j_blues))) return r;
    CK(cudaStreamSynchronize(st));
    en->rf_valid = true;
    return TB200_OK;
}

// ---- source function (source_function.cuh) ---------------------------------------------------------------------------------
namespace {
// e_dot_u[level, shell]: one warp per (level, shell), source_function.cuh's 32 partial sums + butterfly
__global__ void sf_e_dot_u_kernel(const int *lvl_ptr, const int *lvl_lines, int n_levels, int n_shells, int lpad, const double *tau_t,
                                  const double *edotlu_t, const double *norm /* [S]: 1 / (t_sim V) */, double *e /* [S][n_levels] */) {
    const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= (long long)n_shells * n_levels) return;
    const int s = (int)(w / n_levels), u = (int)(w % n_levels);
    const int a = lvl_ptr[u];
    double v = tbsf::e_dot_u_partial(lane, lvl_lines + a, lvl_ptr[u + 1] - a, norm[s], tau_t + (size_t)s * lpad, edotlu_t + (size_t)s * lpad);
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) v = v + __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) e[w] = v;
}
// one Jacobi sweep of C <- e + Q^T C: one warp per (level, shell); delta[2 s] / delta[2 s + 1] = max |change| / max |C| of the sweep
__global__ void sf_jacobi_kernel(const int *in_ptr, const int *in_rows, const int *in_src, int n_levels, int n_shells, int tpad,
                                 const double *tp_norm_t, const double *e, const double *c_old, double *c_new, unsigned long long *delta) {
    const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= (long long)n_shells * n_levels) return;
    const int s = (int)(w / n_levels), j = (int)(w % n_levels);
    const int a = in_ptr[j];
    double q = tbsf::jacobi_partial(lane, in_rows + a, in_src + a, in_ptr[j + 1] - a, tp_norm_t + (size_t)s * tpad, c_old + (size_t)s * n_levels);
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) q = q + __shfl_xor_sync(0xffffffffu, q, o);
    if (lane == 0) {
        const double v = e[w] + q;
        c_new[w] = v;
        // non-negative doubles order like their bit patterns
        atomicMax(&delta[2 * s], (unsigned long long)__double_as_longlong(fabs(v - c_old[w])));
        atomicMax(&delta[2 * s + 1], (unsigned long long)__double_as_longlong(fabs(v)));
    }
}
__global__ void sf_tables_kernel(const int *em_row, const int *upper, const double *wave, int n_lines, int lpad, int n_shells, int tpad, int n_levels,
                                 const double *tp_norm_t, const double *c /* [S][n_levels] */, const double *tau_t, const double *jblue_est_t,
                                 const double *jnorm /* [S] */, double time_explosion, double *att_t, double *jred_t, double *jblue_t) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)n_shells * lpad) return;
    const int s = (int)(i / lpad), l = (int)(i % lpad);
    double att = 0.0, jb = 0.0, jr = 0.0;
    if (l < n_lines) {
        att = tbsf::att_s_ul(wave[l], tp_norm_t[(size_t)s * tpad + em_row[l]], c[(size_t)s * n_levels + upper[l]], time_explosion);
        jb = jblue_est_t[i] * jnorm[s];
        jr = tbsf::j_red_lu(jb, tau_t[i], att);
    }
    att_t[i] = att; jblue_t[i] = jb; jred_t[i] = jr;
}
}  // namespace

int tb200_solve_source_function(tb200_engine *en, const tb200_source_function_params *p, double *att_S_ul, double *Jred_lu, double *Jblue_lu,
                                double *e_dot_u, int32_t *iterations) {
    if (!en || !p || !p->volume || !p->wavelength_cm || !p->lines_upper_level_idx || !p->lines_lower_level_idx) return fail(TB200_ERR_INVALID, "bad argument");
    if (!en->have_model) return fail(TB200_ERR_NO_MODEL, "tb200_set_model has not been called");
    if (en->opacity_pending) return fail(TB200_ERR_INVALID, "the opacity tables are pending: call tb200_build_opacity first");
    if (en->continuum) return fail(TB200_ERR_INVALID, "the source function of the continuum mode is not built");
    const int mode = en->cfg.line_interaction_type;  // 0 scatter, 1 downbranch, 2 macroatom
    if (mode == 0 || !en->have_macro) return fail(TB200_ERR_INVALID, "the formal-integral source function needs line_interaction_type downbranch or macroatom");
    if (!en->op_tp_norm_t.p) return fail(TB200_ERR_INVALID, "the normalised transition probabilities were not kept: set the option keep_opacity_tables = 1 before tb200_set_model / tb200_build_opacity");
    if ((p->j_blue_estimator == nullptr) != (p->e_dot_lu_estimator == nullptr)) return fail(TB200_ERR_INVALID, "j_blue_estimator and e_dot_lu_estimator must be given together (or both NULL for the resident estimators)");
    if (p->n_levels < 1 || p->n_levels > 2000000000LL) return fail(TB200_ERR_INVALID, "n_levels out of range");
    CK(cudaSetDevice(en->device));
    const int S = en->S, L = en->L, lpad = en->lpad, T = en->T, tpad = en->tpad, NL = (int)p->n_levels;
    int r;
    // ---- host side: level -> lines, destination level -> internal rows, line -> its emission row (row order of the model's tables)
    std::vector<int> ttype((size_t)T), tline((size_t)T);
    CK(cudaMemcpy(ttype.data(), en->ttype.p, (size_t)T * sizeof(int), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(tline.data(), en->tline.p, (size_t)T * sizeof(int), cudaMemcpyDeviceToHost));
    std::vector<int> upper((size_t)L), lvl_ptr((size_t)NL + 1, 0), lvl_lines((size_t)L), em_row((size_t)L, -1);
    for (int l = 0; l < L; l++) {
        const int64_t u = p->lines_upper_level_idx[l], lo = p->lines_lower_level_idx[l];
        if (u < 0 || u >= NL || lo < 0 || lo >= NL) return fail(TB200_ERR_INVALID, "line level index out of range");
        upper[(size_t)l] = (int)u; lvl_ptr[(size_t)u + 1]++;
    }
    for (int u = 0; u < NL; u++) lvl_ptr[(size_t)u + 1] += lvl_ptr[(size_t)u];
    { std::vector<int> fill(lvl_ptr.begin(), lvl_ptr.end() - 1); for (int l = 0; l < L; l++) lvl_lines[(size_t)fill[(size_t)upper[(size_t)l]]++] = l; }
    std::vector<int> in_ptr((size_t)NL + 1, 0), in_rows, in_src;
    size_t n_internal = 0;
    for (int t = 0; t < T; t++) {
        const int l = tline[(size_t)t], ty = ttype[(size_t)t];
        if (l < 0 || l >= L || ty < -1 || ty > 1) return fail(TB200_ERR_INVALID, "source function: transition row outside the bound-bound macro atom (type -1 / 0 / 1)");
        if (ty == -1) {
            if (em_row[(size_t)l] >= 0) return fail(TB200_ERR_INVALID, "source function: a line has two emission rows");
            em_row[(size_t)l] = t;
        } else {
            const int dst = ty == 1 ? upper[(size_t)l] : (int)p->lines_lower_level_idx[l];
            in_ptr[(size_t)dst + 1]++; n_internal++;
        }
    }
    for (int l = 0; l < L; l++) if (em_row[(size_t)l] < 0) return fail(TB200_ERR_INVALID, "source function: a line has no emission row (KeyError in the reference's result.loc[line_idx])");
    for (int u = 0; u < NL; u++) in_ptr[(size_t)u + 1] += in_ptr[(size_t)u];
    in_rows.resize(n_internal ? n_internal : 1); in_src.resize(n_internal ? n_internal : 1);
    { std::vector<int> fill(in_ptr.begin(), in_ptr.end() - 1);
      for (int t = 0; t < T; t++) {  // ascending row order inside every destination list
          const int l = tline[(size_t)t], ty = ttype[(size_t)t];
          if (ty < 0) continue;
          const int src = ty == 1 ? (int)p->lines_lower_level_idx[l] : upper[(size_t)l];
          const int dst = ty == 1 ? upper[(size_t)l] : (int)p->lines_lower_level_idx[l];
          const int k = fill[(size_t)dst]++;
          in_rows[(size_t)k] = t; in_src[(size_t)k] = src;
      } }
    std::vector<double> norm((size_t)2 * S);
    for (int s = 0; s < S; s++) {
        norm[(size_t)s] = tbsf::e_dot_lu_norm(p->time_of_simulation, p->volume[s]);
        norm[(size_t)S + s] = tbsf::j_blue_lu_norm(p->c, p->time_explosion, p->time_of_simulation, p->volume[s]);
    }
    const size_t nls = (size_t)S * NL, lps = (size_t)S * lpad;
    if ((r = en->sf_lvl_ptr.ensure((size_t)NL + 1)) || (r = en->sf_lvl_lines.ensure((size_t)L)) || (r = en->sf_in_ptr.ensure((size_t)NL + 1)) ||
        (r = en->sf_in_rows.ensure(in_rows.size())) || (r = en->sf_in_src.ensure(in_src.size())) || (r = en->sf_em_row.ensure((size_t)L)) ||
        (r = en->sf_upper.ensure((size_t)L)) || (r = en->sf_wave.ensure((size_t)L)) || (r = en->sf_norm.ensure((size_t)2 * S)) ||
        (r = en->sf_e.ensure(nls)) || (r = en->sf_c0.ensure(nls)) || (r = en->sf_c1.ensure(nls)) || (r = en->sf_att_t.ensure(lps)) ||
        (r = en->sf_jred_t.ensure(lps)) || (r = en->sf_jblue_t.ensure(lps)) || (r = en->sf_delta.ensure((size_t)2 * S)))
        return r;
    cudaStream_t st = en->stream;
    CK(cudaMemcpyAsync(en->sf_lvl_ptr.p, lvl_ptr.data(), lvl_ptr.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(en->sf_lvl_lines.p, lvl_lines.data(), lvl_lines.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(en->sf_in_ptr.p, in_ptr.data(), in_ptr.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(en->sf_in_rows.p, in_rows.data(), in_rows.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(en->sf_in_src.p, in_src.data(), in_src.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(en->sf_em_row.p, em_row.data(), em_row.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(en->sf_upper.p, upper.data(), upper.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(en->sf_wave.p, p->wavelength_cm, (size_t)L * sizeof(double), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(en->sf_norm.p, norm.data(), norm.size() * sizeof(double), cudaMemcpyHostToDevice, st));
    const double *d_jblue_t = en->est.p + en->off_jblue, *d_edotlu_t = en->est.p + en->off_edotlu;
    if (p->j_blue_estimator) {
        if ((r = upload_strided_table(en, p->j_blue_estimator, L, S, S, 1, lpad, en->sf_in_t))) return r;
        if ((r = upload_strided_table(en, p->e_dot_lu_estimator, L, S, S, 1, lpad, en->sf_in2_t))) return r;
        d_jblue_t = en->sf_in_t.p; d_edotlu_t = en->sf_in2_t.p;
    }
    // ---- e_dot_u, then (macroatom) the fixed point C = e + Q^T C per shell
    const unsigned g_lvl = (unsigned)((nls * 32 + 127) / 128);  // a warp per (level, shell)
    sf_e_dot_u_kernel<<<g_lvl, 128, 0, st>>>(en->sf_lvl_ptr.p, en->sf_lvl_lines.p, NL, S, lpad, en->tau_t.p, d_edotlu_t, en->sf_norm.p, en->sf_e.p);
    en->launches++;
    CK(cudaGetLastError());
    const double *c_final = en->sf_e.p;
    int it = 0;
    if (mode == 2) {
        const int max_it = p->max_iterations > 0 ? p->max_iterations : 100000;
        const double tol = p->tolerance > 0.0 ? p->tolerance : 1e-15;
        CK(cudaMemcpyAsync(en->sf_c0.p, en->sf_e.p, nls * sizeof(double), cudaMemcpyDeviceToDevice, st));
        double *c_old = en->sf_c0.p, *c_new = en->sf_c1.p;
        std::vector<double> delta((size_t)2 * S);
        bool converged = false;
        while (!converged && it < max_it) {
            for (int k = 0; k < 8 && it < max_it; k++, it++) {  // the last sweep of a batch is the one that is judged
                CK(cudaMemsetAsync(en->sf_delta.p, 0, (size_t)2 * S * sizeof(double), st));
                sf_jacobi_kernel<<<g_lvl, 128, 0, st>>>(en->sf_in_ptr.p, en->sf_in_rows.p, en->sf_in_src.p, NL, S, tpad, en->op_tp_norm_t.p, en->sf_e.p,
                                                        c_old, c_new, reinterpret_cast<unsigned long long *>(en->sf_delta.p));
                en->launches++;
                std::swap(c_old, c_new);
            }
            CK(cudaGetLastError());
            CK(cudaMemcpyAsync(delta.data(), en->sf_delta.p, delta.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            converged = true;
            for (int s = 0; s < S; s++) {
                const double d = delta[(size_t)2 * s], m = delta[(size_t)2 * s + 1];
                if (!(d <= tol * m)) converged = false;  // (NaN / inf never converge)
            }
        }
        if (!converged) return fail(TB200_ERR_INVALID, "source function: the macro-atom system C = e + Q^T C did not converge (singular I - Q, non-finite input, or max_iterations too small)");
        c_final = c_old;
    }
    if (iterations) *iterations = it;
    // ---- att_S_ul, Jblue_lu, Jred_lu
    sf_tables_kernel<<<(unsigned)((lps + 255) / 256), 256, 0, st>>>(en->sf_em_row.p, en->sf_upper.p, en->sf_wave.p, L, lpad, S, tpad, NL, en->op_tp_norm_t.p,
                                                                      c_final, en->tau_t.p, d_jblue_t, en->sf_norm.p + S, p->time_explosion,
                                                                      en->sf_att_t.p, en->sf_jred_t.p, en->sf_jblue_t.p);
    en->launches++;
    CK(cudaGetLastError());
    double *outs[3] = {att_S_ul, Jred_lu, Jblue_lu};
    const double *srcs[3] = {en->sf_att_t.p, en->sf_jred_t.p, en->sf_jblue_t.p};
    for (int k = 0; k < 3; k++) {
        if (!outs[k]) continue;
        if ((r = download_line_major(en, srcs[k], L, lpad, outs[k]))) return r;
        CK(cudaStreamSynchronize(st));  // staging is reused
    }
    if (e_dot_u) {  // [n_levels, S] C-order on the host; on the device it lies [S][n_levels]
        std::vector<double> tmp(nls);
        CK(cudaMemcpyAsync(tmp.data(), c_final, nls * sizeof(double), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        for (int s = 0; s < S; s++) for (int u = 0; u < NL; u++) e_dot_u[(size_t)u * S + s] = tmp[(size_t)s * NL + u];
    }
    CK(cudaStreamSynchronize(st));
    en->sf_valid = true;
    return TB200_OK;
}

// ---- formal integral (formal_integral.cuh) --------------------------------------------------------------------------------
namespace {
constexpr int FI_WARPS = 4;  // warps per CTA of the ray kernel; a warp = 32 neighbouring impact parameters of one frequency

__global__ void fi_cells_kernel(tbfi::Tables T, const tbfi::ShellWeights *w, int n_shells, tbfi::Cell *cells) {
    const long long row = tbfi::row_cells(T.n_lines);
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= row * n_shells) return;
    cells[i] = tbfi::build_cell(T, w, n_shells, (int)(i / row), (int)(i % row));
}

// One sweep over the line list per warp: at every step all lanes that are inside their ray's window pass the SAME line, so the
// line frequency is one uniform load and the cells of a step lie in the few shells the 32 neighbouring rays are in.
__global__ void __launch_bounds__(FI_WARPS * 32) fi_rays_kernel(tbfi::Shells g, const double *__restrict__ nu_line, int n_lines,
                                                                const tbfi::Cell *__restrict__ cells, const double *__restrict__ freq,
                                                                int n_freq, int n_p, int n_blocks, double inner_temperature,
                                                                double *__restrict__ I_out) {
    const long long item = (long long)blockIdx.x * FI_WARPS + (threadIdx.x >> 5);
    if (item >= (long long)n_freq * n_blocks) return;  // whole warps leave together
    const int lane = threadIdx.x & 31;
    const int f = (int)(item / n_blocks), b = (int)(item % n_blocks);
    const int p_idx = 1 + b * 32 + lane;
    const long long row = tbfi::row_cells(n_lines);
    tbfi::Ray r;
    if (p_idx < n_p) r.init(g, nu_line, n_lines, freq[f], p_idx, n_p, inner_temperature);
    else { r.done = true; r.I = 0.0; r.line_idx = n_lines; }
    for (;;) {
        // the next line any unfinished lane of the warp will pass (gaps between the lanes' windows are jumped over)
        const int l = __reduce_min_sync(0xffffffffu, r.done ? 0x7fffffff : r.line_idx);
        if (l == 0x7fffffff) break;
        if (l >= n_lines) {  // behind the list only shell boundaries are left
            if (!r.done) r.finish(g, cells, row);
            break;
        }
        const double nl = nu_line[l];
        if (!r.done && r.line_idx == l) r.pass_line(g, cells, row, nl);
    }
    if (p_idx < n_p) I_out[(size_t)f * n_p + p_idx] = r.I;
    if (b == 0 && lane == 0) I_out[(size_t)f * n_p] = 0.0;  // impact parameter 0 is never integrated (formal_integral_numba.py:265, :466)
}

__global__ void __launch_bounds__(tbfi::TRAPZ_LANES) fi_trapz_kernel(const double *I, int n_p, double d, double *lum) {
    __shared__ double part[tbfi::TRAPZ_LANES];
    const int t = threadIdx.x;
    part[t] = tbfi::trapz_partial(t, I + (size_t)blockIdx.x * n_p, n_p, d);
    __syncthreads();
    for (int o = tbfi::TRAPZ_LANES / 2; o >= 1; o >>= 1) {
        if (t < o) part[t] = part[t] + part[t + o];
        __syncthreads();
    }
    if (t == 0) lum[blockIdx.x] = tbfi::luminosity_density(part[0]);
}
}  // namespace

int tb200_formal_integral(tb200_engine *en, const tb200_formal_integral_params *p, const double *frequencies, int64_t n_frequencies,
                          double *luminosity_densities, double *intensities_nu_p) {
    if (!en || !p || !frequencies || !luminosity_densities) return fail(TB200_ERR_INVALID, "bad argument");
    if (!en->have_model) return fail(TB200_ERR_NO_MODEL, "tb200_set_model has not been called");
    if (en->opacity_pending) return fail(TB200_ERR_INVALID, "the opacity tables are pending: call tb200_build_opacity first");
    if (en->continuum) return fail(TB200_ERR_INVALID, "The FormalIntegrator currently does not work for continuum interactions.");
    if (en->cfg.line_interaction_type == 0) return fail(TB200_ERR_INVALID, "The FormalIntegrator currently only works for line_interaction_type downbranch and macroatom");
    const bool host_tables = p->att_S_ul || p->Jred_lu || p->Jblue_lu;
    if (host_tables && !(p->att_S_ul && p->Jred_lu && p->Jblue_lu)) return fail(TB200_ERR_INVALID, "att_S_ul, Jred_lu and Jblue_lu must be given together (or all NULL for the resident tables)");
    if (!host_tables && !en->sf_valid) return fail(TB200_ERR_INVALID, "no source function is resident for this model: call tb200_solve_source_function first (or pass the three tables)");
    if (p->n_impact_parameters < 2) return fail(TB200_ERR_INVALID, "n_impact_parameters must be at least 2");
    if (n_frequencies < 0 || n_frequencies > 2000000000LL) return fail(TB200_ERR_INVALID, "n_frequencies out of range");
    if (p->interpolate_shells == 1) return fail(TB200_ERR_INVALID, "interpolate_shells = 1 leaves no shell");
    CK(cudaSetDevice(en->device));
    const int S = en->S, L = en->L, lpad = en->lpad, P = p->n_impact_parameters;
    if (S < 2) return fail(TB200_ERR_INVALID, "the interpolation over the shell mid-points needs at least two shells (scipy interp1d refuses one)");
    cudaStream_t st = en->stream;
    int r;
    // ---- host side: the integrator's shells and their interpolation weights (formal_integral_solver.py:208-232, :345-352)
    std::vector<double> r_in((size_t)S), r_out((size_t)S), ne((size_t)S);
    CK(cudaMemcpyAsync(r_in.data(), en->r_inner.p, S * sizeof(double), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(r_out.data(), en->r_outer.p, S * sizeof(double), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(ne.data(), en->n_e.p, S * sizeof(double), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (p->electron_densities) for (int s = 0; s < S; s++) ne[(size_t)s] = p->electron_densities[s];
    int n_radii = p->interpolate_shells;
    if (n_radii == 0) n_radii = 2 * S > 80 ? 2 * S : 80;
    const int S2 = n_radii > 0 ? n_radii - 1 : S;
    std::vector<double> shells((size_t)3 * S2), mid((size_t)S);
    for (int s = 0; s < S; s++) mid[(size_t)s] = (r_in[(size_t)s] + r_out[(size_t)s]) / 2.0;
    for (int s = 1; s < S; s++)
        if (!(mid[(size_t)s] > mid[(size_t)s - 1])) return fail(TB200_ERR_INVALID, "shell radii must increase");
    for (int s = 0; s < S2; s++) {
        shells[(size_t)s] = n_radii > 0 ? tbfi::linspace_at(r_in[0], r_out[(size_t)S - 1], n_radii, s) : r_in[(size_t)s];
        shells[(size_t)S2 + s] = n_radii > 0 ? tbfi::linspace_at(r_in[0], r_out[(size_t)S - 1], n_radii, s + 1) : r_out[(size_t)s];
    }
    const double sigma = p->sigma_thomson != 0.0 ? p->sigma_thomson : 6.652458734e-25;
    std::vector<tbfi::ShellWeights> w((size_t)S2);
    for (int s = 0; s < S2; s++) {
        w[(size_t)s] = tbfi::shell_weights(mid.data(), S, (shells[(size_t)s] + shells[(size_t)S2 + s]) / 2.0);
        shells[(size_t)2 * S2 + s] = ne[(size_t)w[(size_t)s].nearest] * sigma;  // electron_densities_interpolated * SIGMA_THOMSON
    }
    const long long row = tbfi::row_cells(L);
    const size_t n_cells = (size_t)row * S2;
    const size_t w_doubles = (sizeof(tbfi::ShellWeights) * (size_t)S2 + sizeof(double) - 1) / sizeof(double);
    const size_t nf = (size_t)(n_frequencies > 0 ? n_frequencies : 1);
    if ((r = en->fi_cells.ensure(n_cells * 4)) || (r = en->fi_shells.ensure((size_t)3 * S2)) || (r = en->fi_weights.ensure(w_doubles)) ||
        (r = en->fi_freq.ensure(nf)) || (r = en->fi_I.ensure(nf * P)) || (r = en->fi_L.ensure(nf)))
        return r;
    CK(cudaMemcpyAsync(en->fi_shells.p, shells.data(), shells.size() * sizeof(double), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(en->fi_weights.p, w.data(), w.size() * sizeof(tbfi::ShellWeights), cudaMemcpyHostToDevice, st));
    tbfi::Tables T{en->tau_t.p, en->sf_att_t.p, en->sf_jred_t.p, en->sf_jblue_t.p, L, lpad};
    if (host_tables) {
        if ((r = upload_strided_table(en, p->att_S_ul, L, S, S, 1, lpad, en->fi_att_t))) return r;
        if ((r = upload_strided_table(en, p->Jred_lu, L, S, S, 1, lpad, en->fi_jred_t))) return r;
        if ((r = upload_strided_table(en, p->Jblue_lu, L, S, S, 1, lpad, en->fi_jblue_t))) return r;
        T.att_t = en->fi_att_t.p; T.jred_t = en->fi_jred_t.p; T.jblue_t = en->fi_jblue_t.p;
    }
    Event e0, e1, e2;
    if (cudaEventCreate(&e0.h) != cudaSuccess || cudaEventCreate(&e1.h) != cudaSuccess || cudaEventCreate(&e2.h) != cudaSuccess)
        return fail(TB200_ERR_CUDA, "cudaEventCreate failed");
    tbfi::Cell *cells = reinterpret_cast<tbfi::Cell *>(en->fi_cells.p);
    cudaEventRecord(e0, st);
    fi_cells_kernel<<<(unsigned)((n_cells + 255) / 256), 256, 0, st>>>(T, reinterpret_cast<const tbfi::ShellWeights *>(en->fi_weights.p), S2, cells);
    en->launches++;
    cudaEventRecord(e1, st);
    if (n_frequencies > 0) {
        cudaError_t cf = cudaMemcpyAsync(en->fi_freq.p, frequencies, (size_t)n_frequencies * sizeof(double), cudaMemcpyHostToDevice, st);
        if (cf != cudaSuccess) return fail(TB200_ERR_CUDA, std::string("cudaMemcpyAsync(frequencies): ") + cudaGetErrorString(cf));
        const int n_blocks = (P - 1 + 31) / 32;  // impact parameters 1 ... P - 1
        const long long items = (long long)n_frequencies * n_blocks;
        if ((items + FI_WARPS - 1) / FI_WARPS > 2147483647LL) return fail(TB200_ERR_INVALID, "n_frequencies x n_impact_parameters too large for one launch");
        tbfi::Shells g{en->fi_shells.p, en->fi_shells.p + S2, en->fi_shells.p + 2 * (size_t)S2, S2, 1 / en->t_exp, en->t_exp / tbfi::C_INV};
        fi_rays_kernel<<<(unsigned)((items + FI_WARPS - 1) / FI_WARPS), FI_WARPS * 32, 0, st>>>(g, en->nu_line.p, L, cells, en->fi_freq.p, (int)n_frequencies, P,
                                                                                              n_blocks, p->inner_temperature, en->fi_I.p);
        fi_trapz_kernel<<<(unsigned)n_frequencies, tbfi::TRAPZ_LANES, 0, st>>>(en->fi_I.p, P, shells[(size_t)2 * S2 - 1] / (double)P, en->fi_L.p);
        en->launches += 2;
    }
    cudaEventRecord(e2, st);
    cudaError_t ce = cudaGetLastError();
    if (ce != cudaSuccess) return fail(TB200_ERR_CUDA, cudaGetErrorString(ce));
    if (n_frequencies > 0) {
        cudaMemcpyAsync(luminosity_densities, en->fi_L.p, (size_t)n_frequencies * sizeof(double), cudaMemcpyDeviceToHost, st);
        if (intensities_nu_p) cudaMemcpyAsync(intensities_nu_p, en->fi_I.p, (size_t)n_frequencies * P * sizeof(double), cudaMemcpyDeviceToHost, st);
    }
    ce = cudaStreamSynchronize(st);
    if (ce != cudaSuccess) return fail(TB200_ERR_CUDA, cudaGetErrorString(ce));
    float a = 0.0f, b = 0.0f;
    cudaEventElapsedTime(&a, e0, e1); cudaEventElapsedTime(&b, e1, e2);
    en->fi_cells_ms = a; en->fi_rays_ms = b;
    return TB200_OK;
}

int tb200_formal_integral_ms(tb200_engine *en, double *interpolation_ms, double *integral_ms) {
    if (!en || !interpolation_ms || !integral_ms) return fail(TB200_ERR_INVALID, "bad argument");
    *interpolation_ms = en->fi_cells_ms; *integral_ms = en->fi_rays_ms;
    return TB200_OK;
}

// ---- opacity build (opacity_build.cuh) ----------------------------------------------------------------------------------
namespace {
// The mode's tau formula, chosen at compile time by the type of `scale`: the homologous mode's time_explosion, or the
// nonhomologous mode's velocity_gradient [S] (the caller's array).  One body, one kernel per mode.
extern "C++" {
__device__ __forceinline__ double line_tau(const tbo::Constants &K, double wfl, double time_explosion, int, double stim, double n_lower) {
    return tbo::tau_sobolev(K, wfl, time_explosion, stim, n_lower);
}
__device__ __forceinline__ double line_tau(const tbo::Constants &K, double wfl, const double *velocity_gradient, int s, double stim, double n_lower) {
    return tbo::tau_sobolev_nonhomologous(K, wfl, velocity_gradient[s], stim, n_lower);
}
template <typename Scale>
__device__ __forceinline__ void opacity_line_cells(const tbo::Constants &K, const double *lnd, int n_shells, const int *lower, const int *upper,
                                                   const double *g, const unsigned char *meta, const unsigned char *nlte, const double *wfl,
                                                   Scale scale, int n_lines, int lpad, double *tau_t, double *beta_t, double *stim_t, int *error) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)n_shells * lpad) return;
    const int s = (int)(i / lpad), l = (int)(i % lpad);
    double tau = 0.0, beta = 0.0, stim = 0.0;
    if (l < n_lines) {
        const int lo = lower[l], up = upper[l];
        const double n_lower = lnd[(size_t)lo * n_shells + s], n_upper = lnd[(size_t)up * n_shells + s];
        stim = tbo::stimulated_emission_factor(n_lower, n_upper, g[lo], g[up], meta[up] != 0, nlte ? nlte[l] != 0 : false);
        tau = line_tau(K, wfl[l], scale, s, stim, n_lower);
        if (isnan(tau) || isinf(tau)) atomicMax(error, tb::ERR_OPACITY);  // "Some tau_sobolevs are nan, inf, -inf" (tau_sobolev.py:63-67)
        beta = tbo::beta_sobolev(tau);
    }
    tau_t[i] = tau; beta_t[i] = beta; stim_t[i] = stim;
}
}  // extern "C++"
__global__ void opacity_line_kernel(tbo::Constants K, const double *lnd, int n_shells, const int *lower, const int *upper, const double *g,
                                    const unsigned char *meta, const unsigned char *nlte, const double *wfl, double time_explosion, int n_lines,
                                    int lpad, double *tau_t, double *beta_t, double *stim_t, int *error) {
    opacity_line_cells(K, lnd, n_shells, lower, upper, g, meta, nlte, wfl, time_explosion, n_lines, lpad, tau_t, beta_t, stim_t, error);
}
__global__ void opacity_line_nonhomologous_kernel(tbo::Constants K, const double *lnd, int n_shells, const int *lower, const int *upper,
                                                  const double *g, const unsigned char *meta, const unsigned char *nlte, const double *wfl,
                                                  const double *velocity_gradient, int n_lines, int lpad, double *tau_t, double *beta_t,
                                                  double *stim_t, int *error) {
    opacity_line_cells(K, lnd, n_shells, lower, upper, g, meta, nlte, wfl, velocity_gradient, n_lines, lpad, tau_t, beta_t, stim_t, error);
}
__global__ void opacity_row_kernel(tbo::Constants K, const int *ttype, const int *tline, const double *beta_t, const double *stim_t,
                                   const double *jblues_t, const double *nu, const double *f_ul, const double *f_lu, const double *e_lo,
                                   const double *e_up, int n_rows, int tpad, int lpad, int n_shells, double *tp_t) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)n_shells * tpad) return;
    const int s = (int)(i / tpad), t = (int)(i % tpad);
    double p = 0.0;
    if (t < n_rows) {
        const int l = tline[t], type = ttype[t];
        const size_t c = (size_t)s * lpad + l;
        p = tbo::raw_probability(K, type, beta_t[c], nu[l], f_ul[l], f_lu[l], e_lo[l], e_up[l], stim_t[c], type == 1 ? jblues_t[c] : 0.0);
    }
    tp_t[i] = p;
}
// normalize_transition_probabilities: divide every row by the sum of its source block; 0 / 0 -> 0
__global__ void opacity_normalize_kernel(double *tp_t, const int *block_edge, int n_blocks, int n_shells, int tpad) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)n_blocks * n_shells) return;
    const int shell = (int)(i / n_blocks), block = (int)(i % n_blocks);
    double *row = tp_t + (size_t)shell * tpad;
    double sum = 0.0;
    for (int t = block_edge[block]; t < block_edge[block + 1]; t++) sum += row[t];
    for (int t = block_edge[block]; t < block_edge[block + 1]; t++) {
        const double q = row[t] / sum;
        row[t] = isnan(q) ? 0.0 : q;
    }
}
// The continuum mode's rows (continuum_macro_build.cuh), one thread per (shell, row) over [S][tpad]: line rows as in
// opacity_row_kernel, continuum rows from the row map and the per-iteration tables.
__global__ void continuum_row_kernel(tbo::Constants K, const int *ttype, const int *tline, const long long *ct_off, const double *ct_energy,
                                     const double *ct_tab, const double *ct_shell, const double *beta_t, const double *stim_t,
                                     const double *jblues_t, const double *nu, const double *f_ul, const double *f_lu, const double *e_lo,
                                     const double *e_up, int n_rows, int tpad, int lpad, int n_shells, double *p_t) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)n_shells * tpad) return;
    const int s = (int)(i / tpad), t = (int)(i % tpad);
    double p = 0.0;
    if (t < n_rows) {
        const int type = ttype[t];
        if (tbcm::is_line_row(type)) {
            const int l = tline[t];
            const size_t c = (size_t)s * lpad + l;
            p = tbo::raw_probability(K, type, beta_t[c], nu[l], f_ul[l], f_lu[l], e_lo[l], e_up[l], stim_t[c], type == 1 ? jblues_t[c] : 0.0);
        } else {
            const long long off = ct_off[t];
            p = tbcm::continuum_probability(type, off >= 0 ? ct_tab[off + s] : 0.0, ct_shell[s], ct_energy[t],
                                            ct_shell[(size_t)tbcm::cooling_rate(type) * n_shells + s]);
        }
    }
    p_t[i] = p;
}
// normalize_transition_probabilities of the continuum mode: one thread per (shell, source block)
__global__ void continuum_normalize_kernel(double *p_t, const int *block_edge, int n_blocks, int n_shells, int tpad) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)n_blocks * n_shells) return;
    const int shell = (int)(i / n_blocks), block = (int)(i % n_blocks);
    tbcm::normalize_block(p_t + (size_t)shell * tpad, block_edge[block], block_edge[block + 1]);
}
}  // namespace

// The continuum row map of tb200_set_atomic_data, checked against the model's rows before anything is allocated.
static int set_continuum_rows(tb200_engine *en, const tb200_continuum_rows *cr) {
    if (!en->continuum) return fail(TB200_ERR_INVALID, "atomic data: continuum_rows is the continuum mode's row map; this model has no continuum");
    if (cr->n_transitions != en->T)
        return fail(TB200_ERR_INVALID, "continuum_rows: n_transitions " + std::to_string(cr->n_transitions) + " differs from the model's " + std::to_string(en->T));
    if (!cr->rate_key || !cr->energy) return fail(TB200_ERR_INVALID, "continuum_rows: rate_key or energy is NULL");
    const int T = en->T, S = en->S;
    long long height[tbcm::N_TABLES];
    for (int k = 0; k < tbcm::N_TABLES; k++) {
        height[k] = k < 6 ? cr->n_rate_rows[k] : cr->n_cooling_rows[k - 6];
        if (height[k] < 0) return fail(TB200_ERR_INVALID, "continuum_rows: negative table height");
    }
    std::vector<int> tt((size_t)(T > 0 ? T : 1));
    CK(cudaMemcpy(tt.data(), en->ttype.p, (size_t)T * sizeof(int), cudaMemcpyDeviceToHost));
    long long base[tbcm::N_TABLES + 1];
    base[0] = 0;
    for (int k = 0; k < tbcm::N_TABLES; k++) base[k + 1] = base[k] + height[k];
    std::vector<long long> off((size_t)(T > 0 ? T : 1), -1);
    for (int t = 0; t < T; t++) {
        const int tab = tbcm::row_table(tt[(size_t)t]);
        if (tab == tbcm::BAD_TYPE)
            return fail(TB200_ERR_INVALID, "continuum_rows: row " + std::to_string(t) + " has transition_type " + std::to_string(tt[(size_t)t]) +
                                               ", which the continuum macro atom does not build");
        if (tab == tbcm::NO_TABLE) continue;
        const long long key = cr->rate_key[t];
        if (key < 0 || key >= height[tab])
            return fail(TB200_ERR_INVALID, "continuum_rows: rate_key " + std::to_string(key) + " of row " + std::to_string(t) + " (type " +
                                               std::to_string(tt[(size_t)t]) + ") is outside its table of " + std::to_string(height[tab]) + " rows");
        off[(size_t)t] = (base[tab] + key) * S;
    }
    int r;
    if ((r = en->ct_off.ensure(off.size())) || (r = en->ct_energy.ensure(off.size()))) return r;
    CK(cudaMemcpy(en->ct_off.p, off.data(), off.size() * sizeof(long long), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(en->ct_energy.p, cr->energy, (size_t)T * sizeof(double), cudaMemcpyHostToDevice));
    for (int k = 0; k <= tbcm::N_TABLES; k++) en->ct_base[k] = base[k];
    en->ct_T = T;
    return TB200_OK;
}

// The per-iteration continuum tables of tb200_build_opacity into ct_tab / ct_shell (checked by the caller).
static int upload_continuum_rates(tb200_engine *en, const tb200_continuum_rates *cr) {
    const int S = en->S;
    int r;
    if ((r = en->ct_tab.ensure((size_t)std::max(en->ct_base[tbcm::N_TABLES], 1LL) * S)) || (r = en->ct_shell.ensure((size_t)tbcm::SHELL_ARRAYS * S))) return r;
    for (int k = 0; k < tbcm::N_TABLES; k++) {
        const long long rows = en->ct_base[k + 1] - en->ct_base[k];
        const double *src = k < 6 ? cr->rate[k] : cr->cooling[k - 6];
        if (rows > 0) CK(cudaMemcpyAsync(en->ct_tab.p + en->ct_base[k] * S, src, (size_t)rows * S * sizeof(double), cudaMemcpyHostToDevice, en->stream));
    }
    const double *shell[tbcm::SHELL_ARRAYS] = {cr->electron_densities, cr->ff_cool_rate, cr->fb_cool_rate, cr->coll_exc_cool_rate, cr->coll_ion_cool_rate};
    for (int k = 0; k < tbcm::SHELL_ARRAYS; k++)
        CK(cudaMemcpyAsync(en->ct_shell.p + (size_t)k * S, shell[k], (size_t)S * sizeof(double), cudaMemcpyHostToDevice, en->stream));
    return TB200_OK;
}

int tb200_set_atomic_data(tb200_engine *en, const tb200_atomic_data *a) {
    if (!en || !a) return fail(TB200_ERR_INVALID, "bad argument");
    if (!en->have_model) return fail(TB200_ERR_NO_MODEL, "tb200_set_model has not been called (the atomic data refer to its line list)");
    if (a->n_lines != en->L) return fail(TB200_ERR_INVALID, "atomic data: n_lines differs from the model's line list");
    if (a->n_levels < 1 || !a->lines_lower_level_index || !a->lines_upper_level_index || !a->g || !a->metastability || !a->wavelength_f_lu ||
        !a->f_lu || !a->f_ul || !a->energy_lower || !a->energy_upper)
        return fail(TB200_ERR_INVALID, "atomic data: missing array");
    if (en->continuum && !a->continuum_rows)
        return fail(TB200_ERR_INVALID, "atomic data: the continuum mode needs continuum_rows (the row map of its macro atom)");
    CK(cudaSetDevice(en->device));
    const int L = en->L;
    for (int64_t l = 0; l < L; l++)
        if (a->lines_lower_level_index[l] < 0 || a->lines_lower_level_index[l] >= a->n_levels || a->lines_upper_level_index[l] < 0 ||
            a->lines_upper_level_index[l] >= a->n_levels)
            return fail(TB200_ERR_INVALID, "atomic data: level index out of range");
    int r;
    if (a->continuum_rows && (r = set_continuum_rows(en, a->continuum_rows))) return r;  // a refused map keeps the previous one
    en->n_levels = a->n_levels;
    if ((r = upload_i64_as_i32(en, a->lines_lower_level_index, L, en->at_lower)) || (r = upload_i64_as_i32(en, a->lines_upper_level_index, L, en->at_upper))) return r;
    if ((r = en->at_g.ensure(a->n_levels)) || (r = en->at_meta.ensure(a->n_levels)) || (r = en->at_nlte.ensure(L)) || (r = en->at_wfl.ensure(L)) ||
        (r = en->at_flu.ensure(L)) || (r = en->at_ful.ensure(L)) || (r = en->at_elo.ensure(L)) || (r = en->at_eup.ensure(L)))
        return r;
    cudaStream_t st = en->stream;
    CK(cudaMemcpyAsync(en->at_g.p, a->g, a->n_levels * sizeof(double), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(en->at_meta.p, a->metastability, a->n_levels, cudaMemcpyHostToDevice, st));
    if (a->nlte_line) CK(cudaMemcpyAsync(en->at_nlte.p, a->nlte_line, L, cudaMemcpyHostToDevice, st));
    else CK(cudaMemsetAsync(en->at_nlte.p, 0, L, st));
    const double *src[5] = {a->wavelength_f_lu, a->f_lu, a->f_ul, a->energy_lower, a->energy_upper};
    double *dst[5] = {en->at_wfl.p, en->at_flu.p, en->at_ful.p, en->at_elo.p, en->at_eup.p};
    for (int k = 0; k < 5; k++) CK(cudaMemcpyAsync(dst[k], src[k], L * sizeof(double), cudaMemcpyHostToDevice, st));
    CK(cudaStreamSynchronize(st));
    en->op_const.sobolev_coefficient = a->sobolev_coefficient; en->op_const.c_einstein = a->c_einstein; en->op_const.c = a->c; en->op_const.h = a->h;
    en->have_atomic = true;
    return TB200_OK;
}

// Waits for tb200_build_opacity's kernels and reports a non-finite tau_sobolev they flagged in the error word.
static int wait_opacity_build(tb200_engine *en) {
    CK(cudaStreamSynchronize(en->stream));
    int err = 0;
    CK(cudaMemcpy(&err, en->error.p, sizeof(int), cudaMemcpyDeviceToHost));
    if (err == tb::ERR_OPACITY) return fail(TB200_ERR_INVALID, "Some tau_sobolevs are nan, inf, -inf in tau_sobolevs. Something went wrong!");
    return TB200_OK;
}

int tb200_build_opacity(tb200_engine *en, const tb200_plasma_state *p) {
    // continuum rates with beta / stim: the line rows read the caller's tables, tau is the model's (not rebuilt)
    const bool host_lines = p && p->continuum && (p->continuum->beta_sobolev || p->continuum->stimulated_emission_factor);
    if (!en || !p) return fail(TB200_ERR_INVALID, "bad argument");
    if (!en->have_model) return fail(TB200_ERR_NO_MODEL, "tb200_set_model has not been called");
    if (!en->have_atomic) return fail(TB200_ERR_NO_MODEL, "tb200_set_atomic_data has not been called");
    // level_number_density NULL: the populations tb200_solve_plasma left in op_lnd
    const bool resident_lnd = !p->level_number_density && !host_lines;
    if (resident_lnd && !en->pl_valid)
        return fail(TB200_ERR_INVALID, "level_number_density is NULL and no tb200_solve_plasma since tb200_set_model has left populations in HBM");
    if (!en->continuum && p->continuum) return fail(TB200_ERR_INVALID, "continuum: the continuum mode's rates; this model has no continuum");
    if (en->continuum) {
        const tb200_continuum_rates *cr = p->continuum;
        if (!cr) return fail(TB200_ERR_INVALID, "the continuum mode's macro atom needs continuum (its rates of this iteration)");
        if (host_lines) {
            if (!cr->beta_sobolev || !cr->stimulated_emission_factor)
                return fail(TB200_ERR_INVALID, "continuum: beta_sobolev and stimulated_emission_factor go together");
            if (p->level_number_density)
                return fail(TB200_ERR_INVALID, "continuum: with beta_sobolev given, level_number_density must be NULL (tau is not rebuilt)");
            if (en->opacity_pending)
                return fail(TB200_ERR_INVALID, "continuum: beta_sobolev given, but the model has no tau_sobolev (tb200_set_model got NULL)");
        }
        if (en->ct_T != en->T) return fail(TB200_ERR_NO_MODEL, "the continuum mode needs tb200_set_atomic_data with continuum_rows for this model");
        if (!cr->electron_densities || !cr->ff_cool_rate || !cr->fb_cool_rate || !cr->coll_exc_cool_rate || !cr->coll_ion_cool_rate)
            return fail(TB200_ERR_INVALID, "continuum: a per-shell array is NULL");
        for (int k = 0; k < tbcm::N_TABLES; k++)
            if (en->ct_base[k + 1] > en->ct_base[k] && !(k < 6 ? cr->rate[k] : cr->cooling[k - 6]))
                return fail(TB200_ERR_INVALID, std::string("continuum: ") + (k < 6 ? "rate[" : "cooling[") + std::to_string(k < 6 ? k : k - 6) +
                                                   "] is NULL but the row map reads it");
    }
    const bool need_jblues = en->have_macro && en->cfg.line_interaction_type == 2;
    if (need_jblues && !p->j_blues && !en->rf_valid)
        return fail(TB200_ERR_INVALID, "j_blues is NULL and tb200_solve_radiation_field has not left a table in HBM");
    // a nonhomologous model carries no usable time_explosion: its tau divides by the velocity gradient instead
    if (en->nonhomologous && !p->velocity_gradient)
        return fail(TB200_ERR_INVALID, "the nonhomologous mode's tau_sobolev divides by velocity_gradient: pass velocity_gradient");
    if (!en->nonhomologous && p->velocity_gradient)
        return fail(TB200_ERR_INVALID, "velocity_gradient is the nonhomologous mode's tau_sobolev; this model is homologous");
    CK(cudaSetDevice(en->device));
    const int S = en->S, L = en->L, lpad = en->lpad;
    int r;
    cudaStream_t st = en->stream;
    CK(cudaMemsetAsync(en->error.p, 0, sizeof(int), st));
    if (host_lines) {
        if ((r = upload_strided_table(en, p->continuum->beta_sobolev, L, S, S, 1, lpad, en->op_beta_t)) ||
            (r = upload_strided_table(en, p->continuum->stimulated_emission_factor, L, S, S, 1, lpad, en->op_stim_t)))
            return r;
    } else {
        if ((r = en->op_lnd.ensure((size_t)en->n_levels * S)) || (r = en->op_beta_t.ensure((size_t)S * lpad)) || (r = en->op_stim_t.ensure((size_t)S * lpad))) return r;
        if (!resident_lnd) {
            en->pl_valid = false;  // op_lnd now holds the caller's populations
            CK(cudaMemcpyAsync(en->op_lnd.p, p->level_number_density, (size_t)en->n_levels * S * sizeof(double), cudaMemcpyHostToDevice, st));
        }
        const long long total = (long long)S * lpad;
        const unsigned grid = (unsigned)((total + 255) / 256);
        if (en->nonhomologous) {
            if ((r = en->op_dvdr.ensure(S))) return r;
            CK(cudaMemcpyAsync(en->op_dvdr.p, p->velocity_gradient, S * sizeof(double), cudaMemcpyHostToDevice, st));
            opacity_line_nonhomologous_kernel<<<grid, 256, 0, st>>>(en->op_const, en->op_lnd.p, S, en->at_lower.p, en->at_upper.p, en->at_g.p,
                en->at_meta.p, en->at_nlte.p, en->at_wfl.p, en->op_dvdr.p, L, lpad, en->tau_t.p, en->op_beta_t.p, en->op_stim_t.p, en->error.p);
        } else {
            opacity_line_kernel<<<grid, 256, 0, st>>>(en->op_const, en->op_lnd.p, S, en->at_lower.p, en->at_upper.p, en->at_g.p, en->at_meta.p,
                en->at_nlte.p, en->at_wfl.p, p->time_explosion, L, lpad, en->tau_t.p, en->op_beta_t.p, en->op_stim_t.p, en->error.p);
        }
        en->launches++;
        CK(cudaGetLastError());
    }
    if (en->have_macro) {
        const double *jb = en->rf_jblues_t.p;
        if (need_jblues && p->j_blues) {
            if ((r = upload_strided_table(en, p->j_blues, L, S, S, 1, lpad, en->rf_in_t))) return r;
            jb = en->rf_in_t.p;
        }
        if (!need_jblues) jb = en->op_stim_t.p;  // never read (no internal-up rows); any mapped table
        const long long total = (long long)S * en->tpad;
        if (en->continuum) {  // into the Markov build's input; tp_t keeps the deactivation table until that build
            en->mk_resident = false;
            if ((r = en->mk_p_t.ensure((size_t)S * en->tpad + TABLE_SLACK)) || (r = upload_continuum_rates(en, p->continuum))) return r;
            continuum_row_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(en->op_const, en->ttype.p, en->tline.p, en->ct_off.p,
                en->ct_energy.p, en->ct_tab.p, en->ct_shell.p, en->op_beta_t.p, en->op_stim_t.p, jb, en->nu_line.p, en->at_ful.p, en->at_flu.p,
                en->at_elo.p, en->at_eup.p, en->T, en->tpad, lpad, S, en->mk_p_t.p);
            const long long nb = (long long)en->n_blocks * S;
            continuum_normalize_kernel<<<(unsigned)((nb + 127) / 128), 128, 0, st>>>(en->mk_p_t.p, en->block_edge.p, en->n_blocks, S, en->tpad);
            en->launches += 2;
            CK(cudaGetLastError());
            if (en->keep_opacity_tables) {
                if ((r = en->op_cont_tp_t.ensure((size_t)S * en->tpad))) return r;
                CK(cudaMemcpyAsync(en->op_cont_tp_t.p, en->mk_p_t.p, (size_t)S * en->tpad * sizeof(double), cudaMemcpyDeviceToDevice, st));
            }
            if ((r = wait_opacity_build(en))) return r;
            // the chain is built from this table next (tb200_build_absorbing_markov with transition_probabilities == NULL),
            // which also finishes the tables the kernels read
            en->op_cont_valid = en->keep_opacity_tables != 0;
            en->mk_resident = true;
            en->markov_pending = true;
            en->opacity_pending = false;
            return TB200_OK;
        }
        opacity_row_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(en->op_const, en->ttype.p, en->tline.p, en->op_beta_t.p, en->op_stim_t.p, jb,
            en->nu_line.p, en->at_ful.p, en->at_flu.p, en->at_elo.p, en->at_eup.p, en->T, en->tpad, lpad, S, en->tp_t.p);
        const long long nb = (long long)en->n_blocks * S;
        opacity_normalize_kernel<<<(unsigned)((nb + 127) / 128), 128, 0, st>>>(en->tp_t.p, en->block_edge.p, en->n_blocks, S, en->tpad);
        en->launches += 2;
        CK(cudaGetLastError());
        if (en->keep_opacity_tables) {
            if ((r = en->op_tp_norm_t.ensure((size_t)S * en->tpad))) return r;
            CK(cudaMemcpyAsync(en->op_tp_norm_t.p, en->tp_t.p, (size_t)S * en->tpad * sizeof(double), cudaMemcpyDeviceToDevice, st));
        }
    }
    if ((r = finish_opacity_tables(en)) || (r = wait_opacity_build(en))) return r;
    en->opacity_pending = false;
    return TB200_OK;
}

int tb200_download_opacity(tb200_engine *en, double *tau, double *beta, double *stim, double *tp) {
    if (!en) return fail(TB200_ERR_INVALID, "bad argument");
    if (!en->have_model || en->opacity_pending) return fail(TB200_ERR_NO_MODEL, "no opacity tables on the device");
    CK(cudaSetDevice(en->device));
    cudaStream_t st = en->stream;
    int r;
    double *dst[3] = {tau, beta, stim};
    const double *src[3] = {en->tau_t.p, en->op_beta_t.p, en->op_stim_t.p};
    for (int k = 0; k < 3; k++) {
        if (!dst[k]) continue;
        if (!src[k]) return fail(TB200_ERR_INVALID, "this table was not built on the device");
        if ((r = download_line_major(en, src[k], en->L, en->lpad, dst[k]))) return r;
        CK(cudaStreamSynchronize(st));
    }
    if (tp) {
        if (en->continuum && !en->op_cont_valid)
            return fail(TB200_ERR_INVALID, "transition_probabilities: no kept table of a continuum-mode tb200_build_opacity (set the option "
                                           "keep_opacity_tables before it; the deactivation table is tb200_download_absorbing_markov's)");
        const double *kept = en->continuum ? en->op_cont_tp_t.p : en->op_tp_norm_t.p;
        if (!en->have_macro || !kept) return fail(TB200_ERR_INVALID, "transition_probabilities: set the option keep_opacity_tables before tb200_build_opacity");
        if ((r = download_line_major(en, kept, en->T, en->tpad, tp))) return r;
        CK(cudaStreamSynchronize(st));
    }
    return TB200_OK;
}

// ---- classic plasma on the device (plasma.cuh) --------------------------------------------------------------------------
namespace {
// (level, shell): the Boltzmann factors, into op_lnd (overwritten in place by the populations at the end)
__global__ void plasma_boltzmann_kernel(const tbp::Shell *sh, const double *g, const unsigned char *meta, const double *energy,
                                        long long n_levels, int n_shells, int dilute, double *lbf) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_levels * n_shells) return;
    const long long l = i / n_shells;
    const int s = (int)(i % n_shells);
    lbf[i] = tbp::boltzmann_factor(g[l], energy[l], sh[s].beta_rad, sh[s].w, dilute && !meta[l]);
}
// (ion, shell): the partition function, then Phi of every ion of charge >= 1 (0 in the rows of charge 0, never read)
__global__ void plasma_partition_kernel(const double *lbf, const int *ion_first, int n_ions, int n_shells, double *z) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)n_ions * n_shells) return;
    const int ion = (int)(i / n_shells), s = (int)(i % n_shells);
    z[i] = tbp::partition_function(lbf, ion_first[ion], ion_first[ion + 1], n_shells, s);
}
__global__ void plasma_phi_kernel(const tbp::Shell *sh, const double *z, const double *charge, const double *chi, const double *zeta, int n_t,
                                  int n_ions, int n_shells, int nebular, double chi_0, double delta_treatment, double *phi) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)n_ions * n_shells) return;
    const int ion = (int)(i / n_shells), s = (int)(i % n_shells);
    if (charge[ion] == 0.0) { phi[i] = 0.0; return; }
    const tbp::Shell h = sh[s];
    double p = tbp::phi_lte(z[i], z[i - n_shells], h.g_e, chi[ion], h.beta_rad);
    if (nebular)
        p = tbp::phi_nebular(h, p, tbp::zeta_value(h, zeta + (size_t)ion * n_t), tbp::radiation_field_correction(h, chi[ion], chi_0, delta_treatment));
    phi[i] = p;
}
// The n_e fixed point in one CTA (tbp::ne_fixed_point): the threads share out the (element, shell) population blocks and
// the shells; the all-shells test is a block-wide AND.  status = {population passes, tbp::NeStatus}.
constexpr int NE_THREADS = 1024;
extern "C++" {  // a template, inside the C-ABI block
struct CtaTeam {
    template <class F> __device__ void each(int n, F f) { for (int i = threadIdx.x; i < n; i += blockDim.x) f(i); }
    __device__ void sync() { __syncthreads(); }
    __device__ bool any(bool v) { return __syncthreads_or(v) != 0; }
    __device__ bool all(bool v) { return __syncthreads_and(v) != 0; }
};
}  // extern "C++"
__global__ void __launch_bounds__(NE_THREADS) plasma_ne_kernel(const double *phi, const double *nd, const int *element_first, int n_elements,
                                                               const double *charge, int n_ions, int n_shells, double threshold,
                                                               const double *fixed_ne, double *pop, double *ne, double *new_ne, int *status) {
    CtaTeam team;
    int passes = 0;
    const tbp::NeStatus r = tbp::ne_fixed_point(team, phi, nd, element_first, n_elements, charge, n_ions, n_shells, threshold, fixed_ne, pop, ne,
                                                new_ne, &passes);
    if (threadIdx.x == 0) { status[0] = passes; status[1] = (int)r; }
}
// (level, shell): Boltzmann factor -> population, in place
__global__ void plasma_level_kernel(const int *level_ion, const double *z, const double *pop, long long n_levels, int n_shells, double *lnd) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_levels * n_shells) return;
    const long long l = i / n_shells;
    const size_t c = (size_t)level_ion[l] * n_shells + (size_t)(i % n_shells);
    lnd[i] = tbp::level_population(lnd[i], z[c], pop[c]);
}
// (shell, line) of the [S][lpad] table the opacity build reads: W B_nu(T_rad) (W = 1 for the black body), 0 in the padding
__global__ void plasma_jblue_kernel(tbr::Constants K, const tbp::Shell *sh, const double *nu_line, int n_lines, int lpad, int n_shells, int blackbody,
                                    double *out_t) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)n_shells * lpad) return;
    const int s = (int)(i / lpad), l = (int)(i % lpad);
    out_t[i] = l < n_lines ? tbr::dilute_planck_intensity(K, nu_line[l], sh[s].t_rad, blackbody ? 1.0 : sh[s].w) : 0.0;
}
inline unsigned blocks_for(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }
}  // namespace

int tb200_set_plasma_data(tb200_engine *en, const tb200_plasma_data *d) {
    if (!en || !d) return fail(TB200_ERR_INVALID, "bad argument");
    if (!en->have_model) return fail(TB200_ERR_NO_MODEL, "tb200_set_model has not been called");
    if (en->continuum) return fail(TB200_ERR_INVALID, "plasma data: the continuum mode's plasma is the IIP one, which tb200_solve_plasma does not build");
    if (!en->have_atomic) return fail(TB200_ERR_NO_MODEL, "tb200_set_atomic_data has not been called (g and metastability come from it)");
    if (d->n_levels != en->n_levels) return fail(TB200_ERR_INVALID, "plasma data: n_levels differs from the atomic data's");
    if (d->n_shells != en->S) return fail(TB200_ERR_INVALID, "plasma data: n_shells differs from the model's");
    if (!d->level_energy || !d->level_ion || !d->ion_atomic_number || !d->ion_charge || !d->ionization_energy || !d->number_density)
        return fail(TB200_ERR_INVALID, "plasma data: missing array");
    if (d->n_ions < 2 || d->n_ions > d->n_levels) return fail(TB200_ERR_INVALID, "plasma data: n_ions out of range");
    const int64_t NL = d->n_levels, NI = d->n_ions;
    // levels grouped by ion, in the ion table's order, every ion with at least one level (the partition function's rows)
    std::vector<int> ion_first((size_t)NI + 1, 0);
    for (int64_t l = 0; l < NL; l++) {
        const int64_t ion = d->level_ion[l], prev = l ? d->level_ion[l - 1] : -1;
        if (ion < 0 || ion >= NI) return fail(TB200_ERR_INVALID, "plasma data: level_ion of level " + std::to_string(l) + " is out of range");
        if (ion != prev && ion != prev + 1)
            return fail(TB200_ERR_INVALID, "plasma data: levels are not grouped by (atomic_number, ion_number) in the ion table's order (level " +
                                               std::to_string(l) + ")");
        if (ion != prev) ion_first[(size_t)ion] = (int)l;
    }
    if (d->level_ion[NL - 1] != NI - 1) return fail(TB200_ERR_INVALID, "plasma data: an ion of the ion table has no level");
    ion_first[(size_t)NI] = (int)NL;
    // ions grouped by element in ascending atomic number, charges 0, 1, 2, ... in each; at least two ions per element
    std::vector<int> element_first;
    std::vector<double> charge((size_t)NI);
    for (int64_t i = 0; i < NI; i++) {
        const bool first = i == 0 || d->ion_atomic_number[i] != d->ion_atomic_number[i - 1];
        if (first) {
            if (i > 0 && d->ion_atomic_number[i] < d->ion_atomic_number[i - 1])
                return fail(TB200_ERR_INVALID, "plasma data: ions are not grouped by element in ascending atomic number (ion " + std::to_string(i) + ")");
            if (d->ion_charge[i] != 0)
                return fail(TB200_ERR_INVALID, "plasma data: the ions of atomic number " + std::to_string(d->ion_atomic_number[i]) +
                                                   " do not start from charge 0");
            if (i > 0 && i - element_first.back() < 2)
                return fail(TB200_ERR_INVALID, "plasma data: atomic number " + std::to_string(d->ion_atomic_number[i - 1]) +
                                                   " has a single ion (its Phi block would be empty and the elements' rows misalign)");
            element_first.push_back((int)i);
        } else {
            if (d->ion_charge[i] != d->ion_charge[i - 1] + 1)
                return fail(TB200_ERR_INVALID, "plasma data: the ions of atomic number " + std::to_string(d->ion_atomic_number[i]) +
                                                   " are not consecutive in charge (ion " + std::to_string(i) + ")");
            if (d->ionization_energy[i] != d->ionization_energy[i])
                return fail(TB200_ERR_INVALID, "plasma data: ion (" + std::to_string(d->ion_atomic_number[i]) + ", " + std::to_string(d->ion_charge[i]) +
                                                   ") has no ionisation energy (a Phi row without one)");
        }
        charge[(size_t)i] = (double)d->ion_charge[i];
    }
    if (NI - element_first.back() < 2)
        return fail(TB200_ERR_INVALID, "plasma data: atomic number " + std::to_string(d->ion_atomic_number[NI - 1]) + " has a single ion");
    const int n_elements = (int)element_first.size();
    element_first.push_back((int)NI);
    const int64_t NT = d->n_zeta_temperatures;
    if (NT < 0 || NT == 1) return fail(TB200_ERR_INVALID, "plasma data: the zeta grid needs at least 2 temperatures (or 0: none)");
    if (NT > 0) {
        if (!d->zeta_temperatures || !d->zeta) return fail(TB200_ERR_INVALID, "plasma data: zeta_temperatures or zeta is NULL");
        for (int64_t k = 1; k < NT; k++)
            if (!(d->zeta_temperatures[k] > d->zeta_temperatures[k - 1]))
                return fail(TB200_ERR_INVALID, "plasma data: zeta_temperatures must be strictly ascending");
    }
    CK(cudaSetDevice(en->device));
    en->pl_set = false;
    const int S = en->S;
    cudaStream_t st = en->stream;
    int r;
    if ((r = en->pl_energy.ensure(NL)) || (r = en->pl_level_ion.ensure(NL)) || (r = en->pl_ion_first.ensure(NI + 1)) || (r = en->pl_charge.ensure(NI)) ||
        (r = en->pl_chi.ensure(NI)) || (r = en->pl_element_first.ensure(element_first.size())) || (r = en->pl_nd.ensure((size_t)n_elements * S)) ||
        (r = en->pl_zeta.ensure((size_t)std::max<int64_t>(NT, 1) * NI)) || (r = en->pl_z.ensure((size_t)NI * S)) || (r = en->pl_phi.ensure((size_t)NI * S)) ||
        (r = en->pl_pop.ensure((size_t)NI * S)) || (r = en->pl_ne.ensure(S)) || (r = en->pl_new.ensure(S)) || (r = en->pl_fixed_ne.ensure(S)) ||
        (r = en->pl_status.ensure(2)) || (r = en->pl_shell.ensure(S)))
        return r;
    std::vector<int> level_ion((size_t)NL);
    for (int64_t l = 0; l < NL; l++) level_ion[(size_t)l] = (int)d->level_ion[l];
    CK(cudaMemcpyAsync(en->pl_energy.p, d->level_energy, NL * sizeof(double), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(en->pl_level_ion.p, level_ion.data(), NL * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(en->pl_ion_first.p, ion_first.data(), (NI + 1) * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(en->pl_charge.p, charge.data(), NI * sizeof(double), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(en->pl_chi.p, d->ionization_energy, NI * sizeof(double), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(en->pl_element_first.p, element_first.data(), element_first.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(en->pl_nd.p, d->number_density, (size_t)n_elements * S * sizeof(double), cudaMemcpyHostToDevice, st));
    if (NT > 0) CK(cudaMemcpyAsync(en->pl_zeta.p, d->zeta, (size_t)NT * NI * sizeof(double), cudaMemcpyHostToDevice, st));
    CK(cudaStreamSynchronize(st));  // the host vectors go out of scope
    en->pl_zeta_t.assign(d->zeta_temperatures, d->zeta_temperatures + NT);
    en->pl_S = S; en->pl_n_levels = NL; en->pl_n_ions = (int)NI; en->pl_n_elements = n_elements;
    en->pl_chi_0 = d->chi_0;
    en->pl_const = tbp::Constants{d->k_b, d->h, d->m_e};
    en->pl_c = d->c;
    en->pl_valid = false;
    en->pl_set = true;
    return TB200_OK;
}

int tb200_solve_plasma(tb200_engine *en, const tb200_plasma_params *p, double *electron_densities, double *ion_number_density,
                       double *level_number_density, double *j_blues, int32_t *iterations) {
    if (!en || !p || !p->t_radiative || !p->dilution_factor) return fail(TB200_ERR_INVALID, "bad argument");
    if (!en->have_model) return fail(TB200_ERR_NO_MODEL, "tb200_set_model has not been called");
    if (en->continuum) return fail(TB200_ERR_INVALID, "the continuum mode's plasma is the IIP one, which tb200_solve_plasma does not build");
    if (!en->pl_set) return fail(TB200_ERR_NO_MODEL, "tb200_set_plasma_data has not been called");
    if (en->pl_S != en->S || en->pl_n_levels != en->n_levels)
        return fail(TB200_ERR_NO_MODEL, "the plasma data were given for another shell or level count: call tb200_set_plasma_data again");
    if (p->ionization < 0 || p->ionization > 1 || p->excitation < 0 || p->excitation > 1 || p->radiative_rates_type < 0 || p->radiative_rates_type > 2)
        return fail(TB200_ERR_INVALID, "ionization must be 0 (nebular) or 1 (lte), excitation 0 (dilute-lte) or 1 (lte), radiative_rates_type 0, 1 or 2");
    const bool nebular = p->ionization == 0, detailed = p->radiative_rates_type == 2;
    if (nebular && en->pl_zeta_t.empty()) return fail(TB200_ERR_INVALID, "nebular ionisation needs the zeta table of tb200_set_plasma_data");
    if (detailed && j_blues && !en->rf_valid) return fail(TB200_ERR_INVALID, "j_blues: detailed keeps tb200_solve_radiation_field's table, and none is resident");
    const int S = en->S, L = en->L, lpad = en->lpad, NI = en->pl_n_ions;
    const long long NL = en->n_levels;
    // DilutePlanckianRadiationField's checks (plasma/radiation_field/planck_rad_field.py:46-48)
    for (int s = 0; s < S; s++)
        if (!(p->t_radiative[s] > 0 && std::isfinite(p->t_radiative[s])) || !(p->dilution_factor[s] >= 0 && std::isfinite(p->dilution_factor[s])))
            return fail(TB200_ERR_INVALID, "t_radiative must be positive and dilution_factor non-negative, both finite (shell " + std::to_string(s) + ")");
    std::vector<tbp::Shell> shells((size_t)S);
    const std::vector<double> &grid = en->pl_zeta_t;
    const int NT = (int)grid.size();
    for (int s = 0; s < S; s++) {
        tbp::Shell &h = shells[(size_t)s];
        h = tbp::shell_state(en->pl_const, p->t_radiative[s], p->dilution_factor[s], p->link_t_rad_t_electron, p->departure_coefficient);
        if (NT >= 2) {  // interp1d(bounds_error=False, fill_value=nan): NaN outside [grid[0], grid[-1]]
            const tbfi::ShellWeights w = tbfi::shell_weights(grid.data(), NT, h.t_rad);
            h.z_lo = w.lo; h.z_w_lo = w.w_lo; h.z_w_hi = w.w_hi;
            h.z_out = h.t_rad < grid[0] || h.t_rad > grid[(size_t)NT - 1];
        }
    }
    CK(cudaSetDevice(en->device));
    int r;
    if ((r = en->op_lnd.ensure((size_t)NL * S))) return r;
    if (!detailed && (r = en->rf_jblues_t.ensure((size_t)S * lpad))) return r;
    cudaStream_t st = en->stream;
    en->pl_valid = false;  // op_lnd is rebuilt from here on
    CK(cudaMemcpyAsync(en->pl_shell.p, shells.data(), (size_t)S * sizeof(tbp::Shell), cudaMemcpyHostToDevice, st));
    if (p->electron_densities) CK(cudaMemcpyAsync(en->pl_fixed_ne.p, p->electron_densities, (size_t)S * sizeof(double), cudaMemcpyHostToDevice, st));
    const long long level_cells = NL * S, ion_cells = (long long)NI * S;
    plasma_boltzmann_kernel<<<blocks_for(level_cells, 256), 256, 0, st>>>(en->pl_shell.p, en->at_g.p, en->at_meta.p, en->pl_energy.p, NL, S,
                                                                          p->excitation == 0, en->op_lnd.p);
    plasma_partition_kernel<<<blocks_for(ion_cells, 128), 128, 0, st>>>(en->op_lnd.p, en->pl_ion_first.p, NI, S, en->pl_z.p);
    plasma_phi_kernel<<<blocks_for(ion_cells, 128), 128, 0, st>>>(en->pl_shell.p, en->pl_z.p, en->pl_charge.p, en->pl_chi.p, en->pl_zeta.p, NT, NI, S,
                                                                  nebular, en->pl_chi_0, p->delta_treatment, en->pl_phi.p);
    plasma_ne_kernel<<<1, NE_THREADS, 0, st>>>(en->pl_phi.p, en->pl_nd.p, en->pl_element_first.p, en->pl_n_elements, en->pl_charge.p, NI, S,
                                               p->ion_zero_threshold, p->electron_densities ? en->pl_fixed_ne.p : nullptr, en->pl_pop.p, en->pl_ne.p,
                                               en->pl_new.p, en->pl_status.p);
    en->launches += 4;
    CK(cudaGetLastError());
    int status[2] = {0, 0};
    CK(cudaMemcpyAsync(status, en->pl_status.p, sizeof(status), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (iterations) *iterations = status[0];
    if (status[1] == tbp::NE_NAN) return fail(TB200_ERR_PLASMA_IONIZATION, "n_electron just turned \"nan\" - aborting");
    if (status[1] == tbp::NE_CAP)
        return fail(TB200_ERR_PLASMA_IONIZATION, "n_electron did not converge within " + std::to_string(tbp::MAX_NE_ITERATIONS) +
                                                     " iterations - aborting (the device's cap; the reference has none)");
    plasma_level_kernel<<<blocks_for(level_cells, 256), 256, 0, st>>>(en->pl_level_ion.p, en->pl_z.p, en->pl_pop.p, NL, S, en->op_lnd.p);
    en->launches++;
    if (!detailed) {
        tbr::Constants K{};
        K.c = en->pl_c; K.h = en->pl_const.h; K.k_b = en->pl_const.k_b;
        plasma_jblue_kernel<<<blocks_for((long long)S * lpad, 256), 256, 0, st>>>(K, en->pl_shell.p, en->nu_line.p, L, lpad, S,
                                                                                  p->radiative_rates_type == 1, en->rf_jblues_t.p);
        en->launches++;
    }
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(en->n_e.p, en->pl_ne.p, (size_t)S * sizeof(double), cudaMemcpyDeviceToDevice, st));
    if (electron_densities) CK(cudaMemcpyAsync(electron_densities, en->pl_ne.p, (size_t)S * sizeof(double), cudaMemcpyDeviceToHost, st));
    if (ion_number_density) CK(cudaMemcpyAsync(ion_number_density, en->pl_pop.p, (size_t)ion_cells * sizeof(double), cudaMemcpyDeviceToHost, st));
    if (level_number_density) CK(cudaMemcpyAsync(level_number_density, en->op_lnd.p, (size_t)level_cells * sizeof(double), cudaMemcpyDeviceToHost, st));
    if (j_blues && (r = download_line_major(en, en->rf_jblues_t.p, L, lpad, j_blues))) return r;
    CK(cudaStreamSynchronize(st));
    en->pl_valid = true;
    if (!detailed) en->rf_valid = true;
    return TB200_OK;
}

// ---- continuum macro atom on the device (markov_build.cuh) ----------------------------------------------------------
// Everything is checked on the host before anything is allocated or launched, so a refused call leaves the engine as it was.
static int check_markov_input(tb200_engine *en, const tb200_markov_input *in, std::vector<long long> &edges) {
    if (!en->have_model) return fail(TB200_ERR_NO_MODEL, "tb200_set_model has not been called");
    if (!en->continuum) return fail(TB200_ERR_INVALID, "tb200_build_absorbing_markov needs a continuum-mode model");
    if (!in->source_level_idx || !in->destination_level_idx || !in->transition_type)
        return fail(TB200_ERR_INVALID, "absorbing Markov chain: an input array is NULL");
    if (!in->transition_probabilities && !en->mk_resident)
        return fail(TB200_ERR_INVALID, "absorbing Markov chain: transition_probabilities is NULL and tb200_build_opacity has built no table "
                                       "since the last tb200_set_model");
    if (in->n_transitions != en->T) return fail(TB200_ERR_INVALID, "absorbing Markov chain: n_transitions differs from the model's");
    if (in->tp_transition_stride < 0 || in->tp_shell_stride < 0) return fail(TB200_ERR_INVALID, "negative strides are not supported");
    const int64_t T = in->n_transitions, n = in->n_states;
    // the model's block edges (uploaded as int32 by tb200_set_model)
    edges.assign((size_t)en->n_blocks + 1, 0);
    {
        std::vector<int> e32((size_t)en->n_blocks + 1);
        CK(cudaMemcpy(e32.data(), en->block_edge.p, e32.size() * sizeof(int), cudaMemcpyDeviceToHost));
        for (size_t b = 0; b < e32.size(); b++) edges[b] = e32[b];
    }
    if (edges[0] != 0 || edges[(size_t)en->n_blocks] != T)
        return fail(TB200_ERR_INVALID, "absorbing Markov chain: macro_block_edge_index must cover every row");
    int64_t max_src = -1;
    for (int64_t t = 0; t < T; t++) {
        const int64_t a = in->source_level_idx[t];
        if (a < 0 || a >= en->n_blocks) return fail(TB200_ERR_INVALID, "absorbing Markov chain: source_level_idx out of range at row " + std::to_string(t));
        max_src = std::max(max_src, a);
    }
    if (n != max_src + 1) return fail(TB200_ERR_INVALID, "absorbing Markov chain: n_states must be max(source_level_idx) + 1");
    for (int64_t b = 0; b < en->n_blocks; b++)
        for (long long t = edges[(size_t)b]; t < edges[(size_t)b + 1]; t++)
            if (in->source_level_idx[t] != b)
                return fail(TB200_ERR_INVALID, "absorbing Markov chain: row " + std::to_string(t) + " has source " +
                                                   std::to_string(in->source_level_idx[t]) + " but lies in block " + std::to_string(b) +
                                                   " of macro_block_edge_index");
    {  // the transport reads the rows by the model's types: the chain must be built from the same ones
        std::vector<int> tt32((size_t)(T > 0 ? T : 1));
        CK(cudaMemcpy(tt32.data(), en->ttype.p, (size_t)T * sizeof(int), cudaMemcpyDeviceToHost));
        for (int64_t t = 0; t < T; t++)
            if (in->transition_type[t] != tt32[(size_t)t])
                return fail(TB200_ERR_INVALID, "absorbing Markov chain: transition_type differs from the model's at row " + std::to_string(t));
    }
    for (int64_t t = 0; t < T; t++)
        if (in->transition_type[t] >= 0 && (in->destination_level_idx[t] < 0 || in->destination_level_idx[t] >= n))
            return fail(TB200_ERR_INVALID, "absorbing Markov chain: destination_level_idx out of range at internal row " + std::to_string(t));
    // the table: [S, n, n] doubles (twice with keep_opacity_tables), indices of the kernels' grids
    if (n > 65535 || en->S > 65535 || (long long)n * en->S >= INT_MAX)
        return fail(TB200_ERR_INVALID, "absorbing Markov chain: " + std::to_string(n) + " states x " + std::to_string(en->S) + " shells do not fit the solver");
    const double need = (double)en->S * n * n * 8.0 * (en->keep_opacity_tables ? 2 : 1) +
                        8.0 * ((double)en->S * (en->tpad + 3.0 * n) + TABLE_SLACK) + 8.0 * en->T;  // + input table, q / r / c, type / dest
    size_t free_b = 0, total_b = 0;
    CK(cudaMemGetInfo(&free_b, &total_b));
    const double have = (double)free_b + 8.0 * ((double)en->markov_cum.n + en->mk_keep.n + en->mk_p_t.n + en->mk_q.n + en->mk_r.n + en->mk_c.n) +
                        4.0 * ((double)en->mk_type.n + en->mk_dest.n);
    if (need > have)
        return fail(TB200_ERR_INVALID, "absorbing Markov chain: the table needs " + std::to_string(need / 1e9) + " GB, " +
                                           std::to_string(have / 1e9) + " GB are free on the device");
    return TB200_OK;
}

int tb200_build_absorbing_markov(tb200_engine *en, const tb200_markov_input *in) {
    if (!en || !in) return fail(TB200_ERR_INVALID, "bad argument");
    CK(cudaSetDevice(en->device));
    std::vector<long long> edges;
    int r;
    if ((r = check_markov_input(en, in, edges))) return r;
    const int S = en->S, n = (int)in->n_states;
    cudaStream_t st = en->stream;
    en->markov_pending = true;  // until the build below has finished
    en->mk_keep_n = 0;
    if (in->transition_probabilities) {  // otherwise mk_p_t holds the table tb200_build_opacity left
        en->mk_resident = false;
        if ((r = upload_strided_table(en, in->transition_probabilities, en->T, S, in->tp_transition_stride, in->tp_shell_stride, en->tpad, en->mk_p_t))) return r;
    }
    if ((r = upload_i64_as_i32(en, in->transition_type, en->T, en->mk_type)) ||
        (r = upload_i64_as_i32(en, in->destination_level_idx, en->T, en->mk_dest)))
        return r;
    const size_t nm = (size_t)S * n * n, sn = (size_t)S * n;
    if ((r = en->markov_cum.ensure(nm)) || (r = en->mk_q.ensure(sn)) || (r = en->mk_r.ensure(sn)) || (r = en->mk_c.ensure(sn)) ||
        (r = en->mk_err.ensure(1)))
        return r;
    if (en->keep_opacity_tables && (r = en->mk_keep.ensure(nm))) return r;
    const int no_error = INT_MAX;
    CK(cudaMemcpyAsync(en->mk_err.p, &no_error, sizeof(int), cudaMemcpyHostToDevice, st));
    double *A = en->markov_cum.p;
    CK(cudaMemsetAsync(A, 0, nm * sizeof(double), st));
    tbm::markov_assemble_kernel<<<(unsigned)((sn + 127) / 128), 128, 0, st>>>(en->mk_p_t.p, en->tpad, en->block_edge.p, en->mk_type.p,
                                                                            en->mk_dest.p, n, S, A, en->mk_q.p);
    tbm::markov_identity_minus_kernel<<<(unsigned)((nm + 255) / 256), 256, 0, st>>>(A, n, (long long)nm);
    en->launches += 2;
    CK(cudaGetLastError());
    if (n <= tbm::SMEM_MAX_N) {
        const size_t smem = ((size_t)n * n + 2 * (size_t)n) * sizeof(double);
        CK(cudaFuncSetAttribute(tbm::markov_solve_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        tbm::markov_solve_smem_kernel<<<S, 256, smem, st>>>(A, n, S, en->mk_err.p);
        en->launches++;
        CK(cudaGetLastError());
    } else {
        const dim3 grid((unsigned)((n + 127) / 128), (unsigned)n, (unsigned)S);
        for (int k = 0; k < n; k++) {
            tbm::markov_pivot_kernel<<<(unsigned)((sn + 255) / 256), 256, 0, st>>>(A, n, S, k, en->mk_r.p, en->mk_c.p, en->mk_err.p);
            tbm::markov_update_kernel<<<grid, 128, 0, st>>>(A, n, k, en->mk_r.p, en->mk_c.p);
        }
        en->launches += 2LL * n;
        CK(cudaGetLastError());
    }
    int err = no_error;
    CK(cudaMemcpyAsync(&err, en->mk_err.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (err != no_error)
        return fail(TB200_ERR_INVALID, "absorbing Markov chain: I - Q is singular in shell " + std::to_string(err % S) + " at state " +
                                           std::to_string(err / S) + " (a pivot <= 0 or not finite: the chain is not absorbing)");
    tbm::markov_scale_kernel<<<(unsigned)((nm + 255) / 256), 256, 0, st>>>(A, en->mk_q.p, n, S, en->keep_opacity_tables ? en->mk_keep.p : nullptr);
    const long long rows = (long long)sn;
    tb::markov_cumsum_kernel<<<(unsigned)((rows + 127) / 128), 128, 0, st>>>(A, rows, n);
    const long long nb = (long long)en->n_blocks * S;
    tbm::markov_deactivation_kernel<<<(unsigned)((nb + 127) / 128), 128, 0, st>>>(en->mk_p_t.p, en->tpad, en->block_edge.p, en->n_blocks,
                                                                                en->mk_type.p, S, en->tp_t.p);
    en->launches += 3;
    CK(cudaGetLastError());
    if (en->keep_opacity_tables) {
        if ((r = en->op_tp_norm_t.ensure((size_t)S * en->tpad))) return r;
        CK(cudaMemcpyAsync(en->op_tp_norm_t.p, en->tp_t.p, (size_t)S * en->tpad * sizeof(double), cudaMemcpyDeviceToDevice, st));
        en->mk_keep_n = n;
    }
    if ((r = finish_opacity_tables(en))) return r;
    CK(cudaStreamSynchronize(st));
    en->n_markov = n;
    en->markov_pending = false;
    return TB200_OK;
}

int tb200_download_absorbing_markov(tb200_engine *en, double *matrix, double *deactivating) {
    if (!en) return fail(TB200_ERR_INVALID, "bad argument");
    if (!en->have_model || !en->continuum || en->markov_pending) return fail(TB200_ERR_NO_MODEL, "no absorbing Markov chain on the device");
    CK(cudaSetDevice(en->device));
    if (en->mk_keep_n == 0)
        return fail(TB200_ERR_INVALID, "the chain was not kept: set the option keep_opacity_tables = 1 before tb200_build_absorbing_markov");
    cudaStream_t st = en->stream;
    const int S = en->S;
    if (matrix) {
        const size_t nm = (size_t)S * en->mk_keep_n * en->mk_keep_n;
        CK(cudaMemcpyAsync(matrix, en->mk_keep.p, nm * sizeof(double), cudaMemcpyDeviceToHost, st));
    }
    int r;
    if (deactivating && (r = download_line_major(en, en->op_tp_norm_t.p, en->T, en->tpad, deactivating))) return r;
    CK(cudaStreamSynchronize(st));
    return TB200_OK;
}

int tb200_get_estimator_layout(tb200_engine *en, tb200_estimator_layout *l) {
    if (!en || !l) return fail(TB200_ERR_INVALID, "bad argument");
    if (!en->have_model) return fail(TB200_ERR_NO_MODEL, "tb200_set_model has not been called");
    l->n_doubles = (int64_t)en->est_count;
    l->n_shells = en->S; l->n_lines = en->L; l->line_pitch = en->lpad; l->n_grid = en->n_grid; l->n_continua = en->continuum ? en->n_continua : 0;
    l->off_j = (int64_t)en->off_J; l->off_nu_bar = (int64_t)en->off_nubar; l->off_vhist = (int64_t)en->off_vhist;
    l->off_spectrum_emitted = en->n_grid > 1 ? (int64_t)en->off_spec : -1;
    l->off_spectrum_reabsorbed = en->n_grid > 1 ? (int64_t)(en->off_spec + (size_t)(en->n_grid - 1)) : -1;
    l->off_luminosity = (int64_t)en->off_lum;
    l->off_ff_heating = en->continuum ? (int64_t)en->off_ffheat : -1;
    l->off_continuum = en->continuum ? (int64_t)en->off_cont : -1;
    l->n_continuum_doubles = en->continuum ? (int64_t)5 * en->n_continua * en->S : 0;
    l->off_j_blue = (int64_t)en->off_jblue; l->off_edotlu = (int64_t)en->off_edotlu;
    return TB200_OK;
}

int tb200_last_kernel_ms(tb200_engine *en, double *ms) {
    if (!en || !ms) return fail(TB200_ERR_INVALID, "bad argument");
    if (!en->timing_valid) return fail(TB200_ERR_INVALID, "no transport kernel has been timed");
    CK(cudaSetDevice(en->device));
    if (en->chunked_timing) { *ms = en->chunk_kernel_ms; return TB200_OK; }
    CK(cudaEventSynchronize(en->ev_stop));
    float f = 0;
    CK(cudaEventElapsedTime(&f, en->ev_start, en->ev_stop));
    *ms = f;
    return TB200_OK;
}

int64_t tb200_kernel_launches(tb200_engine *en) { return en ? en->launches : 0; }

}  // extern "C"

#include "group.cuh"  // engine groups: several engines driven from one call (needs tb200_engine's fields)
