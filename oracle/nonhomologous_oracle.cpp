/*
 * nonhomologous_oracle.cpp -- CPU restatement of the reference's nonhomologous transport mode.
 *
 * TEST INFRASTRUCTURE ONLY (like tardis_oracle.c): compiled by tests/ with g++ -O2 -ffp-contract=off, never called by the
 * product.  Restates, statement by statement (paths relative to the reference's tardis/ package):
 *   montecarlo_transport_with_vpackets   transport/montecarlo/modes/montecarlo_transport.py:239-373 (one thread, packets
 *                                        in order)
 *   packet_propagation                   modes/nonhomologous/packet_propagation.py:53-263
 *   trace_packet                         modes/nonhomologous/rad_packet_transport.py:25-198
 *   line_scatter_event / line_emission / thomson_scatter
 *                                        modes/nonhomologous/interaction_event_callers.py:27-93,189-239,
 *                                        modes/nonhomologous/interaction_events.py:183-262, macro_atom.py:52-104
 *   trace_vpacket_within_shell / trace_vpacket / trace_vpacket_volley
 *                                        modes/nonhomologous/virtual_packet.py:83-378
 * The line distance (the quartic) is NOT restated here: it is the product's own header, tardis_b200/csrc/nonhomologous.cuh,
 * compiled for the host, so that the oracle and the device evaluate it with the same operations.
 * Input / output layouts are tardis_oracle.h's (row-major (line, shell) tables).
 */
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../tardis_b200/csrc/nonhomologous.cuh"
#include "tardis_oracle.h"

namespace {

constexpr double C_SPEED_OF_LIGHT = 2.99792458e10;
enum { IT_BOUNDARY = 1, IT_LINE = 2, IT_ESCATTERING = 4 };
enum { ST_IN_PROCESS = 0, ST_EMITTED = 1, ST_REABSORBED = 2 };

/* Numba's MT19937, numba/_random.c:37-75, numba/cpython/randomimpl.py:109-147 */
struct Mt {
    uint32_t mt[624];
    int index;
    int64_t draws;
    void seed(uint32_t s) {
        for (int pos = 0; pos < 624; pos++) { mt[pos] = s; s = 1812433253U * (s ^ (s >> 30)) + (uint32_t)pos + 1U; }
        index = 624; draws = 0;
    }
    void shuffle() {
        int i; uint32_t y;
        for (i = 0; i < 624 - 397; i++) { y = (mt[i] & 0x80000000U) | (mt[i + 1] & 0x7fffffffU); mt[i] = mt[i + 397] ^ (y >> 1) ^ ((uint32_t)(-(int32_t)(y & 1)) & 0x9908b0dfU); }
        for (; i < 623; i++) { y = (mt[i] & 0x80000000U) | (mt[i + 1] & 0x7fffffffU); mt[i] = mt[i + (397 - 624)] ^ (y >> 1) ^ ((uint32_t)(-(int32_t)(y & 1)) & 0x9908b0dfU); }
        y = (mt[623] & 0x80000000U) | (mt[0] & 0x7fffffffU);
        mt[623] = mt[396] ^ (y >> 1) ^ ((uint32_t)(-(int32_t)(y & 1)) & 0x9908b0dfU);
    }
    uint32_t next_u32() {
        if (index >= 624) { shuffle(); index = 0; }
        uint32_t y = mt[index++];
        y ^= y >> 11; y ^= (y << 7) & 0x9d2c5680U; y ^= (y << 15) & 0xefc60000U; y ^= y >> 18;
        return y;
    }
    double next_double() {
        const uint32_t a = next_u32() >> 5, b = next_u32() >> 6;
        draws++;
        return ((double)b + (double)a * 67108864.0) / 9007199254740992.0;
    }
};

struct Packet {
    double r, mu, nu, energy;
    int64_t next_line_id, prev_line_id, current_shell_id, status, index;
};

struct Tracker {  // TrackerLastInteraction, packets/trackers/tracker_last_interaction.py:7-254
    double radius, before_nu, before_mu, before_energy, after_nu, after_mu, after_energy;
    int64_t shell_id, interaction_type, line_absorb_id, line_emit_id, interactions_count, boundary_buffer;
};

struct Ctx {
    const tardis_oracle_model *m;
    const tardis_oracle_config *c;
    tardis_oracle_outputs *out;
    std::vector<double> dvdr;
    const double *v_inner, *v_outer;
    Mt rng;
    Tracker trk;
    tardis_oracle_event *ev;
    int64_t ev_cap, ev_n;
    std::vector<double> vp_nu, vp_energy, vp_mu, vp_r;
    tardis_oracle_counters cnt;
    int error;

    /* NumbaRadial1DGeometry.get_velocity, model/geometry/radial1d.py:359-375 */
    double velocity(double r, int64_t s) const { return nh::velocity(r, m->r_inner[s], v_inner[s], dvdr[s]); }
    double distance_line(double r, double mu, double nu, int64_t s, double nu_line) const {
        return nh::distance_line(r, mu, nu, nu_line, m->r_inner[s], m->r_outer[s], v_inner[s], v_outer[s], dvdr[s], velocity(r, s));
    }
};

/* frame_transformations.py:12-72, partial relativity */
double doppler_factor(double velocity, double mu) { const double beta = velocity * (1 / C_SPEED_OF_LIGHT); return 1.0 - mu * beta; }
double inverse_doppler_factor(double velocity, double mu) { const double beta = velocity * (1 / C_SPEED_OF_LIGHT); return 1.0 / (1.0 - mu * beta); }

/* calculate_distances.py:25-62 */
double distance_boundary(double r, double mu, double r_inner, double r_outer, int64_t *delta_shell) {
    double distance;
    if (mu > 0.0) { distance = sqrt(r_outer * r_outer + ((mu * mu - 1.0) * r * r)) - (r * mu); *delta_shell = 1; }
    else {
        const double check = r_inner * r_inner + (r * r * (mu * mu - 1.0));
        if (check >= 0.0) { distance = -r * mu - sqrt(check); *delta_shell = -1; }
        else { distance = sqrt(r_outer * r_outer + ((mu * mu - 1.0) * r * r)) - (r * mu); *delta_shell = 1; }
    }
    return distance;
}

void log_event(Ctx *x, const Packet *p, int type, int64_t from_shell, int64_t to_shell, int before) {
    if (!x->ev || x->ev_n >= x->ev_cap) return;
    tardis_oracle_event *e = &x->ev[x->ev_n];
    if (before) {
        e->packet_id = p->index; e->interaction_type = type; e->status = p->status; e->radius = p->r;
        e->before_shell_id = from_shell; e->after_shell_id = to_shell;
        e->before_nu = p->nu; e->before_mu = p->mu; e->before_energy = p->energy;
        e->line_absorb_id = (type == IT_LINE) ? p->next_line_id : -1; e->line_emit_id = -1;
        if (type == IT_BOUNDARY) { e->after_nu = p->nu; e->after_mu = p->mu; e->after_energy = p->energy; x->ev_n++; }
    } else {
        e->after_nu = p->nu; e->after_mu = p->mu; e->after_energy = p->energy;
        if (type == IT_LINE) e->line_emit_id = p->next_line_id - 1;
        x->ev_n++;
    }
}
void track_boundary(Ctx *x, const Packet *p, int64_t from, int64_t to) {
    x->trk.boundary_buffer += 1;
    x->cnt.n_boundary_events++;
    log_event(x, p, IT_BOUNDARY, from, to, 1);
}
void track_before(Ctx *x, const Packet *p, int type) {
    Tracker *t = &x->trk;
    t->before_nu = p->nu; t->before_mu = p->mu; t->before_energy = p->energy;
    if (type == IT_LINE) t->line_absorb_id = p->next_line_id;
    else { t->line_absorb_id = -1; t->line_emit_id = -1; }
    log_event(x, p, type, p->current_shell_id, p->current_shell_id, 1);
}
void track_after(Ctx *x, const Packet *p, int type) {
    Tracker *t = &x->trk;
    t->after_nu = p->nu; t->after_mu = p->mu; t->after_energy = p->energy;
    if (type == IT_LINE) t->line_emit_id = p->next_line_id - 1;
    t->interactions_count += 1 + t->boundary_buffer;
    t->boundary_buffer = 0;
    t->radius = p->r; t->shell_id = p->current_shell_id; t->interaction_type = type;
    log_event(x, p, type, 0, 0, 0);
}

void move_packet_across_shell_boundary(int64_t *shell, int64_t *status, int64_t delta_shell, int64_t n_shells) {
    const int64_t next = *shell + delta_shell;
    if (next >= n_shells) *status = ST_EMITTED;
    else if (next < 0) *status = ST_REABSORBED;
    else *shell = next;
}

/* rad_packet_transport.py:25-198 */
double trace_packet(Ctx *x, Packet *p, double opacity_electron, int *interaction_type, int64_t *delta_shell) {
    const tardis_oracle_model *m = x->m;
    const int64_t s = p->current_shell_id, L = m->n_lines;
    const double r_inner = m->r_inner[s], r_outer = m->r_outer[s], v_inner = x->v_inner[s];
    const double d_b = distance_boundary(p->r, p->mu, r_inner, r_outer, delta_shell);
    const double tau_event = -log(x->rng.next_double());
    double tau_trace_line_combined = 0.0;
    const double dvdr = x->dvdr[s];
    const bool forward = dvdr >= 0.0;
    const int64_t start = forward ? p->next_line_id : p->prev_line_id;
    const int64_t lim = forward ? L : -1, dir = forward ? 1 : -1;
    double distance_electron = tau_event / opacity_electron;
    int64_t cur = start;
    for (int64_t i = start; forward ? i < lim : i > lim; i += dir) {
        cur = i;
        const double nu_line = m->line_list_nu[cur];
        tau_trace_line_combined += m->tau_sobolev[cur * m->n_shells + s];
        const double distance_trace = x->distance_line(p->r, p->mu, p->nu, s, nu_line);
        const double tau_trace_combined = tau_trace_line_combined + opacity_electron * distance_trace;
        double distance = distance_trace;  /* Python's min(a, b, c) */
        if (d_b < distance) distance = d_b;
        if (distance_electron < distance) distance = distance_electron;
        if (distance_trace != 0) {
            if (distance == d_b || distance == distance_electron) {
                if (forward) { p->next_line_id = cur; p->prev_line_id = cur - 1; }
                else { p->next_line_id = cur + 1; p->prev_line_id = cur; }
            }
            if (distance == d_b) { *interaction_type = IT_BOUNDARY; return distance; }
            if (distance == distance_electron) { *interaction_type = IT_ESCATTERING; return distance; }
        }
        const double new_r = sqrt(p->r * p->r + distance_trace * distance_trace + 2.0 * p->r * distance_trace * p->mu);
        const double new_mu = (p->mu * p->r + distance_trace) / new_r;
        const double new_v = v_inner + dvdr * (new_r - r_inner);
        const double energy = p->energy * (1.0 - new_v / C_SPEED_OF_LIGHT * new_mu);
        x->out->j_blue[cur * m->n_shells + s] += energy / p->nu;
        x->out->edotlu[cur * m->n_shells + s] += energy;
        x->cnt.n_line_steps++;
        if (tau_trace_combined > tau_event && !x->c->disable_line_scattering) {
            *interaction_type = IT_LINE;
            p->next_line_id = cur; p->prev_line_id = cur - 1;
            return distance_trace;
        }
        distance_electron = (tau_event - tau_trace_line_combined) / opacity_electron;
    }
    if (forward) {
        if (cur == L - 1) cur += 1;
        p->next_line_id = cur; p->prev_line_id = cur - 1;
    } else {
        if (cur == 0) cur -= 1;
        p->next_line_id = cur + 1; p->prev_line_id = cur;
    }
    if (distance_electron < d_b) { *interaction_type = IT_ESCATTERING; return distance_electron; }
    *interaction_type = IT_BOUNDARY;
    return d_b;
}

/* packets/movement.py:30-76 */
void move_r_packet(Ctx *x, Packet *p, double distance) {
    const double dop = doppler_factor(x->velocity(p->r, p->current_shell_id), p->mu);
    const double r = p->r;
    if (distance > 0.0) {
        const double new_r = sqrt(r * r + distance * distance + 2.0 * r * distance * p->mu);
        p->mu = (p->mu * r + distance) / new_r;
        p->r = new_r;
        const double cnu = p->nu * dop, cen = p->energy * dop;
        x->out->j[p->current_shell_id] += cen * distance;
        x->out->nu_bar[p->current_shell_id] += cen * distance * cnu;
    }
}

void line_emission(Ctx *x, Packet *p, int64_t emission_line_id) {
    const double inv = inverse_doppler_factor(x->velocity(p->r, p->current_shell_id), p->mu);
    p->nu = x->m->line_list_nu[emission_line_id] * inv;
    p->next_line_id = emission_line_id + 1;
}

/* macro_atom.py:52-104 */
int64_t macro_atom_interaction(Ctx *x, int64_t level, int64_t shell, int64_t *ttype) {
    const tardis_oracle_model *m = x->m;
    int64_t type = 0, tid = 0;
    while (type >= 0) {
        double probability = 0.0;
        const double xi = x->rng.next_double();
        x->cnt.n_macro_jumps++;
        const int64_t b0 = m->macro_block_edge_index[level], b1 = m->macro_block_edge_index[level + 1];
        bool found = false;
        for (tid = b0; tid < b1; tid++) {
            probability += m->transition_probabilities[tid * m->n_shells + shell];
            x->cnt.n_macro_scanned++;
            if (probability > xi) { level = m->destination_level_id[tid]; type = m->transition_type[tid]; found = true; break; }
        }
        if (!found) { x->error = TARDIS_ORACLE_ERR_MACRO_ATOM; *ttype = -99; return 0; }
    }
    *ttype = type;
    return m->transition_line_id[tid];
}

void line_scatter_event(Ctx *x, Packet *p) {
    const double v = x->velocity(p->r, p->current_shell_id);
    const double old_dop = doppler_factor(v, p->mu);
    p->mu = 2.0 * x->rng.next_double() - 1.0;
    const double inv_new = inverse_doppler_factor(v, p->mu);
    const double cen = p->energy * old_dop;
    p->energy = cen * inv_new;
    if (x->c->line_interaction_type == 0) {
        line_emission(x, p, p->next_line_id);
    } else {
        const double cnu = p->nu * old_dop;
        p->nu = cnu * inv_new;
        int64_t ttype;
        const int64_t line = macro_atom_interaction(x, x->m->line2macro_level_upper[p->next_line_id], p->current_shell_id, &ttype);
        if (x->error) return;
        if (ttype == -1) line_emission(x, p, line);
        else x->error = TARDIS_ORACLE_ERR_MACRO_ATOM;
    }
}

void thomson_scatter(Ctx *x, Packet *p) {
    const double v = x->velocity(p->r, p->current_shell_id);
    const double old_dop = doppler_factor(v, p->mu);
    const double cnu = p->nu * old_dop, cen = p->energy * old_dop;
    p->mu = 2.0 * x->rng.next_double() - 1.0;
    const double inv_new = inverse_doppler_factor(v, p->mu);
    p->nu = cnu * inv_new;
    p->energy = cen * inv_new;
}

/* virtual_packet.py:83-186 */
double trace_vpacket_within_shell(Ctx *x, Packet *v, double *d_b_out, int64_t *delta_shell) {
    const tardis_oracle_model *m = x->m;
    const int64_t s = v->current_shell_id, L = m->n_lines;
    const double d_b = distance_boundary(v->r, v->mu, m->r_inner[s], m->r_outer[s], delta_shell);
    const double chi_e = m->electron_density[s] * x->c->sigma_thomson;
    double tau = chi_e * d_b;
    const bool forward = x->dvdr[s] >= 0.0;
    const int64_t start = forward ? v->next_line_id : v->prev_line_id, lim = forward ? L : -1, dir = forward ? 1 : -1;
    int64_t cur = start;
    bool broke = false;
    for (int64_t i = start; forward ? i < lim : i > lim; i += dir) {
        cur = i;
        const double d_line = x->distance_line(v->r, v->mu, v->nu, s, m->line_list_nu[cur]);
        x->cnt.n_vpacket_line_steps++;
        if (d_b <= d_line) { broke = true; break; }
        tau += m->tau_sobolev[cur * m->n_shells + s];
    }
    if (!broke) {
        if (forward) { if (cur == L - 1) cur += 1; }
        else { if (cur == 0) cur -= 1; }
    }
    if (forward) { v->next_line_id = cur; v->prev_line_id = cur - 1; }
    else { v->next_line_id = cur + 1; v->prev_line_id = cur; }
    *d_b_out = d_b;
    return tau;
}

double trace_vpacket(Ctx *x, Packet *v) {
    const tardis_oracle_config *c = x->c;
    double tau_total = 0.0;
    int64_t guard = 0;
    while (true) {
        double d_b; int64_t delta;
        tau_total += trace_vpacket_within_shell(x, v, &d_b, &delta);
        move_packet_across_shell_boundary(&v->current_shell_id, &v->status, delta, x->m->n_shells);
        if (tau_total > c->vpacket_tau_russian) {
            const double event_random = x->rng.next_double();
            if (event_random > c->survival_probability) { v->energy = 0.0; v->status = ST_EMITTED; }
            else { v->energy = v->energy / c->survival_probability * exp(-tau_total); tau_total = 0.0; }
        }
        const double new_r = sqrt(v->r * v->r + d_b * d_b + 2.0 * v->r * d_b * v->mu);
        v->mu = (v->mu * v->r + d_b) / new_r;
        v->r = new_r;
        if (v->status == ST_EMITTED) break;
        if (++guard > 4 * x->m->n_shells + 64) { x->error = TARDIS_ORACLE_ERR_VPACKET_LOOP; break; }
    }
    return tau_total;
}

void trace_vpacket_volley(Ctx *x, const Packet *p) {
    const tardis_oracle_model *m = x->m;
    const tardis_oracle_config *c = x->c;
    if ((p->nu < c->vpacket_spawn_start_frequency) || (p->nu > c->vpacket_spawn_end_frequency)) return;
    const int64_t nv = c->number_of_vpackets;
    if (nv == 0) return;
    double mu_min; bool on_inner;
    if (p->r > m->r_inner[0]) { const double q = m->r_inner[0] / p->r; mu_min = -sqrt(1 - q * q); on_inner = false; }
    else { on_inner = true; mu_min = 0.0; }
    const double mu_bin = (1.0 - mu_min) / nv;
    const double v = x->velocity(p->r, p->current_shell_id);
    const double rp_dop = doppler_factor(v, p->mu);
    for (int64_t i = 0; i < nv; i++) {
        const double v_mu = mu_min + i * mu_bin + x->rng.next_double() * mu_bin;
        const double weight = on_inner ? 2 * v_mu / nv : (1 - mu_min) / (2 * nv);
        const double ratio = rp_dop / doppler_factor(v, v_mu);
        Packet vp;
        vp.r = p->r; vp.mu = v_mu; vp.nu = p->nu * ratio; vp.energy = p->energy * weight * ratio;
        vp.current_shell_id = p->current_shell_id; vp.next_line_id = p->next_line_id; vp.prev_line_id = vp.next_line_id - 1;
        vp.status = ST_IN_PROCESS; vp.index = i;
        const double tau = trace_vpacket(x, &vp);
        vp.energy *= exp(-tau);
        x->cnt.n_vpackets++;
        x->vp_nu.push_back(vp.nu); x->vp_energy.push_back(vp.energy); x->vp_mu.push_back(v_mu); x->vp_r.push_back(p->r);
    }
}

/* packet_propagation.py:53-263 */
void packet_propagation(Ctx *x, Packet *p) {
    const tardis_oracle_model *m = x->m;
    const int64_t L = m->n_lines;
    const double v0 = x->velocity(p->r, p->current_shell_id);
    const double inv = inverse_doppler_factor(v0, p->mu);
    p->nu *= inv; p->energy *= inv;
    const double comov_nu = p->nu * doppler_factor(x->velocity(p->r, p->current_shell_id), p->mu);
    int64_t ge = 0;  /* L - searchsorted(nu[::-1], comov_nu, 'left') = #lines with nu_line >= comov_nu */
    for (int64_t lo = 0, hi = L; lo < hi;) { const int64_t mid = (lo + hi) / 2; if (m->line_list_nu[mid] >= comov_nu) lo = ge = mid + 1; else hi = mid; }
    int64_t next = ge;
    if (next == L) next -= 1;
    p->next_line_id = next; p->prev_line_id = next - 1;
    trace_vpacket_volley(x, p);
    track_boundary(x, p, -1, 0);
    while (p->status == ST_IN_PROCESS && !x->error) {
        const int64_t s = p->current_shell_id;
        const double opacity_electron = m->electron_density[s] * x->c->sigma_thomson;
        int itype; int64_t delta;
        const double distance = trace_packet(x, p, opacity_electron, &itype, &delta);
        move_r_packet(x, p, distance);
        if (itype == IT_BOUNDARY) {
            track_boundary(x, p, s, s + delta);
            move_packet_across_shell_boundary(&p->current_shell_id, &p->status, delta, m->n_shells);
        } else if (itype == IT_LINE) {
            track_before(x, p, IT_LINE);
            line_scatter_event(x, p);
            track_after(x, p, IT_LINE);
            x->cnt.n_line_events++;
            trace_vpacket_volley(x, p);
        } else {
            track_before(x, p, IT_ESCATTERING);
            thomson_scatter(x, p);
            track_after(x, p, IT_ESCATTERING);
            x->cnt.n_escat_events++;
            trace_vpacket_volley(x, p);
        }
    }
    track_boundary(x, p, p->current_shell_id, p->current_shell_id + 1);
}

}  // namespace

extern "C" {

/* One Monte Carlo iteration of the nonhomologous mode.  Outputs must be zeroed by the caller; every output pointer
 * except output_nus / output_energies / j / nu_bar / j_blue / edotlu may be NULL. */
int nonhomologous_oracle_run(const tardis_oracle_model *m, const double *v_inner, const double *v_outer,
                             const tardis_oracle_config *c, const tardis_oracle_packets *pk, tardis_oracle_outputs *out) {
    Ctx x{};
    x.m = m; x.c = c; x.out = out; x.v_inner = v_inner; x.v_outer = v_outer;
    x.dvdr.resize((size_t)m->n_shells);
    for (int64_t s = 0; s < m->n_shells; s++) x.dvdr[s] = nh::velocity_gradient(m->r_inner[s], m->r_outer[s], v_inner[s], v_outer[s]);
    int64_t vlog_n = 0;
    for (int64_t i = 0; i < pk->n_packets && !x.error; i++) {
        Packet p{};
        p.r = pk->initial_radii[i]; p.mu = pk->initial_mus[i]; p.nu = pk->initial_nus[i]; p.energy = pk->initial_energies[i];
        p.current_shell_id = 0; p.status = ST_IN_PROCESS; p.index = i;
        x.rng.seed((uint32_t)(pk->packet_seeds[i] & 0xffffffffLL));
        x.trk = Tracker{};
        x.trk.radius = x.trk.before_nu = x.trk.before_mu = x.trk.before_energy = NAN;
        x.trk.after_nu = x.trk.after_mu = x.trk.after_energy = NAN;
        x.trk.shell_id = -1; x.trk.interaction_type = -1; x.trk.line_absorb_id = -1; x.trk.line_emit_id = -1;
        x.trk.boundary_buffer = -1;  /* the first track_boundary(-1, 0) makes it 0 */
        x.ev = nullptr; x.ev_cap = 0; x.ev_n = 0;
        if (out->events && i < out->n_tracked_packets) { x.ev = out->events + i * out->max_events_per_packet; x.ev_cap = out->max_events_per_packet; }
        x.vp_nu.clear(); x.vp_energy.clear(); x.vp_mu.clear(); x.vp_r.clear();
        packet_propagation(&x, &p);
        x.cnt.n_rng_draws += x.rng.draws;
        out->output_nus[i] = p.nu;
        out->output_energies[i] = (p.status == ST_REABSORBED) ? -p.energy : (p.status == ST_EMITTED ? p.energy : -99.0);
        if (out->event_counts && i < out->n_tracked_packets) out->event_counts[i] = x.ev_n;
        if (out->last_interaction_type) {
            out->last_interaction_type[i] = x.trk.interaction_type; out->last_event_id[i] = x.trk.interactions_count;
            out->last_shell_id[i] = x.trk.shell_id; out->last_line_absorb_id[i] = x.trk.line_absorb_id;
            out->last_line_emit_id[i] = x.trk.line_emit_id; out->last_radius[i] = x.trk.radius;
            out->last_before_nu[i] = x.trk.before_nu; out->last_before_mu[i] = x.trk.before_mu;
            out->last_before_energy[i] = x.trk.before_energy; out->last_after_nu[i] = x.trk.after_nu;
            out->last_after_mu[i] = x.trk.after_mu; out->last_after_energy[i] = x.trk.after_energy;
        }
        /* add_vpacket_collection_to_histogram (montecarlo_transport.py:166-195) + the virtual-packet log */
        for (size_t k = 0; k < x.vp_nu.size(); k++) {
            if (out->vhist && c->n_grid > 1) {
                const double *grid = c->spectrum_frequency_grid;
                const double nu = x.vp_nu[k];
                if (!((nu < grid[0]) || (nu > grid[c->n_grid - 1]))) out->vhist[(int64_t)floor((nu - grid[0]) / (grid[1] - grid[0]))] += x.vp_energy[k];
            }
            if (out->vlog_nus && vlog_n < out->vlog_capacity) {
                out->vlog_nus[vlog_n] = x.vp_nu[k]; out->vlog_energies[vlog_n] = x.vp_energy[k];
                out->vlog_initial_mus[vlog_n] = x.vp_mu[k]; out->vlog_initial_rs[vlog_n] = x.vp_r[k];
                out->vlog_packet_index[vlog_n] = i;
            }
            vlog_n++;
        }
    }
    out->vlog_count = vlog_n;
    out->counters = x.cnt;
    return x.error;
}

double nonhomologous_oracle_velocity_gradient(double r_inner, double r_outer, double v_inner, double v_outer) {
    return nh::velocity_gradient(r_inner, r_outer, v_inner, v_outer);
}

}  // extern "C"
