// nonhomologous.cuh -- the nonhomologous transport mode (piecewise-linear velocity law, time_explosion unused).
//
// What it replaces (paths relative to the reference's tardis/ package):
//   depressed_quartic                        transport/montecarlo/nonhomologous_grid.py:9-86
//   calculate_distance_line_nonhomologous    transport/geometry/calculate_distances.py:115-194
//   packet_propagation (nonhomologous)       transport/montecarlo/modes/nonhomologous/packet_propagation.py:53-263
//   trace_packet (nonhomologous)             transport/montecarlo/modes/nonhomologous/rad_packet_transport.py:25-198
//   thomson_scatter / line_emission / line_scatter_event
//                                            modes/nonhomologous/interaction_events.py:183-262,
//                                            modes/nonhomologous/interaction_event_callers.py:27-93,189-239
//   trace_vpacket_within_shell / trace_vpacket / trace_vpacket_volley
//                                            modes/nonhomologous/virtual_packet.py:83-378
//
// Part 1 (host and device): the line distance.  The quartic the reference solves is badly conditioned: one ulp of the
// packet frequency moves a root by up to 1e-2 relative in the tail of the distribution.  So the device kernel and the CPU
// oracle must evaluate it with the SAME operations: this part is compiled by both (nvcc with -fmad=false, g++ with
// -ffp-contract=off) and uses only IEEE + - * / and sqrt.  The libm functions of the cube-root step (hypot, pow, atan2,
// cos, sin) are restated here on top of those, because CUDA's and glibc's differ by ulps.
//
// Part 2 (device only): the nonhomologous device functions and transport_nonhomologous_kernel, one packet per lane.
#pragma once
#include <cmath>
#include <cstring>

#if defined(__CUDACC__)
#define NH_HD __host__ __device__ __forceinline__
#else
#define NH_HD inline
#endif

namespace nh {

constexpr double C_LIGHT = 2.99792458e10;       // configuration/constants.py:5
constexpr double MISS_DISTANCE = 1e99;          // configuration/constants.py:6
constexpr double RESONANCE_WINDOW = 1e-14;      // calculate_distances.py:179
constexpr double QUARTIC_THRESHOLD = 6.0e-7;    // nonhomologous_grid.py:10 threshold_fac
constexpr double PI = 3.141592653589793;

NH_HD long long bits_of(double x) {
#if defined(__CUDA_ARCH__)
    return __double_as_longlong(x);
#else
    long long b; std::memcpy(&b, &x, 8); return b;
#endif
}
NH_HD double from_bits(long long b) {
#if defined(__CUDA_ARCH__)
    return __longlong_as_double(b);
#else
    double x; std::memcpy(&x, &b, 8); return x;
#endif
}
NH_HD double quiet_nan() { return from_bits(0x7ff8000000000000ll); }
NH_HD bool is_nan(double x) { return x != x; }
NH_HD double fabs_(double x) { return from_bits(bits_of(x) & 0x7fffffffffffffffll); }
NH_HD double pow2_of(int k) { return from_bits((long long)(k + 1023) << 52); }  // 2^k, -1022 <= k <= 1023

// x ** (1./3.) for x > 0 (the magnitude step of the complex power, and the real power of the u == 0 branch).
// x = m 2^(3k) with m in [1, 8); Newton's iteration for the cube root of m from a linear guess.  The exponent 1./3. is
// 1/3 - 1.85e-17, so pow(x, 1./3.) = cbrt(x) (1 - 1.85e-17 ln x): up to 1.3e-14 relative at the ends of the double range,
// so the correction is applied (ln x needs three digits only).
constexpr double THIRD_DEFECT = 1.850371707708594e-17;  // 1/3 - (double)(1./3.)
NH_HD double cbrt_pos(double x) {
    int pre = 0;
    if (x < 1e-290) { x = x * pow2_of(180); pre = -60; }             // subnormal / tiny: scale into the normal range
    const int e = (int)((bits_of(x) >> 52) & 0x7ff) - 1023;
    const int k = e >= 0 ? e / 3 : -((-e + 2) / 3);                  // floor(e / 3)
    const double m = x * pow2_of(-k) * pow2_of(-k) * pow2_of(-k);    // exact: [1, 8)
    double y = 0.7 + 0.3 * m;                                        // within 30 % of m^(1/3) on [1, 8)
    for (int i = 0; i < 7; i++) y = y - (y * y * y - m) / (3.0 * y * y);
    const double z = (y - 1.0) / (y + 1.0), z2 = z * z;              // ln y = 2 atanh z, z <= 1/3
    const double ln_x = 3.0 * (2.0 * z * (1.0 + z2 * (1.0 / 3.0 + z2 * (0.2 + z2 / 7.0)))) +
                        3.0 * (double)(k + pre) * 0.6931471805599453;
    y = y - y * (THIRD_DEFECT * ln_x);
    return y * pow2_of(k + pre);
}
NH_HD double real_pow_third(double q) {  // q ** (1.0 / 3.0) with numpy's error model: NaN for q < 0
    if (q > 0.0) return cbrt_pos(q);
    if (q == 0.0) return 0.0;
    return quiet_nan();
}
NH_HD double hypot_(double x, double y) {
    x = fabs_(x); y = fabs_(y);
    if (y == 0.0) return x;
    if (x == 0.0) return y;
    const double big = x > y ? x : y, small = x > y ? y : x;
    const double t = small / big;
    return big * sqrt(1.0 + t * t);
}
// atan(t) for 0 <= t <= 1: two angle halvings (atan t = 2 atan(t / (1 + sqrt(1 + t^2)))) bring t below tan(pi / 16), then
// the Taylor series to z^29
NH_HD double atan_unit(double t) {
    for (int i = 0; i < 2; i++) t = t / (1.0 + sqrt(1.0 + t * t));
    const double z2 = t * t;
    double s = 0.0;
    for (int n = 14; n >= 1; n--) s = z2 * ((n & 1 ? -1.0 : 1.0) / (2 * n + 1) + s);
    return 4.0 * (t + t * s);
}
NH_HD double atan2_(double y, double x) {
    if (is_nan(x) || is_nan(y)) return quiet_nan();
    const double ax = fabs_(x), ay = fabs_(y);
    const bool neg_y = bits_of(y) < 0;
    double a;
    if (ay == 0.0) a = (bits_of(x) < 0) ? PI : 0.0;
    else if (ax == 0.0) a = 0.5 * PI;
    else if (ay <= ax) { a = atan_unit(ay / ax); if (bits_of(x) < 0) a = PI - a; }
    else { a = 0.5 * PI - atan_unit(ax / ay); if (bits_of(x) < 0) a = PI - a; }
    return neg_y ? -a : a;
}
// sin / cos of |x| <= pi: Taylor series to x^27 / x^28 (the phase of a cube root lies in [-pi/3, pi/3])
NH_HD double sin_(double x) {
    const double x2 = x * x;
    double s = 0.0;
    for (int n = 13; n >= 1; n--) s = -x2 / ((2.0 * n) * (2.0 * n + 1.0)) * (1.0 + s);
    return x + x * s;
}
NH_HD double cos_(double x) {
    const double x2 = x * x;
    double s = 0.0;
    for (int n = 14; n >= 1; n--) s = -x2 / ((2.0 * n - 1.0) * (2.0 * n)) * (1.0 + s);
    return 1.0 + s;
}

struct Roots { double x[4]; };

// nonhomologous_grid.py:9-86, in the reference's operation order.  x**2.0 / x**3.0 / x**4.0 are x*x, (x*x)*x and
// (x*x)*(x*x) (what LLVM makes of pow with a small integral exponent).  Complex steps as CPython / Numba define them:
//   np.sqrt(t + 0j)        (sqrt(t), +0) for t >= 0, (+0, sqrt(-t)) for t < 0 (cmath's algorithm is exact there)
//   r ** (1/3)             _Py_c_pow: |r| = hypot, len = |r| ** (1/3), phase = atan2(im, re) * (1/3), len (cos, sin)
//                          -- the principal branch, so a negative real r gives a complex u
//   p / (3 u)              Smith's division of complex(p, 0) by complex(3 u.re, 3 u.im)
NH_HD Roots depressed_quartic(double A, double B, double C, double D, double E) {
    const double A2 = A * A, A3 = A2 * A, A4 = A2 * A2;
    const double B2 = B * B, B3 = B2 * B, B4 = B2 * B2;
    const double a = -3.0 * B2 / (8.0 * A2) + C / A;
    const double b = B3 / (8.0 * A3) - B * C / (2.0 * A2) + D / A;
    const double c = -3.0 * B4 / (256.0 * A4) + C * B2 / (16.0 * A3) - B * D / (4.0 * A2) + E / A;

    const double a2 = a * a, a3 = a2 * a;
    const double p = -a2 / 12.0 - c;
    const double q = -a3 / 108.0 + a * c / 3.0 - b * b / 8.0;

    const double q2p3 = q * q / 4.0 + (p * p * p) / 27.0;
    double s_re, s_im;  // np.sqrt(q2p3 + 0j)
    if (q2p3 >= 0.0) { s_re = sqrt(q2p3); s_im = 0.0; }
    else if (q2p3 < 0.0) { s_re = 0.0; s_im = sqrt(-q2p3); }
    else { s_re = quiet_nan(); s_im = quiet_nan(); }
    const double r_re = -q / 2 + s_re, r_im = 0.0 + s_im;

    double u_re = 0.0, u_im = 0.0;  // r ** (1/3)
    if (!(r_re == 0.0 && r_im == 0.0)) {
        const double third = 1. / 3.;
        const double vabs = hypot_(r_re, r_im);
        const double len = is_nan(vabs) ? vabs : (vabs > 0.0 ? cbrt_pos(vabs) : 0.0);
        const double phase = atan2_(r_im, r_re) * third;
        u_re = len * cos_(phase);
        u_im = len * sin_(phase);
    }
    double y;
    if (u_re == 0.0 && u_im == 0.0) {
        y = -5.0 / 6.0 * a - real_pow_third(q);
    } else {
        // p / (3.0 * u)
        const double br = 3.0 * u_re, bi = 3.0 * u_im, ar = p, ai = 0.0;
        double d_re;
        if (fabs_(br) >= fabs_(bi)) {
            if (br == 0.0) d_re = quiet_nan();
            else { const double ratio = bi / br; const double denom = br + bi * ratio; d_re = (ar + ai * ratio) / denom; }
        } else {
            const double ratio = br / bi; const double denom = br * ratio + bi; d_re = (ar * ratio + ai) / denom;
        }
        y = (-5.0 / 6.0 * a + u_re) - d_re;
    }
    const double w = sqrt(a + 2.0 * y);
    double thresh = fabs_(3.0 * a);
    const double t2 = fabs_(2.0 * y), t3 = fabs_(2.0 * b / w);
    if (t2 > thresh) thresh = t2;
    if (t3 > thresh) thresh = t3;
    thresh = QUARTIC_THRESHOLD * thresh;

    double term[2], cl[2];
    term[0] = -(3.0 * a + 2.0 * y + 2.0 * b / w);
    term[1] = -(3.0 * a + 2.0 * y - 2.0 * b / w);
    for (int i = 0; i < 2; i++) {
        cl[i] = term[i];
        if (fabs_(cl[i]) <= thresh) cl[i] = 0.0;
        else if (cl[i] < 0.0) cl[i] = quiet_nan();
    }
    if (is_nan(cl[0]) && is_nan(cl[1])) {  // no real roots: force the smaller term to zero
        const int k = (fabs_(term[0]) <= fabs_(term[1])) ? 0 : 1;
        cl[k] = 0.0;
    }
    const double shift = -B / (4.0 * A);
    Roots R;
    R.x[0] = shift + 0.5 * (w + sqrt(cl[0]));
    R.x[1] = shift + 0.5 * (w - sqrt(cl[0]));
    R.x[2] = shift + 0.5 * (-w + sqrt(cl[1]));
    R.x[3] = shift + 0.5 * (-w - sqrt(cl[1]));
    return R;
}

// calculate_distance_line_nonhomologous, calculate_distances.py:115-194.  v = get_velocity(r, shell) and
// dvdr = velocity_gradient[shell] are the caller's (the same expressions everywhere: velocity()).
NH_HD double distance_line(double r, double mu, double nu, double nu_line, double r_inner, double r_outer, double v_inner,
                           double v_outer, double dvdr, double v) {
    const double n = C_LIGHT * (1 - nu_line / nu);
    const double m = dvdr;
    const double p = 1.0 - mu * mu;
    const double q = v_outer - m * r_outer;
    const double r0 = r_outer - r_inner;
    const double v0 = v_outer - v_inner;
    if (v0 == 0.0) return MISS_DISTANCE;
    const double rd = r / r0, nd = n / v0, md = 1.0, qd = q / v0;
    const double md2 = md * md, rd2 = rd * rd, nd2 = nd * nd, qd2 = qd * qd;
    const double a = md2;
    const double b = -2.0 * nd * md;
    const double c = nd2 + md * rd2 * p - qd2;
    const double d = -2.0 * nd * md * rd2 * p;
    const double e = nd2 * rd2 * p;
    const double beta = v / C_LIGHT;
    const double doppler = 1.0 - mu * beta;
    const double comov_nu = nu * doppler;
    double distance = MISS_DISTANCE;
    if ((comov_nu - nu_line > RESONANCE_WINDOW * nu_line && m > 0.0) || (comov_nu - nu_line < -RESONANCE_WINDOW * nu_line && m < 0.0)) {
        const Roots x = depressed_quartic(a, b, c, d, e);
        for (int i = 0; i < 4; i++) {
            if (is_nan(x.x[i])) continue;
            const double dc = r0 * x.x[i] - r * mu;
            if (dc > 0.0 && dc < distance) distance = dc;
        }
    }
    return distance;
}

// NumbaRadial1DGeometry (model/geometry/radial1d.py:342-375)
NH_HD double velocity_gradient(double r_inner, double r_outer, double v_inner, double v_outer) {
    return (v_outer - v_inner) / (r_outer - r_inner);
}
NH_HD double velocity(double r, double r_inner, double v_inner, double dvdr) { return v_inner + dvdr * (r - r_inner); }

}  // namespace nh

// ==========================================================================================================================
// Part 2: device functions and the kernel (nvcc only).  Reused from transport_kernel.cuh, as they do not depend on the
// velocity law: Rng, Lane, the trackers and event log, boundary / finish bookkeeping, the counters, the bulk replicas and
// the macro-atom walk.  Everything that evaluates a velocity is written here, as the reference writes it separately.
// ==========================================================================================================================
#if defined(__CUDACC__)
#include "transport_kernel.cuh"

namespace nh {
using tb::cP;
using tb::Counters;
using tb::KParams;
using tb::Lane;
using tb::Rng;

// RPacket plus the prev_line_id of this mode: where a backward (decelerating-shell) line scan starts.  line_emission sets
// next_line only, so prev_line can be stale; the reference's later backward scans start from it as it is.
struct NhPacket {
    Lane p;
    int prev_line;
};

// NumbaRadial1DGeometry.get_velocity (radial1d.py:359-375)
__device__ __forceinline__ double vel_at(double r, int s) {
    const KParams &P = cP;
    return velocity(r, P.r_inner[s], P.v_inner[s], P.dvdr[s]);
}

// calculate_distance_line_nonhomologous for a packet at (r, mu, nu) in shell s (out of line: the quartic is the largest
// block of code in the kernel, and both the trace and the virtual packets call it)
__device__ __noinline__ double line_distance(double r, double mu, double nu, int s, double nu_line) {
    const KParams &P = cP;
    const double r_in = P.r_inner[s], v_in = P.v_inner[s], dvdr = P.dvdr[s];
    return distance_line(r, mu, nu, nu_line, r_in, P.r_outer[s], v_in, P.v_outer[s], dvdr, velocity(r, r_in, v_in, dvdr));
}

// range(start, lim, dir) of the two-way line scan: forward (dvdr >= 0) from next_line to the end of the list, backward
// from prev_line to line 0.  `last` is Python's loop variable after a loop that ran to its end (for-else), including
// the adjustment of rad_packet_transport.py:178-191 / virtual_packet.py:156-163; `ran` says whether the range was empty.
__device__ __forceinline__ int scan_exhausted_index(bool forward, int start, bool ran) {
    const int L = cP.n_lines;
    if (forward) return ran ? L : start;         // last = L - 1 -> L; empty: the start itself (>= L)
    return ran ? -1 : start;                     // last = 0 -> -1; empty: the start itself (<= -1)
}
__device__ __forceinline__ void set_line_ids(NhPacket &q, bool forward, int cur) {
    if (forward) { q.p.next_line = cur; q.prev_line = cur - 1; }
    else { q.p.next_line = cur + 1; q.prev_line = cur; }
}

// trace_vpacket (virtual_packet.py:189-253) of one virtual packet, with trace_vpacket_within_shell (:83-186) inline.
// Returns the tau the reference multiplies the energy by at the end; *energy carries the Russian roulette.
__device__ __noinline__ double trace_vpacket(double v_r, double v_mu, double v_nu, double &v_energy, int v_shell, int v_next,
                                             Rng &rng, unsigned long long &n_vsteps) {
    const KParams &P = cP;
    const int L = P.n_lines;
    int v_prev = v_next - 1;
    int status = tb::ST_IN_PROCESS;
    double tau_total = 0.0;
    int guard = 0;
    while (true) {
        int delta_shell;
        const double d_b = tb::distance_boundary(v_r, v_mu, P.r_inner[v_shell], P.r_outer[v_shell], delta_shell);
        const double chi_e = P.n_e[v_shell] * P.sigma_thomson;
        double tau_comb = chi_e * d_b;
        const bool forward = P.dvdr[v_shell] >= 0.0;
        const int start = forward ? v_next : v_prev;
        int cur = start;
        bool broke = false;
        for (; forward ? cur < L : cur > -1; cur += forward ? 1 : -1) {
            const double d_line = line_distance(v_r, v_mu, v_nu, v_shell, P.nu_line[cur]);
            n_vsteps++;
            if (d_b <= d_line) { broke = true; break; }
            tau_comb += P.tau_t[(size_t)v_shell * P.lpad + cur];
        }
        if (!broke) cur = scan_exhausted_index(forward, start, cur != start);
        if (forward) { v_next = cur; v_prev = cur - 1; } else { v_next = cur + 1; v_prev = cur; }
        tau_total += tau_comb;
        const int next_shell = v_shell + delta_shell;  // move_packet_across_shell_boundary, movement.py:80-102
        if (next_shell >= P.n_shells) status = tb::ST_EMITTED;
        else if (next_shell < 0) status = tb::ST_REABSORBED;
        else v_shell = next_shell;
        if (tau_total > P.tau_russian) {
            const double event_random = rng.next_double();
            if (event_random > P.survival_probability) { v_energy = 0.0; status = tb::ST_EMITTED; }
            else { v_energy = v_energy / P.survival_probability * exp(-tau_total); tau_total = 0.0; }
        }
        const double new_r = sqrt(v_r * v_r + d_b * d_b + 2.0 * v_r * d_b * v_mu);
        v_mu = (v_mu * v_r + d_b) / new_r;
        v_r = new_r;
        if (status == tb::ST_EMITTED) break;
        if (++guard > 4 * P.n_shells + 64) { atomicMax(P.error, tb::ERR_VPACKET_LOOP); break; }
    }
    return tau_total;
}

// trace_vpacket_volley, virtual_packet.py:257-378 (partial relativity only)
__device__ __noinline__ void vpacket_volley(const Lane &p, Rng &rng, unsigned long long &n_vp, unsigned long long &n_vsteps) {
    const KParams &P = cP;
    if ((p.nu < P.spawn_start) || (p.nu > P.spawn_end)) return;
    const int nv = P.n_vpackets;
    if (nv == 0) return;
    double mu_min;
    bool on_inner;
    if (p.r > P.r_inner[0]) {
        const double q = P.r_inner[0] / p.r;
        mu_min = -sqrt(1 - q * q);
        on_inner = false;
    } else {
        on_inner = true;
        mu_min = 0.0;
    }
    const double mu_bin = (1.0 - mu_min) / nv;
    const double v = vel_at(p.r, p.shell);
    const double rp_doppler = tb::doppler_factor<false>(v, p.mu);
    for (int i = 0; i < nv; i++) {
        const double v_mu = mu_min + i * mu_bin + rng.next_double() * mu_bin;
        const double weight = on_inner ? 2 * v_mu / nv : (1 - mu_min) / (2 * nv);
        const double v_doppler = tb::doppler_factor<false>(v, v_mu);
        const double ratio = rp_doppler / v_doppler;
        const double v_nu = p.nu * ratio;
        double v_energy = p.energy * weight * ratio;
        const double tau = trace_vpacket(p.r, v_mu, v_nu, v_energy, p.shell, p.next_line, rng, n_vsteps);
        v_energy *= exp(-tau);
        n_vp++;
        tb::record_vpacket(v_nu, v_energy, v_mu, p.r, p.pid);
    }
}

// packet_propagation.py:101-108: set_packet_props_partial_relativity at get_velocity and the first line id of packet pid,
// written into its StartRecord by the ordering pass (tb::order_scatter_kernel / tb::start_record_kernel)
struct NhStart {
    __device__ __forceinline__ static tb::StartRecord at(long long pid, long long seed64) {
        const KParams &P = cP;
        tb::StartRecord s;
        s.pid = (int)pid;
        s.r = P.in_r[pid]; s.mu = P.in_mu[pid]; s.nu = P.in_nu[pid]; s.energy = P.in_energy[pid];
        const uint2 sx = tb::seed_expand(seed64);
        s.seed = sx.x; s.x397 = sx.y;
        const double v = vel_at(s.r, 0);
        const double inv_doppler = tb::inverse_doppler_factor<false>(v, s.mu);
        s.nu *= inv_doppler; s.energy *= inv_doppler;
        // L - searchsorted(nu[::-1], comov_nu, 'left') == #lines with nu_line >= comov_nu
        int next = tb::first_line_below(s.nu * tb::doppler_factor<false>(v, s.mu));
        if (next == P.n_lines) next -= 1;
        s.next_line = next;
        return s;
    }
};

// packet_propagation.py:101-126 for the packet at processing slot `slot`: its StartRecord, the second line id, the
// tracker, the first volley and the synthetic boundary event -1 -> 0
__device__ __noinline__ void start_packet(NhPacket &q, Rng &rng, long long slot, Counters &c) {
    const KParams &P = cP;
    Lane &p = q.p;
    const int pid = tb::start_from_record(p, rng, slot);
    q.prev_line = p.next_line - 1;
    if (P.last_type) {  // TrackerLastInteraction.__init__, tracker_last_interaction.py:55-82
        const double qnan = __longlong_as_double(0x7ff8000000000000ll);
        P.last_type[pid] = -1; P.last_event_id[pid] = 0; P.last_shell[pid] = -1;
        P.last_absorb[pid] = -1; P.last_emit[pid] = -1;
        P.last_radius[pid] = qnan; P.last_before_nu[pid] = qnan; P.last_before_mu[pid] = qnan;
        P.last_before_energy[pid] = qnan; P.last_after_nu[pid] = qnan; P.last_after_mu[pid] = qnan;
        P.last_after_energy[pid] = qnan;
    }
    if (P.n_vpackets > 0) vpacket_volley(p, rng, c.vp, c.vsteps);
    tb::log_boundary(p, -1, 0);
    c.boundary++;
}

// trace_packet, rad_packet_transport.py:25-198.  Returns the distance; itype / delta_shell as the reference's tuple.
__device__ __forceinline__ double trace_packet(NhPacket &q, Rng &rng, double chi_e, int &itype, int &delta_shell, Counters &c) {
    const KParams &P = cP;
    const int L = P.n_lines;
    Lane &p = q.p;
    const int s = p.shell;
    const double r_in = P.r_inner[s], v_in = P.v_inner[s], dvdr = P.dvdr[s];
    const double d_b = tb::distance_boundary(p.r, p.mu, r_in, P.r_outer[s], delta_shell);
    const double tau_event = -log(rng.next_double());
    double tau_line_comb = 0.0;
    const bool forward = dvdr >= 0.0;
    const int start = forward ? p.next_line : q.prev_line;
    const double *tau_row = P.tau_t + (size_t)s * P.lpad;
    double *jb_row = P.jblue_t + (size_t)s * P.lpad;
    double *ed_row = P.edotlu_t + (size_t)s * P.lpad;
    double d_e = tau_event / chi_e;
    int cur = start;
    for (; forward ? cur < L : cur > -1; cur += forward ? 1 : -1) {
        tau_line_comb += tau_row[cur];
        const double d_t = line_distance(p.r, p.mu, p.nu, s, P.nu_line[cur]);
        const double tau_trace_comb = tau_line_comb + chi_e * d_t;
        double d = d_t;  // min(distance_trace, distance_boundary, distance_electron)
        if (d_b < d) d = d_b;
        if (d_e < d) d = d_e;
        if (d_t != 0) {
            if (d == d_b || d == d_e) set_line_ids(q, forward, cur);
            if (d == d_b) { itype = tb::IT_BOUNDARY; return d; }
            if (d == d_e) { itype = tb::IT_ESCATTERING; return d; }
        }
        // the estimator update at the resonance point (:141-163)
        const double new_r = sqrt(p.r * p.r + d_t * d_t + 2.0 * p.r * d_t * p.mu);
        const double new_mu = (p.mu * p.r + d_t) / new_r;
        const double new_v = v_in + dvdr * (new_r - r_in);
        const double energy = p.energy * (1.0 - new_v / C_LIGHT * new_mu);
        tb::red_f64(&jb_row[cur], energy / p.nu);
        tb::red_f64(&ed_row[cur], energy);
        c.line_steps++;
        if (tau_trace_comb > tau_event && !P.disable_line) {
            itype = tb::IT_LINE;
            p.next_line = cur; q.prev_line = cur - 1;
            return d_t;
        }
        d_e = (tau_event - tau_line_comb) / chi_e;
    }
    set_line_ids(q, forward, scan_exhausted_index(forward, start, cur != start));
    if (d_e < d_b) { itype = tb::IT_ESCATTERING; return d_e; }
    itype = tb::IT_BOUNDARY;
    return d_b;
}

// move_r_packet (movement.py:30-76) at get_velocity + update_estimators_bulk into the warp's replica
__device__ __forceinline__ void move_packet(Lane &p, double distance) {
    const KParams &P = cP;
    if (++p.nsteps > tb::MAX_EVENTS_PER_PACKET) atomicMax(P.error, tb::ERR_STUCK);
    const double dop = tb::doppler_factor<false>(vel_at(p.r, p.shell), p.mu);
    const double r = p.r;
    if (distance > 0.0) {
        const double new_r = sqrt(r * r + distance * distance + 2.0 * r * distance * p.mu);
        p.mu = (p.mu * r + distance) / new_r;
        p.r = new_r;
        const double cnu = p.nu * dop, cen = p.energy * dop;
        double *rep = tb::bulk_replica();
        tb::red_f64(&rep[p.shell], cen * distance);
        tb::red_f64(&rep[P.n_shells + p.shell], cen * distance * cnu);
    }
}

// line_emission, interaction_event_callers.py:27-93: next_line only (prev_line stays)
__device__ __forceinline__ void line_emission(Lane &p, int emission_line_id) {
    const KParams &P = cP;
    const double inv_doppler = tb::inverse_doppler_factor<false>(vel_at(p.r, p.shell), p.mu);
    p.nu = P.nu_line[emission_line_id] * inv_doppler;
    p.next_line = emission_line_id + 1;
}

struct Emission {  // this mode's line_emission, as the emitter of the shared macro-atom walk
    __device__ __forceinline__ void operator()(Lane &p, int emission_line_id) const { line_emission(p, emission_line_id); }
};

// LINE / ESCATTERING branches of packet_propagation.py:171-236: line_scatter_event (interaction_event_callers.py:189-239)
// with the shared macro-atom walk, thomson_scatter (interaction_events.py:226-262), then the volley
__device__ __noinline__ void interaction_event(Lane &p, Rng &rng, int itype, Counters &c) {
    const KParams &P = cP;
    const double v = vel_at(p.r, p.shell);
    const double old_dop = tb::doppler_factor<false>(v, p.mu);
    if (itype == tb::IT_LINE) {
        if (P.last_type || P.events) tb::log_interaction_before(p, tb::IT_LINE);
        p.mu = 2.0 * rng.next_double() - 1.0;
        const double inv_new = tb::inverse_doppler_factor<false>(v, p.mu);
        const double cen = p.energy * old_dop;
        p.energy = cen * inv_new;
        if (P.line_mode == 0) {
            line_emission(p, p.next_line);
        } else {
            const double cnu = p.nu * old_dop;
            p.nu = cnu * inv_new;
            tb::macro_atom_event<false, Emission>(p, rng, P.macro_entry[p.next_line], c.jumps, c.scanned);
        }
        tb::log_interaction_after(p, tb::IT_LINE);
        c.line_ev++;
    } else {
        if (P.last_type || P.events) tb::log_interaction_before(p, tb::IT_ESCATTERING);
        const double cnu = p.nu * old_dop, cen = p.energy * old_dop;
        p.mu = 2.0 * rng.next_double() - 1.0;
        const double inv_new = tb::inverse_doppler_factor<false>(v, p.mu);
        p.nu = cnu * inv_new;
        p.energy = cen * inv_new;
        tb::log_interaction_after(p, tb::IT_ESCATTERING);
        c.escat_ev++;
    }
    if (P.n_vpackets > 0) vpacket_volley(p, rng, c.vp, c.vsteps);
}

// Persistent, one packet per lane: each lane takes the next packet from the global counter when its packet ends.  The
// trace is a sequence of quartic solves (fp64-bound), so lanes are not regrouped; nothing here assumes homology.
__global__ void __launch_bounds__(256, 2) transport_nonhomologous_kernel() {
    const KParams &P = cP;
    Counters c;
    Rng rng;
    rng.start(0u, 0u, 0u);
    rng.ring = threadIdx.x & 31;
    while (*((volatile int *)P.error) == 0) {
        const unsigned long long slot = atomicAdd(P.next_packet, 1ull);
        if (slot >= (unsigned long long)P.n_packets) break;
        // The out-of-line calls get copies (the calling convention of transport_kernel.cuh): an object whose address
        // reaches a real call lives in local memory for its whole life.
        NhPacket q;
        {
            NhPacket lq; Rng lr = rng; Counters lc;
            start_packet(lq, lr, (long long)slot, lc);
            q = lq; rng = lr; tb::flush_rare(lc);
        }
        while (q.p.status == tb::ST_IN_PROCESS) {
            const double chi_e = P.n_e[q.p.shell] * P.sigma_thomson;  // chi_electron_calculator, opacities.py:50-67
            int itype = 0, delta_shell = 0;
            const double distance = trace_packet(q, rng, chi_e, itype, delta_shell, c);
            move_packet(q.p, distance);
            if (itype == tb::IT_BOUNDARY) {
                tb::boundary_event(q.p, delta_shell, c);
            } else {
                Lane lp = q.p; Rng lr = rng; Counters lc;
                interaction_event(lp, lr, itype, lc);
                q.p = lp; rng = lr; tb::flush_rare(lc);
            }
            if (*((volatile int *)P.error) != 0) break;
        }
        tb::finish_packet(q.p, rng, c);
    }
    tb::flush_block(c);
}

}  // namespace nh
#endif  // __CUDACC__
