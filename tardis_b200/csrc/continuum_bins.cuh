// continuum_bins.cuh -- bound-free opacity and bound-free estimators of the continuum (IIP) mode on GLOBAL frequency bins.
//
// What it replaces (paths relative to /root/reference/tardis/):
//   chi_bf_interpolator / chi_continuum_calculator   opacities/opacities.py:89-246
//   update_estimators_bound_free                      transport/montecarlo/estimators/radfield_estimator_calcs.py:57-124
//
// The reference evaluates, for every trace, a loop over ALL continua: threshold test, np.searchsorted in the
// continuum's phot_nus block, two linear interpolations (chi_bf and x_sect), and afterwards five estimator increments
// per active continuum.  On the synthetic config-5 model that is 12 active continua per trace: ~170 dependent memory
// operations and 62 floating-point reductions per trace.
//
// Both are piecewise linear in the comoving frequency between consecutive breakpoints of the UNION of all phot_nus
// blocks.  With B = sorted(phot_nus) and the bin g(nu) = #{B < nu} (so B[g-1] < nu <= B[g]):
//   * the set of active continua and each one's interpolation interval are constants of the bin, hence
//       chi_bf_tot(nu, shell) = C[shell][g] + D[shell][g] * (nu - B[g-1])         (one table entry per trace)
//   * the five bound-free estimators of continuum k are sums over traces of  f(E, d, nu) * xs_k(nu)  with
//     xs_k(nu) = X[k][g] + b[k][g] * (nu - B[g-1]), so a trace adds SEVEN moments to its (shell, bin) cell
//       {1, u, u dl, u dl^2, u z, u z dl, u z dl^2},  u = E d / nu,  dl = nu - B[g-1],  z = exp(-h nu / k T)
//     and continuum_finalize turns the moments of the bins inside each interpolation interval into
//     photo_ion / stim_recomb / bf_heating / stim_recomb_cooling / statistics of every (continuum, shell).
// A frequency that coincides exactly with a breakpoint (where the reference's index arithmetic wraps for the first
// point of a block) is not a bin-constant case: the kernels send it to the literal per-continuum path instead.
//
// Plain IEEE arithmetic shared by the kernels and the host (TBC_HD), unit-tested on a CPU build of this header
// (tests/continuum_bins_shim.cpp) against the literal per-continuum formulas.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define TBC_HD __host__ __device__ __forceinline__
#else
#define TBC_HD inline
#include <cmath>
#include <cstring>
#endif

namespace tbc {

constexpr int GUIDE_SHIFT = 44;   // guide key = sign, exponent and 8 mantissa bits of the binary64 pattern (256 keys per octave)
constexpr int N_MOMENTS = 8;      // 7 used, padded to 64 bytes per (shell, bin) cell

TBC_HD long long f64_bits(double x) {
#if defined(__CUDA_ARCH__)
    return __double_as_longlong(x);
#else
    long long b; memcpy(&b, &x, 8); return b;
#endif
}

struct BinView {
    const double *B;       // [n_phot] ascending union of all phot_nus
    const int *guide;      // [n_gkeys + 1]: guide[j] = #{B_i : key(B_i) < gkey_min + j}
    long long gkey_min;
    int n_gkeys, n_phot;
};

// g = #{B < nu} in [0, n_phot]; *tie = (g < n_phot && B[g] == nu)
TBC_HD int find_bin(const BinView &v, double nu, bool *tie) {
    int g, end;
    *tie = false;
    if (!(nu > 0.0)) return 0;
    const long long kb = (f64_bits(nu) >> GUIDE_SHIFT) - v.gkey_min;
    if (kb < 0) return 0;
    if (kb >= (long long)v.n_gkeys) return v.n_phot;
    g = v.guide[kb]; end = v.guide[kb + 1];
    while (g < end && v.B[g] < nu) g++;
    *tie = (g < v.n_phot) && (v.B[g] == nu);
    return g;
}

// number of points of block [start, start + n) whose position in B is < g (positions ascend inside a block)
TBC_HD int block_rank(const int *pos, int start, int n, int g) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (pos[start + mid] < g) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// {C, D} of one (shell, bin): value at the bin's left edge B[g-1] and slope of chi_bf_tot, summed over the continua in
// the reference's order (opacities/opacities.py:139-161 evaluated at the edge).  chi_row = chi_bf of this shell, [n_phot].
TBC_HD void bin_chi_linear(int g, const double *B, int n_phot, const double *phot_nus, const int *pos, const int *refs, int n_continua,
                           const double *chi_row, double *C, double *D) {
    double c = 0.0, d = 0.0;
    if (g >= 1 && g < n_phot) {
        const double nu_g = B[g - 1];
        for (int k = 0; k < n_continua; k++) {
            const int start = refs[k], n = refs[k + 1] - start;
            const int idx = block_rank(pos, start, n, g);
            if (idx < 1 || idx > n - 1) continue;  // bin outside [pn[0], pn[n-1]]
            const int lo = start + idx - 1, hi = start + idx;
            const double interval = phot_nus[hi] - phot_nus[lo];
            if (!(interval > 0.0)) continue;
            c += (chi_row[hi] * (nu_g - phot_nus[lo]) + chi_row[lo] * (phot_nus[hi] - nu_g)) / interval;
            d += (chi_row[hi] - chi_row[lo]) / interval;
        }
    }
    *C = c; *D = d;
}

// the seven moments a trace adds to its (shell, bin) cell
struct TraceMoments { double m[7]; };
TBC_HD TraceMoments trace_moments(double comov_nu, double comov_energy, double distance, double boltzmann_factor, double nu_left_edge) {
    TraceMoments t;
    const double u = comov_energy * distance / comov_nu;
    const double dl = comov_nu - nu_left_edge;
    const double ub = u * boltzmann_factor;
    t.m[0] = 1.0; t.m[1] = u; t.m[2] = u * dl; t.m[3] = u * dl * dl;
    t.m[4] = ub; t.m[5] = ub * dl; t.m[6] = ub * dl * dl;
    return t;
}

// moments [n_phot + 1][N_MOMENTS] of one shell -> the five estimators of continuum k in that shell (added to out[0..4]:
// photo_ion, stim_recomb, bf_heating, stim_recomb_cooling, statistics)
//   sum u xs                            = X M1 + b M2
//   bf_heating = sum E d xs (1 - thr / nu) = sum u (nu - thr) xs = e X M1 + (X + e b) M2 + b M3,   e = nu_g - thr, nu = nu_g + dl
TBC_HD void continuum_estimators_from_moments(int k, const double *mom_shell, const double *B, const double *phot_nus, const double *x_sect,
                                              const int *pos, const int *refs, double threshold_nu, double out[5]) {
    const int start = refs[k], n = refs[k + 1] - start;
    double pi = 0.0, sr = 0.0, heat = 0.0, cool = 0.0, stats = 0.0;
    for (int idx = 1; idx < n; idx++) {
        const int lo = start + idx - 1, hi = start + idx;
        const double interval = phot_nus[hi] - phot_nus[lo];
        if (!(interval > 0.0)) continue;
        const double b = (x_sect[hi] - x_sect[lo]) / interval;
        for (int g = pos[lo] + 1; g <= pos[hi]; g++) {
            const double *m = mom_shell + (size_t)g * N_MOMENTS;
            if (m[0] == 0.0) continue;
            const double nu_g = B[g - 1];
            const double X = (x_sect[hi] * (nu_g - phot_nus[lo]) + x_sect[lo] * (phot_nus[hi] - nu_g)) / interval;
            const double uxs = X * m[1] + b * m[2];
            const double uxs_b = X * m[4] + b * m[5];
            const double e = nu_g - threshold_nu;  // nu - thr = e + dl: no cancellation against thr * sum u xs
            pi += uxs; sr += uxs_b;
            heat += e * X * m[1] + (X + e * b) * m[2] + b * m[3];
            cool += e * X * m[4] + (X + e * b) * m[5] + b * m[6];
            stats += m[0];
        }
    }
    out[0] += pi; out[1] += sr; out[2] += heat; out[3] += cool; out[4] += stats;
}

}  // namespace tbc

// ---- host-side preparation (tb200_set_model and the CPU test shim) ----
#include <algorithm>
#include <numeric>
#include <vector>
namespace tbc {

struct HostBins {
    std::vector<double> B;     // [n_phot] ascending
    std::vector<int> pos;      // [n_phot] position of every phot_nus entry in B (stable: equal values keep their order)
    std::vector<int> guide;    // [n_gkeys + 1]
    long long gkey_min = 0;
    int n_gkeys = 0;
    // the continua active in bin g, in continuum order: act[2 i] = continuum k, act[2 i + 1] = phot_nus index of the lower
    // point of its interval, for i in [act_start[g], act_start[g + 1]).  For a frequency strictly inside the bin these are
    // exactly the continua and intervals the reference's threshold test and searchsorted select.
    std::vector<int> act_start;  // [n_phot + 2]
    std::vector<int> act;
    bool usable = false;       // false: the tables do not have the structure the bins assume -> literal path for every trace
};

// pi_min / pi_max must be the first / last frequency of each block and the blocks strictly ascending
// (opacities/continuum/continuum_state.py:110-146); otherwise `usable` stays false.
inline HostBins build_bins(const double *phot_nus, int n_phot, const long long *refs, int n_continua, const double *pi_min,
                           const double *pi_max) {
    HostBins h;
    if (n_phot < 2 || n_continua < 1) return h;
    for (int k = 0; k < n_continua; k++) {
        const long long a = refs[k], b = refs[k + 1];
        if (a < 0 || b > n_phot || b - a < 2) return h;
        if (pi_min[k] != phot_nus[a] || pi_max[k] != phot_nus[b - 1]) return h;
        for (long long i = a + 1; i < b; i++) if (!(phot_nus[i] > phot_nus[i - 1])) return h;
    }
    for (int i = 0; i < n_phot; i++) if (!(phot_nus[i] > 0.0) || !(phot_nus[i] < 1e300)) return h;
    std::vector<int> order(n_phot);
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return phot_nus[a] < phot_nus[b]; });
    h.B.resize(n_phot); h.pos.resize(n_phot);
    for (int r = 0; r < n_phot; r++) { h.B[r] = phot_nus[order[r]]; h.pos[order[r]] = r; }
    const long long kmin = f64_bits(h.B.front()) >> GUIDE_SHIFT, kmax = f64_bits(h.B.back()) >> GUIDE_SHIFT;
    if (kmax - kmin + 1 > (1 << 22)) return h;
    h.gkey_min = kmin; h.n_gkeys = (int)(kmax - kmin + 1);
    h.guide.assign(h.n_gkeys + 1, n_phot);
    int r = 0;
    for (int j = 0; j <= h.n_gkeys; j++) {
        while (r < n_phot && (f64_bits(h.B[r]) >> GUIDE_SHIFT) < kmin + j) r++;
        h.guide[j] = r;
    }
    h.act_start.assign(n_phot + 2, 0);
    for (int g = 0; g <= n_phot; g++) {
        h.act_start[g] = (int)(h.act.size() / 2);
        if (g < 1 || g >= n_phot) continue;
        for (int k = 0; k < n_continua; k++) {  // bin_chi_linear's selection (the blocks ascend strictly)
            const int start = (int)refs[k], n = (int)(refs[k + 1] - refs[k]);
            const int idx = block_rank(h.pos.data(), start, n, g);
            if (idx >= 1 && idx <= n - 1) { h.act.push_back(k); h.act.push_back(start + idx - 1); }
        }
    }
    h.act_start[n_phot + 1] = (int)(h.act.size() / 2);
    h.usable = true;
    return h;
}

}  // namespace tbc
