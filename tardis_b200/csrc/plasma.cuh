// plasma.cuh -- the classic plasma solved on the device: nebular / LTE ionisation, dilute-LTE / LTE level populations,
// the electron densities and the dilute black-body J_blue table the macro atom reads.
//
// Replaces, per iteration, what Simulation.advance_state hands to plasma.update (simulation/base.py:363-415, paths relative
// to the reference's tardis/) for the graphs without NLTE, helium NLTE or continuum-interaction species:
//   BetaRadiation / ElectronTemperature / BetaElectron / GElectron        plasma/properties/general.py:20-121
//   LevelBoltzmannFactorLTE / LevelBoltzmannFactorDiluteLTE              plasma/properties/partition_function.py:32-114
//   PartitionFunction (pandas' Kahan group sum, row order)               partition_function.py:337-353
//   PhiSahaLTE / PhiSahaNebular (zeta: scipy interp1d, NaN -> 1.0)        plasma/properties/ion_population.py:37-182
//   RadiationFieldCorrection                                             ion_population.py:185-258
//   IonNumberDensity (the n_e fixed point)                               ion_population.py:261-390
//   LevelNumberDensity                                                   plasma/properties/level_population.py:13-70
//   radiative_rates_type dilute-blackbody / blackbody                    simulation/base.py:378-401
//
// Every function is plain IEEE arithmetic in the reference's operation order (the library is built with -fmad=false), shared
// by the kernels in engine.cu and by tests/plasma_shim.cpp, which drives them with the kernels' loops on the CPU.
//
// Layout in HBM: levels are grouped by ion and ions by element, each in the reference's row order.  Every [rows, S] table
// (Boltzmann factors -- overwritten in place by the level populations --, partition functions, Phi, ion populations) is
// row-major with the shells contiguous, as the reference's frames hold them, so a download is one copy.
//
// The reference's axis-0 sums (number_density.sum, the sum of the cumulative products, the free electrons) run over
// Fortran-ordered .values of its frames, so numpy sums them pairwise down the rows; pairwise_sum restates that order.
//
// One deliberate deviation: the reference iterates n_e without a bound (it only warns above 100 iterations); the device stops
// after MAX_NE_ITERATIONS with the error it raises for a NaN n_e.
#pragma once
#include <cmath>

#include "markov_build.cuh"   // tbm::kahan_add: pandas' group_sum
#include "packet_source.cuh"  // tbps::pw_leaf_sum / pw_split: numpy's pairwise sum

#ifdef __CUDACC__
#define TBP_HD __host__ __device__ __forceinline__
#define TBP_HD_CALL __host__ __device__  // recursive, or calling a caller-supplied Team
#else
#define TBP_HD inline
#define TBP_HD_CALL inline
#endif

namespace tbp {

constexpr int MAX_NE_ITERATIONS = 1000;
constexpr double ION_ZERO_THRESHOLD = 1e-20;                  // ion_population.py:17
constexpr double CHI_0_CA_II = 1.9020591570241798e-11;        // RadiationFieldCorrection._set_chi_0, ion_population.py:211-215
constexpr double NE_CONVERGENCE_THRESHOLD = 0.05;             // ion_population.py:340
constexpr double DBL_MAX_ = 1.7976931348623157e308;

struct Constants {  // as the reference's modules take them from tardis.constants (cgs)
    double k_b, h, m_e;
};

// Everything the per-(row, shell) functions need of one shell, from its T_rad and W.
struct Shell {
    double t_rad, w, beta_rad, t_e, beta_e, g_e, factor_a;
    // zeta: interp1d's linear weights on the temperature grid; out = 1 outside the grid (interp1d's NaN, then 1.0)
    int z_lo, z_out;
    double z_w_lo, z_w_hi;
};

// departure_coefficient NaN: the reference's default 1 / W (ion_population.py:223-228)
TBP_HD Shell shell_state(const Constants &K, double t_rad, double w, double link_t_rad_t_electron, double departure_coefficient) {
    Shell s{};
    s.t_rad = t_rad; s.w = w;
    s.beta_rad = 1 / (K.k_b * t_rad);                                 // general.py:35-36
    s.t_e = t_rad * link_t_rad_t_electron;                            // general.py:101-102
    s.beta_e = 1 / (K.k_b * s.t_e);                                   // general.py:120-121
    s.g_e = pow((2 * M_PI * K.m_e / s.beta_rad) / (K.h * K.h), 1.5);  // general.py:52-56
    const double dep = departure_coefficient != departure_coefficient ? 1.0 / w : departure_coefficient;
    s.factor_a = s.t_e / (dep * w * t_rad);                           // ion_population.py:233
    return s;
}

// numpy's pairwise sum of n values taken in order from next() (pairwise_sum, numpy/_core/src/umath/loops_utils.h.src)
template <class Next> TBP_HD_CALL double pairwise_sum(unsigned long long n, Next &next) {
    if (n <= tbps::PW_BLOCK) return tbps::pw_leaf_sum(n, next);
    const unsigned long long n2 = tbps::pw_split(n);
    const double a = pairwise_sum(n2, next);
    return a + pairwise_sum(n - n2, next);
}

// number_density.sum(axis=0): the start of the fixed point
TBP_HD double total_number_density(const double *nd, int n_elements, int n_shells, int s) {
    int e = 0;
    auto next = [&]() { return nd[(size_t)(e++) * n_shells + s]; };
    return pairwise_sum((unsigned long long)n_elements, next);
}

// ---- per (level, shell) -----------------------------------------------------------------------------------------------
// g exp(E * -beta), times W for a non-metastable level of the dilute-LTE excitation (partition_function.py:50-60,107-114)
TBP_HD double boltzmann_factor(double g, double energy, double beta_rad, double w, bool dilute_non_metastable) {
    const double b = g * exp(energy * -beta_rad);
    return dilute_non_metastable ? b * w : b;
}

// ---- per (ion, shell) ---------------------------------------------------------------------------------------------------
// the partition function: the ion's levels [first, last) summed in row order with pandas' Kahan compensation
TBP_HD double partition_function(const double *lbf, long long first, long long last, int n_shells, int s) {
    double sum = 0.0, comp = 0.0;
    for (long long l = first; l < last; l++) tbm::kahan_add(sum, comp, lbf[l * n_shells + s]);
    return sum;
}

// Phi of ion j (charge >= 1) from ion j - 1: Z_j / Z_{j-1} * (2 g_e exp(chi * -beta))  (ion_population.py:66-86)
TBP_HD double phi_lte(double z_ion, double z_below, double g_e, double chi, double beta_rad) {
    return (z_ion / z_below) * ((2 * g_e) * exp(chi * -beta_rad));
}

// zeta of one ion at this shell's T_rad (ion_population.py:166-182): interp1d's w_hi * y_hi + w_lo * y_lo; NaN -> 1.0
TBP_HD double zeta_value(const Shell &sh, const double *zeta_row) {
    const double z = sh.z_out ? NAN : sh.z_w_hi * zeta_row[sh.z_lo + 1] + sh.z_w_lo * zeta_row[sh.z_lo];
    return z != z ? 1.0 : z;
}

// delta (ion_population.py:217-258); delta_treatment NaN: computed
TBP_HD double radiation_field_correction(const Shell &sh, double chi, double chi_0, double delta_treatment) {
    if (delta_treatment == delta_treatment) return delta_treatment;
    if (chi < chi_0) {
        const double d = 1 - exp(chi * sh.beta_rad - sh.beta_rad * chi_0);
        return d + sh.factor_a * exp(chi * sh.beta_rad - chi_0 * sh.beta_e);
    }
    return sh.factor_a * exp(chi * (sh.beta_rad - sh.beta_e));
}

// phi_lte * w * ((zeta * delta) + w * (1 - zeta)) * (t_e / t_rad) ** 0.5, left to right (ion_population.py:157-162; numpy
// evaluates ** 0.5 as sqrt)
TBP_HD double phi_nebular(const Shell &sh, double phi_lte_value, double zeta, double delta) {
    return phi_lte_value * sh.w * ((zeta * delta) + sh.w * (1 - zeta)) * sqrt(sh.t_e / sh.t_rad);
}

// ---- the n_e fixed point (IonNumberDensity.calculate_with_n_electron / calculate, ion_population.py:296-390) --------------
// np.nan_to_num(phi / n_e)
TBP_HD double phi_over_ne(double phi, double n_e) {
    const double x = phi / n_e;
    if (x != x) return 0.0;
    if (x > DBL_MAX_) return DBL_MAX_;
    if (x < -DBL_MAX_) return -DBL_MAX_;
    return x;
}

// The populations of one element's ions [first, last) in one shell: N_0 = N_elem / (1 + sum of the cumulative products of
// Phi / n_e), N_k = N_0 * product_k, then every population below the threshold set to 0.  phi rows are those of the ions
// (row `first` is not read).
TBP_HD void ion_populations(const double *phi, long long first, long long last, int n_shells, int s, double n_e, double n_element,
                            double threshold, double *pop) {
    double prod = 1.0;
    long long i = first + 1;
    auto next = [&]() { prod *= phi_over_ne(phi[(i++) * n_shells + s], n_e); return prod; };  // np.cumprod, row by row
    const double sum = pairwise_sum((unsigned long long)(last - first - 1), next);             // np.sum(axis=0)
    const double n0 = n_element / (1 + sum);
    pop[first * n_shells + s] = n0 < threshold ? 0.0 : n0;
    prod = 1.0;
    for (i = first + 1; i < last; i++) {
        prod *= phi_over_ne(phi[i * n_shells + s], n_e);
        const double n = n0 * prod;
        pop[i * n_shells + s] = n < threshold ? 0.0 : n;
    }
}

// new n_e = (N_ion * charge).sum(axis=0)
TBP_HD double electron_sum(const double *pop, const double *charge, long long n_ions, int n_shells, int s) {
    long long i = 0;
    auto next = [&]() { const double v = pop[i * n_shells + s] * charge[i]; i++; return v; };
    return pairwise_sum((unsigned long long)n_ions, next);
}

TBP_HD bool ne_converged(double new_n_e, double n_e) { return fabs(new_n_e - n_e) / n_e < NE_CONVERGENCE_THRESHOLD; }
TBP_HD double ne_next(double new_n_e, double n_e) { return 0.5 * (new_n_e + n_e); }

enum NeStatus { NE_OK = 0, NE_NAN = 1, NE_CAP = 2 };

// IonNumberDensity.calculate: the whole fixed point, for a Team that runs it -- one CTA on the device (engine.cu), plain loops
// on the CPU (tests/plasma_shim.cpp).  team.each(n, f) calls f(i) for i < n, each i on one member, with the same i -> member
// map on every call (so a member reads back the new_ne it wrote); team.sync() is a barrier; team.any / team.all reduce a
// member's flag over the team (and are barriers).  n_e starts at number_density.sum(axis=0), or is fixed_ne (no iteration).
// Every pass computes the populations at n_e; it stops when ALL shells satisfy |new - n_e| / n_e < 0.05, and returns the
// n_e those populations were computed with, not `new`; otherwise every shell gets n_e = (new + n_e) / 2.
// *passes = the number of population passes (the reference's n_electron_iterations; 0 with fixed n_e).
template <class Team>
TBP_HD_CALL NeStatus ne_fixed_point(Team &team, const double *phi, const double *nd, const int *element_first, int n_elements,
                                    const double *charge, int n_ions, int n_shells, double threshold, const double *fixed_ne,
                                    double *pop, double *ne, double *new_ne, int *passes) {
    team.each(n_shells, [&](int s) { ne[s] = fixed_ne ? fixed_ne[s] : total_number_density(nd, n_elements, n_shells, s); });
    team.sync();
    int it = 0;
    for (;;) {
        team.each(n_elements * n_shells, [&](int b) {
            const int e = b / n_shells, s = b % n_shells;
            ion_populations(phi, element_first[e], element_first[e + 1], n_shells, s, ne[s], nd[(size_t)e * n_shells + s], threshold, pop);
        });
        team.sync();
        it++;
        if (fixed_ne) { *passes = 0; return NE_OK; }
        bool nan = false, converged = true;
        team.each(n_shells, [&](int s) {
            const double v = electron_sum(pop, charge, n_ions, n_shells, s);
            new_ne[s] = v;
            nan |= v != v;
            converged &= ne_converged(v, ne[s]);
        });
        *passes = it;
        if (team.any(nan)) return NE_NAN;  // PlasmaIonizationError('n_electron just turned "nan" - aborting')
        if (team.all(converged)) return NE_OK;
        if (it >= MAX_NE_ITERATIONS) return NE_CAP;
        team.each(n_shells, [&](int s) { ne[s] = ne_next(new_ne[s], ne[s]); });
        team.sync();
    }
}

// ---- per (level, shell) -----------------------------------------------------------------------------------------------
// LevelNumberDensity: lbf / Z[ion] * N[ion]
TBP_HD double level_population(double lbf, double z_ion, double n_ion) { return lbf / z_ion * n_ion; }

}  // namespace tbp
