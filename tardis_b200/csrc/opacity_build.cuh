// opacity_build.cuh -- tau_Sobolev, beta_Sobolev and the macro-atom transition probabilities on the device
// (SURVEY.md §8f rank 3): the step immediately BEFORE the packet-propagation path in every iteration.
//
// What it replaces (paths relative to /root/reference/tardis/):
//   StimulatedEmissionFactor.calculate                 plasma/properties/radiative_properties.py:66-116
//   calculate_sobolev_line_opacity                     opacities/tau_sobolev.py:21-75
//     (nonhomologous mode: divided by the velocity gradient)  transport/montecarlo/modes/nonhomologous/tau_sobolev.py:21-75
//   numba_calculate_beta_sobolev                       opacities/tau_sobolev.py:77-88
//   probability_emission_down / _internal_down / _internal_up   opacities/macro_atom/macroatom_line_transitions.py:94-139,213-247,324-367
//   BoundBoundMacroAtomSolver.normalize_transition_probabilities / _solve_next_macroatom_iteration
//                                                      opacities/macro_atom/macroatom_solver.py:491-585,708-739
//   OpacityState.to_numba (the [L,S] / [T,S] host tables the reference then hands to the MC loop)  opacities/opacity_state.py:157-342
// Inputs per iteration: the level populations [n_levels, S] (5 MB at 3e4 levels) and the J_blue table -- which
// tb200_solve_radiation_field has just left in HBM.  The [L,S] tau table (80 MB) and the [T,S] probability table (240 MB)
// are produced where the transport kernels read them (shell-major) instead of being built by pandas and re-uploaded.
//
// Plain IEEE arithmetic in the reference's operation order, shared by the kernels and the host (TBO_HD) and unit-tested
// on a CPU build of this header (tests/opacity_build_shim.cpp).
#pragma once

#if defined(__CUDACC__)
#define TBO_HD __host__ __device__ __forceinline__
#else
#define TBO_HD inline
#include <cmath>
#endif

namespace tbo {

struct Constants {  // as the reference's modules compute them (tau_sobolev.py:9-18, macroatom_line_transitions.py:7-11)
    double sobolev_coefficient, c_einstein, c, h;
};

// StimulatedEmissionFactor.calculate, one (line, shell) cell
TBO_HD double stimulated_emission_factor(double n_lower, double n_upper, double g_lower, double g_upper, bool metastable_upper, bool nlte_line) {
    if (n_lower == 0.0) return 0.0;                                      // :88-94
    double s = 1 - ((g_lower * n_upper) / (g_upper * n_lower));
    if (s < -1.7976931348623157e308) s = 0.0;                            // np.isneginf, :97-99
    if (metastable_upper && s < 0) s = 0.0;                              // :100-102
    if (nlte_line && s < 0) s = 0.0;                                     // :103-115 (nlte_line is false when there are no NLTE species)
    return s;
}

// calculate_sobolev_line_opacity, one cell: ((((lambda f_lu) * COEFF) * t_exp) * stim) * n_lower
TBO_HD double tau_sobolev(const Constants &K, double wavelength_f_lu, double time_explosion, double stim, double n_lower) {
    return wavelength_f_lu * K.sobolev_coefficient * time_explosion * stim * n_lower;
}

// the nonhomologous mode's calculate_sobolev_line_opacity (transport/montecarlo/modes/nonhomologous/tau_sobolev.py:21-75),
// one cell: ((((lambda f_lu) * COEFF) / dvdr) * stim) * n_lower.  dvdr < 0 (a decelerating shell) gives tau < 0, as there;
// dvdr == 0 gives +-inf or NaN, which the build reports as the reference's ValueError.
TBO_HD double tau_sobolev_nonhomologous(const Constants &K, double wavelength_f_lu, double velocity_gradient, double stim, double n_lower) {
    return wavelength_f_lu * K.sobolev_coefficient / velocity_gradient * stim * n_lower;
}

// numba_calculate_beta_sobolev, one cell
TBO_HD double beta_sobolev(double tau) {
    if (tau > 1e3) return 1.0 / tau;          // tau ** -1
    if (tau < 1e-4) return 1 - 0.5 * tau;
    return (1 - exp(-tau)) / tau;
}

// raw transition probability of one macro-atom row in one shell
TBO_HD double raw_probability(const Constants &K, int transition_type, double beta, double nu, double f_ul, double f_lu, double e_lower,
                              double e_upper, double stim, double j_blue) {
    if (transition_type == -1) return beta * (2 * (nu * nu) * f_ul / (K.c * K.c) * (e_upper - e_lower)) * K.c_einstein;   // :356-367
    if (transition_type == 0) return beta * (2 * (nu * nu) * f_ul / (K.c * K.c) * e_lower) * K.c_einstein;                // :242-247
    return beta * (f_lu / (K.h * nu) * stim * j_blue * e_lower) * K.c_einstein;                                            // :129-139
}

}  // namespace tbo
