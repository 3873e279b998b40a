// continuum_macro_build.cuh -- the continuum (IIP) macro atom's unnormalised transition probabilities and their
// normalisation, on the device: the host step of ContinuumMacroAtomSolver._solve_next_macroatom_iteration that feeds
// tb200_build_absorbing_markov (paths relative to /root/reference/tardis/):
//   the continuum rows        opacities/macro_atom/macroatom_solver.py:1533-1631, macroatom_continuum_transitions.py:10-816
//   the cooling block         normalize_cooling_block_by_rate_fractions, macroatom_solver.py:1817-1833
//   the normalisation         normalize_transition_probabilities, macroatom_solver.py:709-739
// The line rows (-1 / 0 / 1) are tbo::raw_probability of opacity_build.cuh, as in the other modes.
//
// Each continuum row is one or two IEEE multiplications in the reference's order, so the rows are bit for bit the
// reference's; which table and which energy a row reads (the reference's mix of .loc / .iloc / positional lookups) is
// resolved once on the host into a per-row (table, key, energy) map.  Shared by the kernels and by the CPU build of this
// header (tests/continuum_macro_build_shim.cpp).
#pragma once
#include "markov_build.cuh"

#if defined(__CUDACC__)
#define TBCM_HD __host__ __device__ __forceinline__
#else
#define TBCM_HD inline
#endif

namespace tbcm {

// The per-iteration tables a row reads, in the order of tb200_continuum_rates: six rate coefficients, then three cooling
// arrays.  Each is [key][S].
enum Table {
    PHOTOIONIZATION = 0,  // stim_recomb_corrected_photoionization_rate_coeff
    SPONT_RECOMB,         // spontaneous_recombination_coeff
    COLL_DEEXC,
    COLL_EXC,
    COLL_ION,
    COLL_RECOMB,
    FB_COOL,              // fb_cool_probs_arr.T
    COLL_EXC_COOL,        // coll_exc_cool_arr.T
    COLL_ION_COOL,        // coll_ion_cool_arr.T
    N_TABLES,
    NO_TABLE = -1,        // line rows and free-free cooling
    BAD_TYPE = -2
};

// The per-shell arrays besides the tables: [SHELL_ARRAYS][S]
enum ShellArray { N_E = 0, FF_COOL_RATE, FB_COOL_RATE, COLL_EXC_COOL_RATE, COLL_ION_COOL_RATE, SHELL_ARRAYS };

// MacroAtomTransitionType (transport/montecarlo/macro_atom.py:19-48) -> the table the row reads
TBCM_HD int row_table(long long type) {
    switch (type) {
        case -1: case 0: case 1: return NO_TABLE;   // BB_EMISSION, INTERNAL_DOWN, INTERNAL_UP
        case 2: return PHOTOIONIZATION;               // PHOTOIONIZATION_INTERNAL
        case 3: case -7: return SPONT_RECOMB;         // PHOTO_RECOMB_INTERNAL, PHOTO_RECOMB_EMISSION
        case 11: case 5: return COLL_DEEXC;           // COLL_DOWN_TO_K_PACKET, COLL_DOWN_INTERNAL
        case 4: return COLL_EXC;                      // COLL_UP_INTERNAL
        case 6: return COLL_ION;                      // COLL_ION_INTERNAL
        case 7: case 14: return COLL_RECOMB;          // COLL_RECOMB_INTERNAL, COLL_RECOMB_TO_K_PACKET
        case -21: return NO_TABLE;                    // FF_COOLING
        case -20: return FB_COOL;                     // FB_COOLING
        case 21: return COLL_EXC_COOL;                // COLL_EXC_COOL
        case 22: return COLL_ION_COOL;                // COLL_ION_COOL
        default: return BAD_TYPE;
    }
}
TBCM_HD bool is_line_row(long long type) { return type == -1 || type == 0 || type == 1; }
// the per-shell cooling rate that scales a cooling row (normalize_cooling_block_by_rate_fractions), or N_E
TBCM_HD int cooling_rate(long long type) {
    return type == -21 ? FF_COOL_RATE : type == -20 ? FB_COOL_RATE : type == 21 ? COLL_EXC_COOL_RATE : type == 22 ? COLL_ION_COOL_RATE : N_E;
}

// Unnormalised probability of one continuum row in one shell.  `rate` = table[key][s], `shell` = the shell array
// cooling_rate(type) names, at s.
TBCM_HD double continuum_probability(long long type, double rate, double n_e, double energy, double shell) {
    switch (type) {
        case 2: case 3: case -7: return rate * energy;                        // rate.multiply(energies, axis=0)
        case -21: return shell;                                               // probabilities[FF_COOLING] = ff_cool_rate
        case -20: case 21: case 22: return shell * rate;                      // cool_rate * cool_arr.T
        default: return rate * n_e * energy;                                  // (rate * n_e).multiply(energies, axis=0)
    }
}

// normalize_transition_probabilities on the rows [t0, t1) of one source block of one shell, in place:
// probabilities_df.div(groupby("source").transform("sum")), then NaN -> 0.  pandas' group_sum skips NaN addends
// (an infinite rate times a zero energy) and accumulates the others with Kahan compensation in row order.
TBCM_HD void normalize_block(double *p, int t0, int t1) {
    double sum = 0.0, comp = 0.0;
    for (int t = t0; t < t1; t++)
        if (p[t] == p[t]) tbm::kahan_add(sum, comp, p[t]);
    for (int t = t0; t < t1; t++) p[t] = tbm::normalized(p[t], sum);
}

}  // namespace tbcm
