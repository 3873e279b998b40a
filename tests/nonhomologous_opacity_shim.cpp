// CPU build of tardis_b200/csrc/opacity_build.cuh in the nonhomologous mode, for tests/test_nonhomologous_opacity.py: the SAME
// functions opacity_line_nonhomologous_kernel and the row / normalisation kernels run, driven as tb200_build_opacity drives
// them, with tau divided by the per-shell velocity gradient.  Test harness only.
#include "../tardis_b200/csrc/opacity_build.cuh"
#include <cstdint>
#include <cstddef>

extern "C" void shim_opacity_build_nonhomologous(int n_lines, int n_shells, int n_rows, int n_blocks, const long long *lower,
                                                 const long long *upper, const double *g, const uint8_t *meta, const uint8_t *nlte,
                                                 const double *wfl, const double *f_lu, const double *f_ul, const double *e_lo,
                                                 const double *e_up, const double *nu, const long long *ttype, const long long *tline,
                                                 const long long *block_edge, const double *lnd, const double *j_blues,
                                                 const double *velocity_gradient /* [S] */, const double *constants /* sobolev, c_einstein, c, h */,
                                                 double *stim, double *tau, double *beta, double *raw, double *norm) {
    tbo::Constants K{constants[0], constants[1], constants[2], constants[3]};
    const int S = n_shells;
    for (int l = 0; l < n_lines; l++)
        for (int s = 0; s < S; s++) {
            const long long lo = lower[l], up = upper[l];
            const double n_lower = lnd[lo * S + s], n_upper = lnd[up * S + s];
            const size_t c = (size_t)l * S + s;
            stim[c] = tbo::stimulated_emission_factor(n_lower, n_upper, g[lo], g[up], meta[up] != 0, nlte[l] != 0);
            tau[c] = tbo::tau_sobolev_nonhomologous(K, wfl[l], velocity_gradient[s], stim[c], n_lower);
            beta[c] = tbo::beta_sobolev(tau[c]);
        }
    for (int t = 0; t < n_rows; t++)
        for (int s = 0; s < S; s++) {
            const long long l = tline[t];
            const size_t c = (size_t)l * S + s;
            raw[(size_t)t * S + s] = tbo::raw_probability(K, (int)ttype[t], beta[c], nu[l], f_ul[l], f_lu[l], e_lo[l], e_up[l], stim[c], j_blues[c]);
        }
    for (int b = 0; b < n_blocks; b++)
        for (int s = 0; s < S; s++) {
            double sum = 0.0;
            for (long long t = block_edge[b]; t < block_edge[b + 1]; t++) sum += raw[(size_t)t * S + s];
            for (long long t = block_edge[b]; t < block_edge[b + 1]; t++) {
                const double q = raw[(size_t)t * S + s] / sum;
                norm[(size_t)t * S + s] = std::isnan(q) ? 0.0 : q;
            }
        }
}
