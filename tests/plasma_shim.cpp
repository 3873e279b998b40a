// CPU build of tardis_b200/csrc/plasma.cuh for tests/test_plasma.py: the SAME functions the CUDA kernels run, driven the way
// tb200_solve_plasma drives them -- per-shell state on the host, then the (level, shell), (ion, shell) loops, the n_e fixed
// point with a one-member team, the level populations and the J_blue table.  Test harness only.
#include "../tardis_b200/csrc/plasma.cuh"
#include "../tardis_b200/csrc/radfield.cuh"
#include "../tardis_b200/csrc/formal_integral.cuh"
#include <vector>

namespace {
struct SerialTeam {
    template <class F> void each(int n, F f) { for (int i = 0; i < n; i++) f(i); }
    void sync() {}
    bool any(bool v) { return v; }
    bool all(bool v) { return v; }
};
}  // namespace

// constants: k_b, h, m_e, c.  options: ionization (0 nebular), excitation (0 dilute-lte), radiative_rates_type (0, 1, 2).
// Returns the tbp::NeStatus; outputs as tb200_solve_plasma downloads them ([rows, S] C-order).
extern "C" int shim_plasma(int n_levels, int n_ions, int n_shells, int n_lines, const double *level_energy, const long long *level_ion,
                           const double *g, const unsigned char *meta, const long long *ion_z, const long long *ion_q, const double *chi,
                           const double *nd, int n_t, const double *zeta_t, const double *zeta, const double *t_rad, const double *w,
                           const double *nu, const int *options, double link, double delta_treatment, double departure_coefficient,
                           double chi_0, double threshold, const double *fixed_ne, const double *constants, double *ne, double *pop,
                           double *lnd, double *j_blues, int *passes) {
    const int S = n_shells;
    const tbp::Constants K{constants[0], constants[1], constants[2]};
    std::vector<tbp::Shell> sh((size_t)S);
    for (int s = 0; s < S; s++) {
        sh[(size_t)s] = tbp::shell_state(K, t_rad[s], w[s], link, departure_coefficient);
        if (n_t >= 2) {
            const tbfi::ShellWeights wt = tbfi::shell_weights(zeta_t, n_t, t_rad[s]);
            sh[(size_t)s].z_lo = wt.lo; sh[(size_t)s].z_w_lo = wt.w_lo; sh[(size_t)s].z_w_hi = wt.w_hi;
            sh[(size_t)s].z_out = t_rad[s] < zeta_t[0] || t_rad[s] > zeta_t[n_t - 1];
        }
    }
    std::vector<int> ion_first((size_t)n_ions + 1), element_first;
    for (int l = n_levels - 1; l >= 0; l--) ion_first[(size_t)level_ion[l]] = l;
    ion_first[(size_t)n_ions] = n_levels;
    std::vector<double> charge((size_t)n_ions);
    for (int i = 0; i < n_ions; i++) {
        if (i == 0 || ion_z[i] != ion_z[i - 1]) element_first.push_back(i);
        charge[(size_t)i] = (double)ion_q[i];
    }
    const int n_elements = (int)element_first.size();
    element_first.push_back(n_ions);
    for (long long i = 0; i < (long long)n_levels * S; i++) {
        const long long l = i / S;
        const int s = (int)(i % S);
        lnd[i] = tbp::boltzmann_factor(g[l], level_energy[l], sh[(size_t)s].beta_rad, sh[(size_t)s].w, options[1] == 0 && !meta[l]);
    }
    std::vector<double> z((size_t)n_ions * S), phi((size_t)n_ions * S), new_ne((size_t)S);
    for (long long i = 0; i < (long long)n_ions * S; i++) {
        const int ion = (int)(i / S), s = (int)(i % S);
        z[(size_t)i] = tbp::partition_function(lnd, ion_first[(size_t)ion], ion_first[(size_t)ion + 1], S, s);
    }
    for (long long i = 0; i < (long long)n_ions * S; i++) {
        const int ion = (int)(i / S), s = (int)(i % S);
        if (charge[(size_t)ion] == 0.0) { phi[(size_t)i] = 0.0; continue; }
        const tbp::Shell &h = sh[(size_t)s];
        double p = tbp::phi_lte(z[(size_t)i], z[(size_t)(i - S)], h.g_e, chi[ion], h.beta_rad);
        if (options[0] == 0)
            p = tbp::phi_nebular(h, p, tbp::zeta_value(h, zeta + (size_t)ion * n_t), tbp::radiation_field_correction(h, chi[ion], chi_0, delta_treatment));
        phi[(size_t)i] = p;
    }
    SerialTeam team;
    const tbp::NeStatus r = tbp::ne_fixed_point(team, phi.data(), nd, element_first.data(), n_elements, charge.data(), n_ions, S, threshold,
                                                fixed_ne, pop, ne, new_ne.data(), passes);
    if (r != tbp::NE_OK) return (int)r;
    for (long long i = 0; i < (long long)n_levels * S; i++) {
        const size_t c = (size_t)level_ion[i / S] * S + (size_t)(i % S);
        lnd[i] = tbp::level_population(lnd[i], z[c], pop[c]);
    }
    if (options[2] != 2) {
        tbr::Constants KR{};
        KR.k_b = constants[0]; KR.h = constants[1]; KR.c = constants[3];
        for (long long l = 0; l < n_lines; l++)
            for (int s = 0; s < S; s++)
                j_blues[l * S + s] = tbr::dilute_planck_intensity(KR, nu[l], t_rad[s], options[2] == 1 ? 1.0 : w[s]);
    }
    return 0;
}
