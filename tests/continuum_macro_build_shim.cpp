// CPU build of tardis_b200/csrc/continuum_macro_build.cuh for tests/test_continuum_macro_build.py: the header's row
// function and normalisation, on [T, S] C-order tables.
#include <vector>

#include "../tardis_b200/csrc/continuum_macro_build.cuh"

extern "C" {
// p[t, s] for the continuum rows (line rows are left as given); tab: the nine tables concatenated, row (table, key) at
// (base[table] + key) * S; shell: [5][S] (n_e, ff, fb, coll exc, coll ion cooling rates)
void shim_continuum_rows(int T, int S, const long long *type, const long long *key, const double *energy, const long long *base,
                         const double *tab, const double *shell, double *p) {
    for (int t = 0; t < T; t++) {
        const int k = tbcm::row_table(type[t]);
        if (tbcm::is_line_row(type[t])) continue;
        for (int s = 0; s < S; s++) {
            const double rate = k >= 0 ? tab[(base[k] + key[t]) * S + s] : 0.0;
            p[(size_t)t * S + s] = tbcm::continuum_probability(type[t], rate, shell[s], energy[t], shell[(size_t)tbcm::cooling_rate(type[t]) * S + s]);
        }
    }
}
// normalize_transition_probabilities on p [T, S] in place, blocks [edges[b], edges[b + 1])
void shim_normalize(int T, int S, int n_blocks, const long long *edges, double *p) {
    std::vector<double> col((size_t)T);
    for (int s = 0; s < S; s++) {
        for (int t = 0; t < T; t++) col[(size_t)t] = p[(size_t)t * S + s];
        for (int b = 0; b < n_blocks; b++) tbcm::normalize_block(col.data(), (int)edges[b], (int)edges[b + 1]);
        for (int t = 0; t < T; t++) p[(size_t)t * S + s] = col[(size_t)t];
    }
}
}
