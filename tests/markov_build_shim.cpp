// CPU build of tardis_b200/csrc/markov_build.cuh for the unit tests (tests/test_markov_build.py): the SAME functions the
// CUDA kernels run, driven the way tb200_build_absorbing_markov drives them (assembly, Gauss-Jordan steps, column scaling,
// deactivation table).  Test harness only.  Returns -1, or k * S + s of the first failing pivot.
#include "../tardis_b200/csrc/markov_build.cuh"
#include <vector>

extern "C" long long shim_markov_build(int n_rows, int n_shells, int n_states, const double *p /* [T,S] */, const long long *type,
                                       const long long *dest, const long long *edges, double *X /* [S,n,n] */,
                                       double *deact /* [T,S] */) {
    const int S = n_shells, n = n_states;
    long long err = -1;
    std::vector<double> q((size_t)n), r((size_t)n), c((size_t)n);
    for (int s = 0; s < S; s++) {
        double *A = X + (size_t)s * n * n;
        for (int i = 0; i < n; i++) {
            double *row = A + (size_t)i * n;
            for (int j = 0; j < n; j++) row[j] = 0.0;
            q[i] = tbm::accumulate_row(edges[i], edges[i + 1], type, dest, [&](long long t) { return p[(size_t)t * S + s]; }, row);
            for (int j = 0; j < n; j++) row[j] = tbm::identity_minus(j == i, row[j]);
        }
        for (int k = 0; k < n; k++) {
            const double piv = A[(size_t)k * n + k];
            if (!tbm::pivot_ok(piv)) {
                const long long code = (long long)k * S + s;
                if (err < 0 || code < err) err = code;
                break;
            }
            for (int j = 0; j < n; j++) {
                r[j] = tbm::pivot_row(j, k, A[(size_t)k * n + j], 1.0 / piv);
                c[j] = A[(size_t)j * n + k];
            }
            for (int i = 0; i < n; i++)
                for (int j = 0; j < n; j++) A[(size_t)i * n + j] = tbm::gj_cell(i, j, k, A[(size_t)i * n + j], c[i], r[j]);
        }
        for (int i = 0; i < n; i++)
            for (int j = 0; j < n; j++) A[(size_t)i * n + j] = tbm::column_scale(A[(size_t)i * n + j], q[j]);
    }
    for (int b = 0; b < n; b++)
        for (int s = 0; s < S; s++) {
            double sum = 0.0, comp = 0.0;
            for (long long t = edges[b]; t < edges[b + 1]; t++) tbm::kahan_add(sum, comp, tbm::deactivating(type[t], p[(size_t)t * S + s]));
            for (long long t = edges[b]; t < edges[b + 1]; t++)
                deact[(size_t)t * S + s] = tbm::normalized(tbm::deactivating(type[t], p[(size_t)t * S + s]), sum);
        }
    return err;
}
