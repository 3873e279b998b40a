// markov_build.cuh -- the continuum (IIP) macro atom's absorbing Markov chain, solved on the device.
//
// Replaces, per iteration, steps 2-3 of ContinuumMacroAtomSolver._solve_next_macroatom_iteration
// (opacities/macro_atom/macroatom_solver.py:1648-1662):
//   create_absorbing_probs (opacities/macro_atom/absorbing_markov_chain.py:19-134): per shell, Q = the internal rows
//   (transition_type >= 0) scattered into [n, n] with duplicate (source, destination) pairs summed, q_i = the sum of
//   row i of Q, and X = (I - Q)^-1 diag(1 - q) -- scipy's splu there, dense Gauss-Jordan here;
//   and the second normalize_transition_probabilities (macroatom_solver.py:709-739) of the deactivating rows, the
//   internal rows multiplied by 0 first: a pandas group-by sum per source block, which pandas accumulates with Kahan
//   compensation in row order, then p / sum with NaN -> 0.
//
// Why no pivoting.  For an absorbing chain Q >= 0, every row sum of Q is <= 1 and every state reaches a deactivation,
// so A = I - Q is a nonsingular M-matrix (Z-matrix with a non-negative inverse).  Gaussian elimination on an M-matrix
// without pivoting only meets positive pivots, and each Schur complement is again an M-matrix.  So off the diagonal the
// update a_ij - a_ik a_kj / a_kk subtracts a non-negative product from a non-positive number: it never cancels, and an
// entry is zero only where no path connects the two states.  The inverse block of Gauss-Jordan stays non-negative for
// the same reason.  Hence X is zero exactly where no path leads (the reference's sparse LU agrees, except that its
// permuted factors leave ~1e-16 roundoff in the rows of states whose probabilities are all zero, which are exactly the
// identity row here), and a pivot <= 0, infinite or
// NaN means the chain is not absorbing (splu raises "singular matrix" there): the build names the shell and the state.
//
// The arithmetic is in __host__ __device__ functions so that tests/markov_build_shim.cpp runs exactly what the kernels
// run.  No sum that reaches X or the deactivation table uses atomics: every cell is written by one thread, in a fixed
// order, so two builds are bit-identical.
#pragma once
#include <cmath>
#include <climits>

#ifdef __CUDACC__
#define TBM_HD __host__ __device__ __forceinline__
#else
#define TBM_HD inline
#endif

namespace tbm {

// Largest n solved by one CTA per shell with the matrix in shared memory (n^2 doubles + two work vectors: 129 KiB).
constexpr int SMEM_MAX_N = 128;

// ---- the deactivation table -------------------------------------------------------------------------------------
// pandas' group_sum (Kahan): y = v - c; t = sum + y; c = (t - sum) - y; a NaN compensation (an infinite addend) resets.
TBM_HD void kahan_add(double &sum, double &comp, double v) {
    const double y = v - comp;
    const double t = sum + y;
    comp = t - sum - y;
    if (comp != comp) comp = 0.0;
    sum = t;
}
// deactivating_probs[internal_mask] *= 0 (absorbing_markov_chain.py:128-129)
TBM_HD double deactivating(long long type, double p) { return type >= 0 ? p * 0.0 : p; }
// probabilities_df.div(group sum), then NaN -> 0 (macroatom_solver.py:731-737)
TBM_HD double normalized(double p, double sum) {
    const double q = p / sum;
    return q != q ? 0.0 : q;
}

// ---- assembly of A = I - Q, one row (= one source block) at a time ---------------------------------------------
// Row i of Q from the rows [t0, t1) of block i in row order: duplicates add up in row order; returns q_i.  `prob(t)`
// is the row's normalised probability in this shell.  a_row must be zero on entry.
template <class Index, class Prob>
TBM_HD double accumulate_row(long long t0, long long t1, const Index *type, const Index *dest, Prob prob, double *a_row) {
    double q = 0.0;
    for (long long t = t0; t < t1; t++) {
        if (type[t] < 0) continue;
        const double p = prob(t);
        a_row[dest[t]] += p;
        q += p;
    }
    return q;
}
// identity - Q: 1 - Q_ii on the diagonal, 0 - Q_ij elsewhere (0 - 0 is +0: no negative zeros in A)
TBM_HD double identity_minus(bool diagonal, double q_ij) { return diagonal ? 1.0 - q_ij : 0.0 - q_ij; }

// ---- Gauss-Jordan inversion in place, step k ---------------------------------------------------------------------
// A pivot that is not positive and finite makes the chain singular.
TBM_HD bool pivot_ok(double piv) { return piv > 0.0 && piv <= 1.7976931348623157e308; }
// Row k after the step: r_k = 1 / a_kk, r_j = a_kj / a_kk (as a_kj * r_k).
TBM_HD double pivot_row(int j, int k, double a_kj, double inv) { return j == k ? inv : a_kj * inv; }
// Every other row i: a_ij <- a_ij - a_ik r_j, where column k enters as 0 (so a_ik <- -a_ik / a_kk).  One rounding (fma):
// a zero a_ik or r_j leaves a_ij bit for bit.
TBM_HD double gj_update(int j, int k, double a_ij, double a_ik, double r_j) { return fma(-a_ik, r_j, j == k ? 0.0 : a_ij); }
// Whole cell: row k takes the pivot row, the others the update.
TBM_HD double gj_cell(int i, int j, int k, double a_ij, double a_ik, double r_j) {
    return i == k ? r_j : gj_update(j, k, a_ij, a_ik, r_j);
}

// X = A^-1 diag(1 - q): column j of the inverse times 1 - q_j (a state without deactivation gives a zero column).
TBM_HD double column_scale(double ainv_ij, double q_j) { return ainv_ij * (1.0 - q_j); }

}  // namespace tbm

#ifdef __CUDACC__
namespace tbm {

// Assembly, part 1 (A zeroed before): one thread per (shell, state) scatters the block's internal rows into row i of Q and
// sums q_i.  The thread owns the row, so the duplicate sums need no atomics; it touches only the row's non-zero cells.
__global__ void markov_assemble_kernel(const double *p_t, int tpad, const int *block_edge, const int *type, const int *dest,
                                       int n, int S, double *A, double *q) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= (long long)S * n) return;
    const int s = (int)(g / n), i = (int)(g % n);
    double *row = A + ((size_t)s * n + i) * n;
    const double *ps = p_t + (size_t)s * tpad;
    q[g] = accumulate_row((long long)block_edge[i], (long long)block_edge[i + 1], type, dest, [&](long long t) { return ps[t]; }, row);
}

// Assembly, part 2: Q -> I - Q, one thread per cell (coalesced).
__global__ void markov_identity_minus_kernel(double *A, int n, long long total) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= total) return;
    const long long cell = g % ((long long)n * n);
    A[g] = identity_minus(cell / n == cell % n, A[g]);
}

// Step k, part 1: the pivot row r and the pivot column c of every shell (read before part 2 overwrites them).
// err keeps the smallest k * S + s whose pivot failed: the first failing step, lowest shell.
__global__ void markov_pivot_kernel(const double *A, int n, int S, int k, double *r, double *c, int *err) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= (long long)S * n) return;
    const int s = (int)(g / n), j = (int)(g % n);
    const double *As = A + (size_t)s * n * n;
    const double piv = As[(size_t)k * n + k];
    if (j == k && !pivot_ok(piv)) atomicMin(err, k * S + s);
    r[g] = pivot_row(j, k, As[(size_t)k * n + j], 1.0 / piv);
    c[g] = As[(size_t)j * n + k];
}

// Step k, part 2: every cell of every shell.  Cells that the step leaves bit for bit (a_ik == 0 or r_j == 0) are
// neither read nor written.
__global__ void markov_update_kernel(double *A, int n, int k, const double *r, const double *c) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y, s = blockIdx.z;
    if (j >= n) return;
    const double *rs = r + (size_t)s * n;
    double *cell = A + ((size_t)s * n + i) * n + j;
    if (i == k) { *cell = rs[j]; return; }
    const double a_ik = c[(size_t)s * n + i], r_j = rs[j];
    if (j == k) { *cell = gj_update(j, k, 0.0, a_ik, r_j); return; }
    if (a_ik == 0.0 || r_j == 0.0) return;
    *cell = gj_update(j, k, *cell, a_ik, r_j);
}

// n <= SMEM_MAX_N: one CTA per shell runs all n steps on its matrix in shared memory, with the same cell function.
__global__ void markov_solve_smem_kernel(double *A, int n, int S, int *err) {
    extern __shared__ double sm[];
    double *a = sm, *r = sm + (size_t)n * n, *c = r + n;
    __shared__ int failed;
    const int s = blockIdx.x;
    double *As = A + (size_t)s * n * n;
    const int nn = n * n;
    for (int e = threadIdx.x; e < nn; e += blockDim.x) a[e] = As[e];
    if (threadIdx.x == 0) failed = 0;
    __syncthreads();
    for (int k = 0; k < n; k++) {
        const double piv = a[k * n + k];
        if (threadIdx.x == 0 && !pivot_ok(piv)) { atomicMin(err, k * S + s); failed = 1; }
        for (int j = threadIdx.x; j < n; j += blockDim.x) {
            r[j] = pivot_row(j, k, a[k * n + j], 1.0 / piv);
            c[j] = a[j * n + k];
        }
        __syncthreads();
        if (failed) break;
        for (int e = threadIdx.x; e < nn; e += blockDim.x) {
            const int i = e / n, j = e - i * n;
            a[e] = gj_cell(i, j, k, a[e], c[i], r[j]);
        }
        __syncthreads();
    }
    for (int e = threadIdx.x; e < nn; e += blockDim.x) As[e] = a[e];
}

// X = A^-1 diag(1 - q) in place (and into `keep`, the copy tb200_download_absorbing_markov reads, when given).
__global__ void markov_scale_kernel(double *A, const double *q, int n, int S, double *keep) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)S * n * n;
    if (g >= total) return;
    const int j = (int)(g % n), s = (int)(g / ((long long)n * n));
    const double x = column_scale(A[g], q[(size_t)s * n + j]);
    A[g] = x;
    if (keep) keep[g] = x;
}

// One thread per (shell, block): the deactivation table, shell-major like every transition table the kernels read.
__global__ void markov_deactivation_kernel(const double *p_t, int tpad, const int *block_edge, int n_blocks, const int *type, int S,
                                           double *out_t) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= (long long)S * n_blocks) return;
    const int s = (int)(g / n_blocks), b = (int)(g % n_blocks);
    const double *ps = p_t + (size_t)s * tpad;
    double *os = out_t + (size_t)s * tpad;
    const int t0 = block_edge[b], t1 = block_edge[b + 1];
    double sum = 0.0, comp = 0.0;
    for (int t = t0; t < t1; t++) kahan_add(sum, comp, deactivating(type[t], ps[t]));
    for (int t = t0; t < t1; t++) os[t] = normalized(deactivating(type[t], ps[t]), sum);
}

}  // namespace tbm
#endif
