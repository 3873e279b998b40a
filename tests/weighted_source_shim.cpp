// CPU build of the weighted-source functions of tardis_b200/csrc/packet_source.cuh for tests/test_weighted_source.py: the
// SAME functions the CUDA kernels run, driven the way engine.cu's create_weighted_packets drives them -- members holding
// packet ranges, threads of `chunk` packets, leaf sums by "leaves that start in my range", the host combine walking the
// members.  Test harness only.
#include "../tardis_b200/csrc/packet_source.cuh"
#include <algorithm>
#include <vector>

namespace {
// the seed segment's rejected draws and the generator parameters (as packet_source_setup)
std::vector<uint64_t> setup(tbps::SourceParams &P, uint64_t seed, uint64_t n, uint32_t rng, double radius, double temperature_kb,
                            double h_planck, const double *l_array, int n_l, double l_coef) {
    using namespace tbps;
    P.origin = pcg64_from_seed(seed);
    P.n = n; P.rng_excl = rng + 1u; P.threshold = lemire_threshold(rng);
    std::vector<uint64_t> rej;
    for (int it = 0; it < 64; it++) {
        std::vector<uint64_t> found;
        const uint64_t n_raw = n + rej.size();
        for (uint64_t k0 = 0; k0 < n_raw; k0 += 4096) {
            uint64_t buf[4096];
            const int c = scan_chunk(P.origin, k0, std::min(n_raw, k0 + 4096), P.rng_excl, P.threshold, buf, 4096);
            found.insert(found.end(), buf, buf + c);
        }
        const bool settled = found.size() == rej.size();
        rej = found;
        if (settled) break;
    }
    std::sort(rej.begin(), rej.end());
    P.n_rej = (int)rej.size();
    P.dbl_start = (n + rej.size() + 1) / 2;
    P.l_array = l_array; P.n_l = n_l; P.l_coef = l_coef; P.k_b_t = temperature_kb; P.h_planck = h_planck;
    P.radius = radius; P.energy = 1.0 / (double)n;
    P.relativistic = 0; P.beta = 0.0;
    return rej;
}
}  // namespace

// bounds[0 .. G]: member g holds packets [bounds[g], bounds[g + 1]).  Outputs are whole-set arrays.  normalize = 0 leaves
// I(nu) in e.  sum_out: the combined sum; minmax_out: {min, max} of the Carter-Cashwell nus.
extern "C" int shim_weighted_packets(uint64_t seed, uint64_t n, uint32_t rng, double radius, double temperature, double k_boltzmann,
                                     double h_planck, double c_light, const double *l_array, int n_l, double l_coef, int G,
                                     const int64_t *bounds, uint64_t chunk, double *r, double *nu, double *mu, double *e, long long *seeds,
                                     int normalize, double *sum_out, double *minmax_out) {
    using namespace tbps;
    if (n == 0 || G < 1 || chunk < 1 || bounds[0] != 0 || (uint64_t)bounds[G] != n) return 1;
    SourceParams P;
    const std::vector<uint64_t> rej = setup(P, seed, n, rng, radius, k_boltzmann * temperature, h_planck, l_array, n_l, l_coef);
    P.rejected = rej.data();
    // pass 1: per member, per thread chunk
    bool first = true;
    double lo_nu = 0.0, hi_nu = 0.0;
    for (int g = 0; g < G; g++) {
        const uint64_t lo = (uint64_t)bounds[g], hi = (uint64_t)bounds[g + 1];
        if (lo == hi) continue;
        double mn = 1.0 / 0.0, mx = 0.0;
        for (uint64_t i0 = lo; i0 < hi; i0 += chunk) blackbody_nu_minmax(P, i0, std::min(hi, i0 + chunk), mn, mx);
        lo_nu = first || mn < lo_nu ? mn : lo_nu;
        hi_nu = first || mx > hi_nu ? mx : hi_nu;
        first = false;
    }
    WeightedParams W;
    W.nu_lo = lo_nu; W.nu_range = hi_nu - lo_nu;
    W.h_planck = h_planck; W.beta_rad = 1 / (k_boltzmann * temperature); W.coefficient = 2 * h_planck / (c_light * c_light);
    // pass 2: each member writes its own range (element i - lo of its arrays) and the leaves that start in it
    std::vector<std::vector<double>> slots((size_t)G);
    for (int g = 0; g < G; g++) {
        const uint64_t lo = (uint64_t)bounds[g], hi = (uint64_t)bounds[g + 1];
        if (lo == hi) continue;
        slots[(size_t)g].assign((size_t)(pw_slot(hi) - pw_slot(lo) + 1), -1.0);
        for (uint64_t a = lo; a < hi; a += chunk)
            weighted_fill_leaves(P, W, a, std::min(hi, a + chunk), lo, hi, r + lo, nu + lo, mu + lo, e + lo, seeds + lo,
                                 slots[(size_t)g].data(), pw_slot(lo));
    }
    int owner = 0;
    const double sum = pw_combine(0, n, [&](uint64_t s) {
        while ((int64_t)s >= bounds[owner + 1]) owner++;
        return slots[(size_t)owner][pw_slot(s) - pw_slot((uint64_t)bounds[owner])];
    });
    if (normalize)
        for (uint64_t i = 0; i < n; i++) e[i] = e[i] / sum;
    *sum_out = sum;
    minmax_out[0] = lo_nu; minmax_out[1] = hi_nu;
    return 0;
}

// the leaf of an n-element pairwise tree holding element p
extern "C" void shim_leaf_at(uint64_t n, uint64_t p, uint64_t *start, uint64_t *len) { tbps::pw_leaf_at(n, p, *start, *len); }

// a[0 .. n) summed as the device sums it: every leaf by pw_leaf_sum, the leaves along pw_combine
extern "C" double shim_pairwise_sum(const double *a, uint64_t n) {
    return tbps::pw_combine(0, n, [&](uint64_t s) {
        uint64_t start, len;
        tbps::pw_leaf_at(n, s, start, len);
        uint64_t i = start;
        auto next = [&]() { return a[i++]; };
        return tbps::pw_leaf_sum(len, next);
    });
}
