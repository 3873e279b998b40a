// packet_source.cuh -- device-side packet source (SURVEY.md §8f rank 1).
//
// What it replaces (paths relative to /root/reference/tardis/transport/montecarlo/packet_source/):
//   BasePacketSource.create_packets          base.py:195-253   (reseed, seeds by rng.choice, radii, nus, mus, energies)
//   BlackBodySimpleSource.create_packet_nus  black_body.py:140-179  (Carter & Cashwell sampler as in Bjorkman & Wood 2001)
//   BlackBodySimpleSource.create_packet_mus  black_body.py:181-199  (mu = sqrt(xi))
//   .create_packet_radii / _energies         black_body.py:122-138, 201-219
// and the third-party arithmetic underneath, numpy's `default_rng` (numpy 2.x, not vendored in the reference):
//   SeedSequence (numpy/random/bit_generator.pyx: hashmix / mix / generate_state), PCG64 XSL-RR 128/64
//   (numpy/random/src/pcg64/pcg64.h), Generator.random (53-bit doubles), Generator.choice -> integers ->
//   buffered_bounded_lemire_uint32 (numpy/random/src/distributions/distributions.c).
//
// The stream is consumed in the reference's order: N bounded 32-bit draws (two per 64-bit step, low half first; a
// draw whose Lemire remainder falls below the threshold is redrawn), then 5 N doubles (xis[0..4], row-major), then N
// doubles (mus).  Every position of that stream can be reached directly: PCG64 is a 128-bit LCG, so the state after
// k steps is a closed form evaluated by square-and-multiply (pcg_advance).  One thread therefore produces a chunk of
// consecutive packets from seven independently positioned generators.
//
// Everything in this header is plain integer / IEEE arithmetic shared by the kernel and by the host (TB_HD), so the
// same functions can be unit-tested on a CPU build of this header (tests/packet_source_shim.cpp).
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define TB_HD __host__ __device__ __forceinline__
#else
#define TB_HD inline
#include <cmath>
#endif

namespace tbps {

typedef unsigned __int128 u128;

struct Pcg64 { u128 state, inc; };

// numpy/random/src/pcg64/pcg64.h: PCG_DEFAULT_MULTIPLIER_128
TB_HD u128 pcg_mult() { return ((u128)0x2360ED051FC65DA4ull << 64) | (u128)0x4385DF649FCCF645ull; }

TB_HD void pcg_step(Pcg64 &g) { g.state = g.state * pcg_mult() + g.inc; }

// pcg_output_xsl_rr_128_64
TB_HD uint64_t pcg_output(u128 s) {
    const uint64_t x = (uint64_t)(s >> 64) ^ (uint64_t)s;
    const unsigned r = (unsigned)(s >> 122);
    return (x >> r) | (x << ((64u - r) & 63u));
}

// pcg64_next64: step, then the output of the NEW state
TB_HD uint64_t pcg_next64(Pcg64 &g) { pcg_step(g); return pcg_output(g.state); }

// state after `delta` further steps (pcg_advance_lcg_128): acc_mult = a^delta, acc_plus = c (a^delta - 1)/(a - 1)
TB_HD void pcg_advance(Pcg64 &g, uint64_t delta) {
    u128 cur_mult = pcg_mult(), cur_plus = g.inc, acc_mult = 1, acc_plus = 0;
    while (delta > 0) {
        if (delta & 1) { acc_mult *= cur_mult; acc_plus = acc_plus * cur_mult + cur_plus; }
        cur_plus = (cur_mult + 1) * cur_plus;
        cur_mult *= cur_mult;
        delta >>= 1;
    }
    g.state = acc_mult * g.state + acc_plus;
}

// Generator.random: next_double = (next_uint64 >> 11) * (1 / 2^53)
TB_HD double u64_to_double(uint64_t v) { return (double)(v >> 11) * (1.0 / 9007199254740992.0); }

// ---- the 32-bit view of the stream (pcg64_next32): raw draw k is the low (k even) or high (k odd) half of step k/2 + 1
struct Raw32 {
    Pcg64 g;          // state after the 64-bit step that produced `cur`
    uint64_t cur;     // that step's output
    uint64_t k;       // index of the next raw draw
    // position the view so that next() returns raw draw k0
    TB_HD void seek(const Pcg64 &origin, uint64_t k0) {
        g = origin; k = k0;
        const uint64_t step = k0 >> 1;  // number of 64-bit steps completed before the one holding draw k0
        pcg_advance(g, step);
        cur = 0;
        if (k0 & 1) cur = pcg_next64(g);  // the step holding k0 has already been taken by draw k0 - 1
    }
    TB_HD uint32_t next() {
        uint32_t v;
        if ((k & 1) == 0) { cur = pcg_next64(g); v = (uint32_t)cur; }
        else v = (uint32_t)(cur >> 32);
        k++;
        return v;
    }
};

// buffered_bounded_lemire_uint32 (distributions.c) for rng_excl = rng + 1 != 0: the value, or a redraw request
TB_HD bool lemire_rejected(uint32_t x, uint32_t rng_excl, uint32_t threshold) {
    const uint32_t leftover = (uint32_t)((uint64_t)x * rng_excl);
    return leftover < threshold;  // (the reference tests `leftover < rng_excl` first; threshold < rng_excl always)
}
TB_HD uint32_t lemire_value(uint32_t x, uint32_t rng_excl) { return (uint32_t)(((uint64_t)x * rng_excl) >> 32); }
// threshold = (UINT32_MAX - rng) % rng_excl
TB_HD uint32_t lemire_threshold(uint32_t rng) { const uint32_t e = rng + 1u; return (0xFFFFFFFFu - rng) % e; }

// index of raw draw that yields bounded output i: i plus the number of rejected raw draws at or before it.
// rejected[0..n_rej) holds the ascending indices of all rejected raw draws below the end of the seed segment.
TB_HD uint64_t raw_index_of_output(uint64_t i, const uint64_t *rejected, int n_rej) {
    uint64_t raw = i;
    for (int j = 0; j < n_rej; j++) { if (rejected[j] <= raw) raw++; else break; }
    return raw;
}

// np.searchsorted(a, v) (side='left'): number of elements < v
TB_HD int searchsorted_left(const double *a, int n, double v) {
    int lo = 0, hi = n;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (a[mid] < v) lo = mid + 1; else hi = mid; }
    return lo;
}

// create_packet_nus, black_body.py:166-179:  l = searchsorted(l_array, xi0 * l_coef) + 1;  x = -log(xi1 xi2 xi3 xi4) / l;
// nu = x * (k_B T) / h.   `log` is the one transcendental: glibc / numexpr / CUDA libm agree to an ulp, hence the 1e-15
// tolerance of the parity tests for nu (everything else is exact).
TB_HD double blackbody_nu(double xi0, double xi1, double xi2, double xi3, double xi4, const double *l_array, int n_l, double l_coef,
                          double k_b_t, double h_planck) {
    const double l = (double)searchsorted_left(l_array, n_l, xi0 * l_coef) + 1.0;
    const double prod = ((xi1 * xi2) * xi3) * xi4;  // np.prod(xis[1:], 0)
    const double x = -log(prod) / l;
    return x * k_b_t / h_planck;
}

// ---- SeedSequence(entropy).generate_state(4, uint64) -> PCG64 (host only: a few dozen 32-bit operations) -------------
// numpy/random/bit_generator.pyx: SeedSequence.mix_entropy / generate_state, pool_size = 4; PCG64._seed_seq ->
// pcg64_set_seed(initstate = {s0 high, s1 low}, initseq = {s2 high, s3 low}) -> pcg_setseq_128_srandom_r.
inline Pcg64 pcg64_from_seed(uint64_t seed) {
    const uint32_t INIT_A = 0x43b0d7e5u, MULT_A = 0x931e8875u, INIT_B = 0x8b51f9ddu, MULT_B = 0x58f38dedu;
    const uint32_t MIX_L = 0xca01f9ddu, MIX_R = 0x4973f715u;
    uint32_t entropy[2];  // the seed as little-endian 32-bit words, without leading zero words (0 -> one zero word)
    int n_ent = 0;
    for (uint64_t s = seed; s != 0; s >>= 32) entropy[n_ent++] = (uint32_t)s;
    if (n_ent == 0) entropy[n_ent++] = 0u;
    uint32_t hash_const = INIT_A;
    auto hashmix = [&](uint32_t v) { v ^= hash_const; hash_const *= MULT_A; v *= hash_const; v ^= v >> 16; return v; };
    auto mix = [&](uint32_t x, uint32_t y) { uint32_t r = MIX_L * x - MIX_R * y; r ^= r >> 16; return r; };
    uint32_t pool[4];
    for (int i = 0; i < 4; i++) pool[i] = hashmix(i < n_ent ? entropy[i] : 0u);
    for (int i_src = 0; i_src < 4; i_src++)
        for (int i_dst = 0; i_dst < 4; i_dst++)
            if (i_src != i_dst) pool[i_dst] = mix(pool[i_dst], hashmix(pool[i_src]));
    uint32_t w[8];
    hash_const = INIT_B;
    for (int i = 0; i < 8; i++) {
        uint32_t d = pool[i % 4];
        d ^= hash_const; hash_const *= MULT_B; d *= hash_const; d ^= d >> 16;
        w[i] = d;
    }
    uint64_t s64[4];
    for (int i = 0; i < 4; i++) s64[i] = (uint64_t)w[2 * i] | ((uint64_t)w[2 * i + 1] << 32);
    const u128 initstate = ((u128)s64[0] << 64) | s64[1], initseq = ((u128)s64[2] << 64) | s64[3];
    Pcg64 g;
    g.state = 0; g.inc = (initseq << 1) | 1;
    pcg_step(g); g.state += initstate; pcg_step(g);
    return g;
}

// ---- one chunk of packets / raw draws: the kernel body, callable on the host for the unit tests --------------------
struct SourceParams {
    Pcg64 origin;              // generator right after seeding
    uint64_t n;                // packets
    uint32_t rng_excl, threshold;  // bounded draw: [0, rng_excl), Lemire threshold
    const uint64_t *rejected;  // ascending raw indices of rejected draws of the seed segment
    int n_rej;
    uint64_t dbl_start;        // 64-bit steps consumed by the seed segment = ceil((n + n_rej) / 2)
    const double *l_array;     // cumsum(arange(1, l_samples) ** -4), from the host (numpy's own pow)
    int n_l;
    double l_coef, k_b_t, h_planck, radius, energy;
    // BlackBodySimpleSourceRelativistic (packet_source/black_body_relativistic.py:120-177): mu = -beta + sqrt(beta^2 + 2 beta z + z);
    // `energy` then carries the (2 beta + 1) / (1 - beta^2) / gamma factor, computed by the caller in the reference's order
    int relativistic;
    double beta;
};

// packets [i0, i1): radii, nus, mus, energies, seeds (any output pointer may be null); packet i goes to element i - base
TB_HD void fill_chunk(const SourceParams &P, uint64_t i0, uint64_t i1, double *r, double *nu, double *mu, double *e, long long *seeds,
                      uint64_t base = 0) {
    Raw32 sr;
    sr.seek(P.origin, raw_index_of_output(i0, P.rejected, P.n_rej));
    Pcg64 gx[5], gm = P.origin;
    for (int j = 0; j < 5; j++) { gx[j] = P.origin; pcg_advance(gx[j], P.dbl_start + (uint64_t)j * P.n + i0); }
    pcg_advance(gm, P.dbl_start + 5ull * P.n + i0);
    for (uint64_t i = i0; i < i1; i++) {
        uint32_t x = sr.next();
        while (lemire_rejected(x, P.rng_excl, P.threshold)) x = sr.next();
        double xi[5];
        for (int j = 0; j < 5; j++) xi[j] = u64_to_double(pcg_next64(gx[j]));
        const double m = u64_to_double(pcg_next64(gm));
        const uint64_t k = i - base;
        if (seeds) seeds[k] = (long long)lemire_value(x, P.rng_excl);
        if (nu) nu[k] = blackbody_nu(xi[0], xi[1], xi[2], xi[3], xi[4], P.l_array, P.n_l, P.l_coef, P.k_b_t, P.h_planck);
        if (mu) mu[k] = P.relativistic ? -P.beta + sqrt(P.beta * P.beta + 2 * P.beta * m + m) : sqrt(m);
        if (r) r[k] = P.radius;
        if (e) e[k] = P.energy;
    }
}

// rejected raw draws among [k0, k1): writes up to max_found indices, returns how many there are
TB_HD int scan_chunk(const Pcg64 &origin, uint64_t k0, uint64_t k1, uint32_t rng_excl, uint32_t threshold, uint64_t *found, int max_found) {
    Raw32 sr;
    sr.seek(origin, k0);
    int c = 0;
    for (uint64_t k = k0; k < k1; k++) {
        if (lemire_rejected(sr.next(), rng_excl, threshold)) { if (c < max_found) found[c] = k; c++; }
    }
    return c;
}

// ---- BlackBodyWeightedSource (packet_source/black_body_weighted.py:9-108) ------------------------------------------
// The stream after the seed segment: 5 N doubles for the Carter-Cashwell nus, which only give their min and max; N
// doubles for rng.uniform(min, max, N) (numpy's random_uniform: lo + (hi - lo) * u); N doubles for the mus.  Energies
// are I(nu) / sum(I) with I = intensity_black_body(nu, T) (util/base.py:279-302) and the sum in numpy's pairwise order.
// Products and sums that numpy does not fuse are written as *_rn, so that nvcc cannot contract them into an FMA.
TB_HD double mul_rn(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
TB_HD double add_rn(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}

struct WeightedParams {
    double nu_lo, nu_range;  // min of the Carter-Cashwell nus, max - min (numpy forms the range once, as a double)
    double coefficient;      // 2 h / c**2
    double h_planck, beta_rad;  // beta_rad = 1 / (k_B T)
};

// coefficient * nu**3 / (exp(h * nu * beta_rad) - 1), evaluated left to right as numpy does.  pow and exp are the two
// transcendentals: CUDA's and numpy's differ by about an ulp.
TB_HD double blackbody_intensity(double nu, const WeightedParams &W) {
    const double num = mul_rn(W.coefficient, pow(nu, 3.0));
    const double den = add_rn(exp(mul_rn(mul_rn(W.h_planck, nu), W.beta_rad)), -1.0);
    return num / den;
}

// min and max of the Carter-Cashwell nus of packets [i0, i1), folded into mn / mx (nothing is stored)
TB_HD void blackbody_nu_minmax(const SourceParams &P, uint64_t i0, uint64_t i1, double &mn, double &mx) {
    Pcg64 gx[5];
    for (int j = 0; j < 5; j++) { gx[j] = P.origin; pcg_advance(gx[j], P.dbl_start + (uint64_t)j * P.n + i0); }
    for (uint64_t i = i0; i < i1; i++) {
        double xi[5];
        for (int j = 0; j < 5; j++) xi[j] = u64_to_double(pcg_next64(gx[j]));
        const double v = blackbody_nu(xi[0], xi[1], xi[2], xi[3], xi[4], P.l_array, P.n_l, P.l_coef, P.k_b_t, P.h_planck);
        mn = v < mn ? v : mn;
        mx = v > mx ? v : mx;
    }
}

// numpy's pairwise summation of a contiguous float64 array (pairwise_sum in numpy/_core/src/umath/loops_utils.h.src):
// a run of more than PW_BLOCK splits at n2 = n / 2 - (n / 2) % 8 and recurses; a run of 8 .. PW_BLOCK is summed by eight
// interleaved accumulators, combined as ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)), then its tail in order; a run
// shorter than 8 in order.  The runs where the recursion stops -- the leaves -- depend on N alone.  Every split point is
// a multiple of 8 and every leaf of an N > PW_BLOCK tree holds at least 64 elements, so start >> 6 names a leaf.
constexpr uint64_t PW_BLOCK = 128;
TB_HD uint64_t pw_split(uint64_t n) { const uint64_t n2 = n / 2; return n2 - n2 % 8; }
TB_HD uint64_t pw_slot(uint64_t start) { return start >> 6; }

// the leaf of an n-element tree that holds element p
TB_HD void pw_leaf_at(uint64_t n, uint64_t p, uint64_t &start, uint64_t &len) {
    uint64_t lo = 0;
    while (n > PW_BLOCK) {
        const uint64_t n2 = pw_split(n);
        if (p < lo + n2) n = n2;
        else { lo += n2; n -= n2; }
    }
    start = lo; len = n;
}

// The sum of an n-element tree from its leaf sums (leaf(start) -> that leaf's sum), along numpy's recursion.  Host only.
template <class LeafSum> inline double pw_combine(uint64_t lo, uint64_t n, const LeafSum &leaf) {
    if (n <= PW_BLOCK) return leaf(lo);
    const uint64_t n2 = pw_split(n);
    return pw_combine(lo, n2, leaf) + pw_combine(lo + n2, n - n2, leaf);
}

// One leaf of n elements, next() yielding them in order, summed as numpy sums it.  The eight accumulators rotate through
// r0 .. r7 (the element's accumulator is always r0), so they stay in registers.
template <class Next> TB_HD double pw_leaf_sum(uint64_t n, Next &next) {
    const uint64_t m = n < 8 ? 0 : n - n % 8;
    double r0 = 0, r1 = 0, r2 = 0, r3 = 0, r4 = 0, r5 = 0, r6 = 0, r7 = 0, res = -0.0;
    for (uint64_t q = 0; q < n; q++) {
        const double v = next();
        if (q < m) {
            const double t = q < 8 ? v : add_rn(r0, v);
            r0 = r1; r1 = r2; r2 = r3; r3 = r4; r4 = r5; r5 = r6; r6 = r7; r7 = t;
            if (q + 1 == m) res = add_rn(add_rn(add_rn(r0, r1), add_rn(r2, r3)), add_rn(add_rn(r4, r5), add_rn(r6, r7)));
        } else {
            res = add_rn(res, v);
        }
    }
    return res;
}

// The weighted source's packets one after the other from packet i: seed, nu = lo + range * u, mu = sqrt(u'), radius, and
// I(nu) in the energy slot (the caller divides by the sum).  Packet i is stored at element i - lo when lo <= i < hi.
struct WeightedStream {
    const SourceParams &P;
    const WeightedParams &W;
    uint64_t i, lo, hi;
    double *r, *nu, *mu, *e;
    long long *seeds;
    Raw32 sr;
    Pcg64 gu, gm;
    TB_HD WeightedStream(const SourceParams &P_, const WeightedParams &W_, uint64_t i0, uint64_t lo_, uint64_t hi_, double *r_, double *nu_,
                         double *mu_, double *e_, long long *seeds_)
        : P(P_), W(W_), i(i0), lo(lo_), hi(hi_), r(r_), nu(nu_), mu(mu_), e(e_), seeds(seeds_) {
        sr.seek(P.origin, raw_index_of_output(i0, P.rejected, P.n_rej));
        gu = P.origin; pcg_advance(gu, P.dbl_start + 5ull * P.n + i0);
        gm = P.origin; pcg_advance(gm, P.dbl_start + 6ull * P.n + i0);
    }
    TB_HD double operator()() {
        uint32_t x = sr.next();
        while (lemire_rejected(x, P.rng_excl, P.threshold)) x = sr.next();
        const double v = add_rn(W.nu_lo, mul_rn(W.nu_range, u64_to_double(pcg_next64(gu))));
        const double m = u64_to_double(pcg_next64(gm));
        const double I = blackbody_intensity(v, W);
        if (i >= lo && i < hi) {
            const uint64_t k = i - lo;
            if (seeds) seeds[k] = (long long)lemire_value(x, P.rng_excl);
            if (nu) nu[k] = v;
            if (mu) mu[k] = sqrt(m);
            if (r) r[k] = P.radius;
            if (e) e[k] = I;
        }
        i++;
        return I;
    }
};

// The leaves that start in [a, b), and when a == lo also the leaf holding packet lo: their packets in [lo, hi) are
// stored (element i - lo), and every leaf that starts at or after lo leaves its sum in slots[pw_slot(start) - slot_base].
// A leaf that runs past hi is generated to its end for its sum; those packets are not stored.
TB_HD void weighted_fill_leaves(const SourceParams &P, const WeightedParams &W, uint64_t a, uint64_t b, uint64_t lo, uint64_t hi,
                                double *r, double *nu, double *mu, double *e, long long *seeds, double *slots, uint64_t slot_base) {
    uint64_t s, len;
    pw_leaf_at(P.n, a, s, len);
    if (s < a && a != lo) {
        s += len;
        if (s >= b || s >= P.n) return;
        pw_leaf_at(P.n, s, s, len);
    }
    WeightedStream next(P, W, s, lo, hi, r, nu, mu, e, seeds);
    while (true) {
        const double sum = pw_leaf_sum(len, next);
        if (s >= lo && slots) slots[pw_slot(s) - slot_base] = sum;
        s += len;
        if (s >= b || s >= P.n) break;
        pw_leaf_at(P.n, s, s, len);
    }
}

}  // namespace tbps
