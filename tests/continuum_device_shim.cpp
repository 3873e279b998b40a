// CPU build of tardis_b200/csrc/continuum_bins.cuh for tests/test_continuum_device.py: the harness of
// tests/continuum_bins_shim.cpp (shim_continuum_bins) plus the per-bin active lists the continuum event reads.
// Test harness only.
#include "continuum_bins_shim.cpp"

// HostBins::act_start [n_phot + 2] and HostBins::act (up to act_capacity ints) of the tables; returns the number of ints
// of act, or -1 where build_bins refuses the tables.
extern "C" long long shim_bin_actives(int n_phot, int n_continua, const double *phot_nus, const long long *refs, const double *pi_min,
                                      const double *pi_max, int *act_start, int *act, long long act_capacity) {
    using namespace tbc;
    const HostBins h = build_bins(phot_nus, n_phot, refs, n_continua, pi_min, pi_max);
    if (!h.usable) return -1;
    for (size_t i = 0; i < h.act_start.size(); i++) act_start[i] = h.act_start[i];
    for (size_t i = 0; i < h.act.size() && (long long)i < act_capacity; i++) act[i] = h.act[i];
    return (long long)h.act.size();
}
