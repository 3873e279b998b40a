// group.cuh -- engine groups (tb200_group_* of include/tardis_b200.h): G ordinary engines, on one device or on several,
// driven from one host call.  Member g transports packets [g N / G, (g + 1) N / G) of the caller's set, one host thread
// per member; then one collective sums what the members accumulated and leaves the sum on every member.
//
// Exactness: every packet's trajectory depends only on its seed, and the line estimators are accumulated as int64
// fixed-point difference words whose sum does not depend on the order of the addends.  Summing those words (with the
// fixed-point scales of the WHOLE packet set imposed on every member) and finalizing them gives J_blue / Edotlu bit for bit
// what one engine computes over the same packets.  The rest of the estimator buffer is summed in f64 in member order.
// Included at the end of engine.cu: it needs tb200_engine's fields and run_pipelined / create_packets_range.
#include <chrono>
#include <memory>
#include <mutex>
#include <thread>
#include <type_traits>

namespace tbg {

constexpr int MAX_MEMBERS = 32;

struct SlicePtrs {
    const void *src[MAX_MEMBERS];  // the slice on every member, in member order (or its staged copy)
    void *dst[MAX_MEMBERS];        // where the sum goes: every member this owner can write directly
};

// Sums element pairs [0, n_pairs) of the n_src sources in source order and stores the sum to the n_dst destinations
// (16-byte loads and stores).  WORDS: 64-bit fixed-point words, wrapping integer adds.  Otherwise f64: the fixed order
// makes every member's copy the same bits.  Each pair is read and written by one thread, so a source may be a destination.
template <bool WORDS>
__global__ void __launch_bounds__(256) reduce_slice_kernel(const __grid_constant__ SlicePtrs p, int n_src, int n_dst, long long n_pairs) {
    using V = typename std::conditional<WORDS, ulonglong2, double2>::type;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_pairs; i += stride) {
        V acc = reinterpret_cast<const V *>(p.src[0])[i];
        for (int k = 1; k < n_src; k++) {
            const V v = reinterpret_cast<const V *>(p.src[k])[i];
            acc.x += v.x;
            acc.y += v.y;
        }
        for (int d = 0; d < n_dst; d++) reinterpret_cast<V *>(p.dst[d])[i] = acc;
    }
}

}  // namespace tbg

struct tb200_group {
    std::vector<tb200_engine *> m;
    std::vector<char> peer;                 // [G][G]: member a's device may access member b's memory (peer access enabled)
    int peer_access = 1;                    // 0: every slice another member holds is staged through cudaMemcpyPeerAsync
    std::vector<DBuf<unsigned char>> staging;  // per owner: staged copies of the slices it cannot read directly
    std::vector<char> fi_ran;               // members that integrated frequencies in the last tb200_group_formal_integral
    // One lock per device, shared by the members on it: the transport kernels read their parameters from one __constant__
    // block per device, so members on the same device transport one after the other (each fills the device anyway).
    std::vector<std::shared_ptr<std::mutex>> device_lock;
    double allreduce_ms = 0.0;
    bool allreduce_timed = false;
};

namespace {

int64_t shard_lo(int64_t n, int g, int G) { return n * g / G; }  // parallel.shard_bounds

std::string member_label(const tb200_group *g, int i, const std::vector<int64_t> *bounds) {
    std::string s = "group member " + std::to_string(i) + " (device " + std::to_string(g->m[(size_t)i]->device);
    if (bounds) s += ", global packets [" + std::to_string((*bounds)[(size_t)i]) + ", " + std::to_string((*bounds)[(size_t)i + 1]) + ")";
    return s + "): ";
}

// Runs f(i) for every member, one host thread each (pageable host buffers make every copy a host-side wait), joins them
// all, and returns the first member's error with the member named (g_last_error is per thread).
template <class F> int group_parallel(tb200_group *g, const std::vector<int64_t> *bounds, F f) {
    const int G = (int)g->m.size();
    std::vector<int> rc((size_t)G, TB200_OK);
    std::vector<std::string> msg((size_t)G);
    std::vector<std::thread> threads;
    threads.reserve((size_t)G);
    bool spawn_failed = false;
    for (int i = 0; i < G && !spawn_failed; i++) {
        try {
            threads.emplace_back([&, i] {
                rc[(size_t)i] = f(i);
                if (rc[(size_t)i]) msg[(size_t)i] = g_last_error;
            });
        } catch (...) {
            spawn_failed = true;
        }
    }
    for (auto &t : threads) t.join();
    if (spawn_failed) return fail(TB200_ERR_INVALID, "could not start a host thread per group member");
    for (int i = 0; i < G; i++)
        if (rc[(size_t)i]) return fail(rc[(size_t)i], member_label(g, i, bounds) + msg[(size_t)i]);
    return TB200_OK;
}

bool direct(const tb200_group *g, int owner, int k) {
    return owner == k || (g->peer_access && g->peer[(size_t)owner * g->m.size() + k]);
}

// Reduce-scatter + all-gather of n_elems 8-byte elements at ptr(k) on every member k: owner o sums pair range
// [o P / G, (o + 1) P / G) of every member (P = n_elems / 2) and writes the sum back to every member.  Asynchronous on
// the owners' streams.
template <bool WORDS, class Ptr> int reduce_buffers(tb200_group *g, Ptr ptr, size_t n_elems) {
    const int G = (int)g->m.size();
    if (n_elems % 2) return fail(TB200_ERR_INVALID, "collective: odd element count");
    const long long pairs = (long long)(n_elems / 2);
    for (int o = 0; o < G; o++) {
        tb200_engine *own = g->m[(size_t)o];
        const long long lo = pairs * o / G, count = pairs * (o + 1) / G - lo;
        if (count == 0) continue;
        const size_t bytes = (size_t)count * 16;
        CK(cudaSetDevice(own->device));
        int staged = 0;
        for (int k = 0; k < G; k++) staged += direct(g, o, k) ? 0 : 1;
        if (staged) {
            int r = g->staging[(size_t)o].ensure((size_t)staged * bytes);
            if (r) return r;
        }
        tbg::SlicePtrs p{};
        int nd = 0, j = 0;
        for (int k = 0; k < G; k++) {
            char *slice = (char *)ptr(g->m[(size_t)k]) + (size_t)lo * 16;
            if (direct(g, o, k)) {
                p.src[k] = slice;
                p.dst[nd++] = slice;
            } else {
                unsigned char *copy = g->staging[(size_t)o].p + (size_t)j++ * bytes;
                CK(cudaMemcpyPeerAsync(copy, own->device, slice, g->m[(size_t)k]->device, bytes, own->stream));
                p.src[k] = copy;
            }
        }
        const long long want = (count + 255) / 256, cap = (long long)own->sm_count * 8;
        tbg::reduce_slice_kernel<WORDS><<<(unsigned)(want < cap ? want : cap), 256, 0, own->stream>>>(p, G, nd, count);
        own->launches++;
        CK(cudaGetLastError());
        const char *sum = (const char *)ptr(own) + (size_t)lo * 16;
        for (int k = 0; k < G; k++)
            if (!direct(g, o, k))
                CK(cudaMemcpyPeerAsync((char *)ptr(g->m[(size_t)k]) + (size_t)lo * 16, g->m[(size_t)k]->device, sum, own->device, bytes, own->stream));
    }
    return TB200_OK;
}

int sync_members(tb200_group *g) {
    for (tb200_engine *e : g->m) {
        CK(cudaSetDevice(e->device));
        CK(cudaStreamSynchronize(e->stream));
    }
    return TB200_OK;
}

// Member views of the caller's arrays for packets [lo, lo + count): per-packet outputs at the range offset, the event
// rows of the tracked packets inside the range; no estimators (they come from the collective).
tb200_outputs member_outputs(const tb200_outputs *o, int64_t lo, int64_t count) {
    tb200_outputs q{};
    auto at = [lo](auto *p) { return p ? p + lo : p; };
    q.output_nus = at(o->output_nus); q.output_energies = at(o->output_energies);
    q.last_interaction_type = at(o->last_interaction_type); q.last_event_id = at(o->last_event_id);
    q.last_shell_id = at(o->last_shell_id); q.last_line_absorb_id = at(o->last_line_absorb_id); q.last_line_emit_id = at(o->last_line_emit_id);
    q.last_radius = at(o->last_radius); q.last_before_nu = at(o->last_before_nu); q.last_before_mu = at(o->last_before_mu);
    q.last_before_energy = at(o->last_before_energy); q.last_after_nu = at(o->last_after_nu); q.last_after_mu = at(o->last_after_mu);
    q.last_after_energy = at(o->last_after_energy);
    if (o->events && o->max_events_per_packet > 0) {
        int64_t nt = o->n_tracked_packets - lo;
        nt = nt < 0 ? 0 : (nt > count ? count : nt);
        if (nt > 0) {
            q.events = o->events + lo * o->max_events_per_packet;
            q.event_counts = at(o->event_counts);
            q.n_tracked_packets = nt;
            q.max_events_per_packet = o->max_events_per_packet;
        }
    }
    return q;
}

// Host packets in (pk), or the members' resident packets (pk == nullptr); see tb200_group_run.
int group_run(tb200_group *g, const tb200_packets *pk, tb200_outputs *o) {
    const int G = (int)g->m.size();
    std::vector<int64_t> b((size_t)G + 1, 0);
    if (pk) {
        if (pk->n_packets < 0 || pk->n_packets > 2000000000LL) return fail(TB200_ERR_INVALID, "n_packets out of range");
        for (int i = 0; i <= G; i++) b[(size_t)i] = shard_lo(pk->n_packets, i, G);
    } else {
        for (int i = 0; i < G; i++) b[(size_t)i + 1] = b[(size_t)i] + g->m[(size_t)i]->N;
        if (b[(size_t)G] <= 0) return fail(TB200_ERR_INVALID, "no packets are resident: call tb200_group_upload_packets or tb200_group_create_packets first");
    }
    const int64_t n = b[(size_t)G];
    // virtual-packet logs: each member logs into its device buffer (it cannot know beforehand how many rows the members
    // before it will need); the rows that fit are copied into the caller's arrays afterwards, in member order
    const bool vlog = o->vlog_nus && o->vlog_capacity > 0;
    const int64_t cap = vlog ? o->vlog_capacity : 0;
    std::vector<tb200_packets> pks((size_t)G);
    std::vector<tb200_outputs> os((size_t)G);
    for (int i = 0; i < G; i++) {
        const int64_t lo = b[(size_t)i], count = b[(size_t)i + 1] - lo;
        if (pk) pks[(size_t)i] = {count, pk->initial_radii + lo, pk->initial_nus + lo, pk->initial_mus + lo, pk->initial_energies + lo,
                                  pk->packet_seeds + lo};
        tb200_outputs &q = os[(size_t)i];
        q = member_outputs(o, lo, count);
        if (vlog) {  // arms the member's log (run_pipelined with log_on_device writes none of these arrays)
            q.vlog_nus = o->vlog_nus;
            q.vlog_capacity = cap;
        }
    }
    // the fixed-point scales of the whole set, the same on every member (host packets; resident ones got it when they came)
    if (pk && n > 0) {
        const double e_typ = typical_energy(pk->initial_energies, n);
        for (tb200_engine *e : g->m) e->e_typ_group = e_typ;
    }
    int r = group_parallel(g, &b, [&](int i) {
        std::lock_guard<std::mutex> lock(*g->device_lock[(size_t)i]);
        return run_pipelined(g->m[(size_t)i], pk ? &pks[(size_t)i] : nullptr, &os[(size_t)i], true);
    });
    for (tb200_engine *e : g->m) e->e_typ_group = 0.0;
    if (r) return r;
    // global packet ids in the event rows and the virtual-packet log; the logs in member order
    for (int i = 0; i < G; i++) {
        const tb200_outputs &q = os[(size_t)i];
        const int64_t lo = b[(size_t)i];
        for (int64_t p = 0; p < q.n_tracked_packets; p++) {
            int64_t rows = q.max_events_per_packet;
            if (q.event_counts && q.event_counts[p] < rows) rows = q.event_counts[p];
            for (int64_t k = 0; k < rows; k++) q.events[p * q.max_events_per_packet + k].packet_id += lo;
        }
    }
    if (vlog) {
        int64_t total = 0, stored = 0;
        for (int i = 0; i < G; i++) {
            tb200_engine *e = g->m[(size_t)i];
            const int64_t cnt = os[(size_t)i].vlog_count, mine = cnt < cap ? cnt : cap;
            const int64_t take = mine < cap - stored ? mine : cap - stored;
            total += cnt;
            if (take <= 0) continue;
            CK(cudaSetDevice(e->device));
            double *dst[4] = {o->vlog_nus, o->vlog_energies, o->vlog_initial_mus, o->vlog_initial_rs};
            for (int c = 0; c < 4; c++)
                if (dst[c]) CK(cudaMemcpy(dst[c] + stored, e->vlog_d.p + (size_t)c * e->vlog_capacity, (size_t)take * sizeof(double), cudaMemcpyDeviceToHost));
            if (o->vlog_packet_index) {
                CK(cudaMemcpy(o->vlog_packet_index + stored, e->vlog_pid.p, (size_t)take * sizeof(long long), cudaMemcpyDeviceToHost));
                for (int64_t k = 0; k < take; k++) o->vlog_packet_index[stored + k] += b[(size_t)i];
            }
            stored += take;
        }
        o->vlog_count = total;
    } else {
        o->vlog_count = 0;
    }
    int exact = 0;
    if ((r = tb200_group_allreduce(g, &exact))) return r;
    // the estimators, now the same on every member, from member 0
    tb200_outputs est = *o;
    est.output_nus = est.output_energies = nullptr;
    est.last_interaction_type = est.last_event_id = est.last_shell_id = est.last_line_absorb_id = est.last_line_emit_id = nullptr;
    est.last_radius = est.last_before_nu = est.last_before_mu = est.last_before_energy = nullptr;
    est.last_after_nu = est.last_after_mu = est.last_after_energy = nullptr;
    est.events = nullptr; est.event_counts = nullptr; est.n_tracked_packets = 0;
    est.vlog_nus = nullptr; est.vlog_capacity = 0;
    if ((r = tb200_download(g->m[0], &est))) return fail(r, member_label(g, 0, nullptr) + g_last_error);
    // work counters: exact integer sums
    int64_t *sum = reinterpret_cast<int64_t *>(&o->counters);
    constexpr int n_counters = (int)(sizeof(tb200_counters) / sizeof(int64_t));
    for (int c = 0; c < n_counters; c++) {
        sum[c] = 0;
        for (int i = 0; i < G; i++) sum[c] += reinterpret_cast<const int64_t *>(&os[(size_t)i].counters)[c];
    }
    return TB200_OK;
}

}  // namespace

extern "C" {

int tb200_group_create(const int *device_ids, int n, tb200_group **group) {
    if (!group) return fail(TB200_ERR_INVALID, "group is NULL");
    *group = nullptr;
    if (!device_ids || n < 1 || n > tbg::MAX_MEMBERS) return fail(TB200_ERR_INVALID, "a group needs 1 to 32 device ids");
    int caller_device = 0;  // creating engines and enabling peer access switch devices: the caller's current one is restored
    const bool restore = cudaGetDevice(&caller_device) == cudaSuccess;
    if (!restore) cudaGetLastError();
    tb200_group *g = new tb200_group();
    for (int i = 0; i < n; i++) {
        tb200_engine *e = nullptr;
        const int r = tb200_create(device_ids[i], &e);
        if (r) {
            const std::string why = g_last_error;
            tb200_group_destroy(g);
            if (restore) cudaSetDevice(caller_device);
            return fail(r, "group member " + std::to_string(i) + ": " + why);
        }
        g->m.push_back(e);
    }
    g->staging.resize((size_t)n);
    g->fi_ran.assign((size_t)n, 0);
    g->peer.assign((size_t)n * n, 0);
    g->device_lock.resize((size_t)n);
    for (int i = 0; i < n; i++) {
        for (int j = 0; j < i && !g->device_lock[(size_t)i]; j++)
            if (device_ids[j] == device_ids[i]) g->device_lock[(size_t)i] = g->device_lock[(size_t)j];
        if (!g->device_lock[(size_t)i]) g->device_lock[(size_t)i] = std::make_shared<std::mutex>();
    }
    for (int a = 0; a < n; a++)
        for (int b = 0; b < n; b++) {
            const int da = device_ids[a], db = device_ids[b];
            if (da == db) { g->peer[(size_t)a * n + b] = 1; continue; }
            int can = 0;
            if (cudaDeviceCanAccessPeer(&can, da, db) != cudaSuccess || !can) { cudaGetLastError(); continue; }
            if (cudaSetDevice(da) != cudaSuccess) { cudaGetLastError(); continue; }
            cudaError_t e = cudaDeviceEnablePeerAccess(db, 0);
            if (e == cudaErrorPeerAccessAlreadyEnabled) e = cudaSuccess;
            cudaGetLastError();
            g->peer[(size_t)a * n + b] = e == cudaSuccess ? 1 : 0;
        }
    // Peer access stays enabled after tb200_group_destroy: it belongs to the process's device contexts, and another group
    // (or the caller) may be using it.
    if (restore) cudaSetDevice(caller_device);
    *group = g;
    return TB200_OK;
}

void tb200_group_destroy(tb200_group *g) {
    if (!g) return;
    for (size_t i = 0; i < g->m.size(); i++) {
        if (i < g->staging.size()) {
            cudaSetDevice(g->m[i]->device);
            g->staging[i].release();  // here, with its device current: its destructor would run on whichever device is
        }
        tb200_destroy(g->m[i]);
    }
    delete g;
}

int tb200_group_size(tb200_group *g) { return g ? (int)g->m.size() : 0; }

int tb200_group_member(tb200_group *g, int i, tb200_engine **engine) {
    if (!g || !engine || i < 0 || i >= (int)g->m.size()) return fail(TB200_ERR_INVALID, "bad argument");
    *engine = g->m[(size_t)i];
    return TB200_OK;
}

int tb200_group_set_option(tb200_group *g, const char *name, int64_t value) {
    if (!g || !name) return fail(TB200_ERR_INVALID, "bad argument");
    if (std::string(name) == "peer_access") { g->peer_access = value ? 1 : 0; return TB200_OK; }
    for (tb200_engine *e : g->m) {
        const int r = tb200_set_option(e, name, value);
        if (r) return r;
    }
    return TB200_OK;
}

int tb200_group_set_model(tb200_group *g, const tb200_model *model, const tb200_config *config) {
    if (!g) return fail(TB200_ERR_INVALID, "bad argument");
    return group_parallel(g, nullptr, [&](int i) { return tb200_set_model(g->m[(size_t)i], model, config); });
}

int tb200_group_set_atomic_data(tb200_group *g, const tb200_atomic_data *atomic) {
    if (!g) return fail(TB200_ERR_INVALID, "bad argument");
    return group_parallel(g, nullptr, [&](int i) { return tb200_set_atomic_data(g->m[(size_t)i], atomic); });
}

int tb200_group_build_opacity(tb200_group *g, const tb200_plasma_state *plasma) {
    if (!g) return fail(TB200_ERR_INVALID, "bad argument");
    return group_parallel(g, nullptr, [&](int i) {
        int r = tb200_build_opacity(g->m[(size_t)i], plasma);
        return r ? r : tb200_sync(g->m[(size_t)i]);
    });
}

int tb200_group_set_plasma_data(tb200_group *g, const tb200_plasma_data *data) {
    if (!g) return fail(TB200_ERR_INVALID, "bad argument");
    return group_parallel(g, nullptr, [&](int i) { return tb200_set_plasma_data(g->m[(size_t)i], data); });
}

int tb200_group_solve_plasma(tb200_group *g, const tb200_plasma_params *params, double *electron_densities, double *ion_number_density,
                             double *level_number_density, double *j_blues, int32_t *iterations) {
    if (!g) return fail(TB200_ERR_INVALID, "bad argument");
    return group_parallel(g, nullptr, [&](int i) {
        if (i == 0) return tb200_solve_plasma(g->m[0], params, electron_densities, ion_number_density, level_number_density, j_blues, iterations);
        return tb200_solve_plasma(g->m[(size_t)i], params, nullptr, nullptr, nullptr, nullptr, nullptr);
    });
}

int tb200_group_build_absorbing_markov(tb200_group *g, const tb200_markov_input *input) {
    if (!g) return fail(TB200_ERR_INVALID, "bad argument");
    return group_parallel(g, nullptr, [&](int i) { return tb200_build_absorbing_markov(g->m[(size_t)i], input); });
}

int tb200_group_upload_packets(tb200_group *g, const tb200_packets *pk) {
    if (!g || !pk) return fail(TB200_ERR_INVALID, "bad argument");
    if (pk->n_packets < 0 || pk->n_packets > 2000000000LL) return fail(TB200_ERR_INVALID, "n_packets out of range");
    const int G = (int)g->m.size();
    const int64_t n = pk->n_packets;
    std::vector<int64_t> b((size_t)G + 1);
    for (int i = 0; i <= G; i++) b[(size_t)i] = shard_lo(n, i, G);
    if (n > 0) {
        const double e_typ = typical_energy(pk->initial_energies, n);
        for (tb200_engine *e : g->m) e->e_typ_group = e_typ;
    }
    const int r = group_parallel(g, &b, [&](int i) {
        const int64_t lo = b[(size_t)i];
        const tb200_packets q = {b[(size_t)i + 1] - lo, pk->initial_radii + lo, pk->initial_nus + lo, pk->initial_mus + lo,
                                 pk->initial_energies + lo, pk->packet_seeds + lo};
        const int rr = tb200_upload_packets(g->m[(size_t)i], &q);
        return rr ? rr : tb200_sync(g->m[(size_t)i]);
    });
    for (tb200_engine *e : g->m) e->e_typ_group = 0.0;
    return r;
}

int tb200_group_create_packets(tb200_group *g, const tb200_packet_source *src) {
    if (!g || !src) return fail(TB200_ERR_INVALID, "bad argument");
    const int G = (int)g->m.size();
    std::vector<int64_t> b((size_t)G + 1);
    for (int i = 0; i <= G; i++) b[(size_t)i] = shard_lo(src->n_packets, i, G);
    if (src->weighted)  // two sums over the whole set: the passes meet on the host (create_weighted_packets)
        return create_weighted_packets(src, g->m.data(), b.data(), G, [&](auto f) { return group_parallel(g, &b, f); });
    return group_parallel(g, &b, [&](int i) {
        const int r = create_packets_range(g->m[(size_t)i], src, b[(size_t)i], b[(size_t)i + 1]);
        return r ? r : tb200_sync(g->m[(size_t)i]);
    });
}

int tb200_group_run(tb200_group *g, const tb200_packets *packets, tb200_outputs *outputs) {
    if (!g || !packets || !outputs) return fail(TB200_ERR_INVALID, "bad argument");
    return group_run(g, packets, outputs);
}

int tb200_group_run_resident(tb200_group *g, tb200_outputs *outputs) {
    if (!g || !outputs) return fail(TB200_ERR_INVALID, "bad argument");
    return group_run(g, nullptr, outputs);
}

int tb200_group_sync(tb200_group *g) {
    if (!g) return fail(TB200_ERR_INVALID, "bad argument");
    return group_parallel(g, nullptr, [&](int i) { return tb200_sync(g->m[(size_t)i]); });
}

int tb200_group_allreduce(tb200_group *g, int *exact) {
    if (!g || !exact) return fail(TB200_ERR_INVALID, "bad argument");
    *exact = 0;
    const int G = (int)g->m.size();
    tb200_engine *m0 = g->m[0];
    for (int i = 0; i < G; i++) {
        const tb200_engine *e = g->m[(size_t)i];
        if (!e->have_model) return fail(TB200_ERR_NO_MODEL, member_label(g, i, nullptr) + "tb200_set_model has not been called");
        if (e->est_count != m0->est_count || e->off_jblue != m0->off_jblue || e->S != m0->S || e->lpad != m0->lpad)
            return fail(TB200_ERR_INVALID, member_label(g, i, nullptr) + "holds another model than member 0");
    }
    for (int i = 0; i < G; i++)
        if (!g->m[(size_t)i]->est_unreduced)
            return fail(TB200_ERR_INVALID, member_label(g, i, nullptr) + "no transport since the last collective (summing again would multiply the estimators)");
    // the fixed-point words are summed when every member filled them at the same scales; otherwise the doubles
    bool ex = true;
    for (const tb200_engine *e : g->m)
        ex = ex && e->algorithm == 1 && e->diff.p && e->diff_scale1 != 0.0 && e->diff_scale1 == m0->diff_scale1 &&
             e->diff_scale2 == m0->diff_scale2;
    const auto t0 = std::chrono::steady_clock::now();
    int r;
    if ((r = sync_members(g))) return r;
    if (G > 1) {
        auto est = [](tb200_engine *e) { return (void *)e->est.p; };
        if (ex) {
            const size_t n_words = (size_t)m0->S * (m0->lpad + 1) * 4;
            if ((r = reduce_buffers<true>(g, [](tb200_engine *e) { return (void *)e->diff.p; }, n_words))) return r;
            if ((r = reduce_buffers<false>(g, est, m0->off_jblue))) return r;
        } else if ((r = reduce_buffers<false>(g, est, m0->est_count))) {
            return r;
        }
        if ((r = sync_members(g))) return r;
        if (ex) {
            for (int i = 0; i < G; i++)
                if ((r = tb200_finalize_line_estimators(g->m[(size_t)i]))) return fail(r, member_label(g, i, nullptr) + g_last_error);
            for (int i = 0; i < G; i++)
                if ((r = tb200_sync(g->m[(size_t)i]))) return fail(r, member_label(g, i, nullptr) + g_last_error);
        }
    }
    for (tb200_engine *e : g->m) e->est_unreduced = false;
    g->allreduce_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    g->allreduce_timed = true;
    *exact = ex ? 1 : 0;
    return TB200_OK;
}

int tb200_group_allreduce_ms(tb200_group *g, double *ms) {
    if (!g || !ms) return fail(TB200_ERR_INVALID, "bad argument");
    if (!g->allreduce_timed) return fail(TB200_ERR_INVALID, "no collective has run yet");
    *ms = g->allreduce_ms;
    return TB200_OK;
}

int tb200_group_formal_integral(tb200_group *g, const tb200_formal_integral_params *params, const double *frequencies,
                                int64_t n_frequencies, double *luminosity_densities, double *intensities_nu_p) {
    if (!g || !params || !frequencies || !luminosity_densities || n_frequencies < 0) return fail(TB200_ERR_INVALID, "bad argument");
    const int G = (int)g->m.size();
    std::vector<int64_t> b((size_t)G + 1);
    for (int i = 0; i <= G; i++) b[(size_t)i] = shard_lo(n_frequencies, i, G);
    for (int i = 0; i < G; i++) g->fi_ran[(size_t)i] = b[(size_t)i + 1] > b[(size_t)i] ? 1 : 0;
    return group_parallel(g, nullptr, [&](int i) {
        const int64_t lo = b[(size_t)i], count = b[(size_t)i + 1] - lo;
        if (count == 0) return (int)TB200_OK;
        return tb200_formal_integral(g->m[(size_t)i], params, frequencies + lo, count, luminosity_densities + lo,
                                     intensities_nu_p ? intensities_nu_p + lo * params->n_impact_parameters : nullptr);
    });
}

int tb200_group_formal_integral_ms(tb200_group *g, double *interpolation_ms, double *integral_ms) {
    if (!g || !interpolation_ms || !integral_ms) return fail(TB200_ERR_INVALID, "bad argument");
    *interpolation_ms = *integral_ms = 0.0;
    for (size_t i = 0; i < g->m.size(); i++) {
        if (!g->fi_ran[i]) continue;  // the members ran concurrently: the slowest one's times
        *interpolation_ms = std::max(*interpolation_ms, g->m[i]->fi_cells_ms);
        *integral_ms = std::max(*integral_ms, g->m[i]->fi_rays_ms);
    }
    return TB200_OK;
}

}  // extern "C"
