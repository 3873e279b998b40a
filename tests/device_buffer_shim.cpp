// Host build of tardis_b200/csrc/device_buffer.cuh against counting stand-ins for the CUDA runtime calls it makes: every
// allocation, event and stream gets an id, and every call is logged ("M3": cudaMalloc gave id 3, "F3": cudaFree of it;
// E / e: events, S / s: streams; "X": a free or destroy of something that is not live, i.e. a double free or a null).
// tests/test_device_buffer.py compiles it with g++ and drives the scenarios below.  cudart is not linked.
#include <cstdint>
#include <cstring>
#include <set>
#include <string>
#include <vector>

#include "../tardis_b200/csrc/device_buffer.cuh"

namespace {
std::string g_log;
std::set<uintptr_t> g_live;
uintptr_t g_next = 0;
bool g_fail_next_malloc = false;

uintptr_t make(char tag) {
    const uintptr_t id = ++g_next;
    g_live.insert(id);
    g_log += std::string(g_log.empty() ? "" : " ") + tag + std::to_string(id);
    return id;
}
cudaError_t drop(char tag, uintptr_t id) {
    if (!g_live.erase(id)) {
        g_log += std::string(g_log.empty() ? "" : " ") + "X";
        return cudaErrorInvalidValue;
    }
    g_log += std::string(g_log.empty() ? "" : " ") + tag + std::to_string(id);
    return cudaSuccess;
}
}  // namespace

extern "C" {
cudaError_t cudaMalloc(void **p, size_t) {
    if (g_fail_next_malloc) {
        g_fail_next_malloc = false;
        return cudaErrorMemoryAllocation;
    }
    *p = reinterpret_cast<void *>(make('M'));
    return cudaSuccess;
}
cudaError_t cudaFree(void *p) { return drop('F', reinterpret_cast<uintptr_t>(p)); }
cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = reinterpret_cast<cudaEvent_t>(make('E')); return cudaSuccess; }
cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned int) { return cudaEventCreate(e); }
cudaError_t cudaEventDestroy(cudaEvent_t e) { return drop('e', reinterpret_cast<uintptr_t>(e)); }
cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned int) { *s = reinterpret_cast<cudaStream_t>(make('S')); return cudaSuccess; }
cudaError_t cudaStreamDestroy(cudaStream_t s) { return drop('s', reinterpret_cast<uintptr_t>(s)); }
const char *cudaGetErrorString(cudaError_t e) { return e == cudaErrorMemoryAllocation ? "out of memory" : "stand-in error"; }

void shim_reset() { g_log.clear(); g_live.clear(); g_next = 0; g_fail_next_malloc = false; g_last_error.clear(); }
const char *shim_log() { return g_log.c_str(); }
int shim_live() { return (int)g_live.size(); }
const char *shim_last_error() { return g_last_error.c_str(); }

// A struct laid out as tb200_engine is: streams and events first, then buffers (one never allocated, one of 0 elements).
// Returns 0, or the number of the first check that failed.
int shim_owners_struct() {
    struct Owners {
        Stream stream, spare_stream;
        Event ev_a, ev_b, spare_event;
        DBuf<double> a;
        DBuf<int> b;
        DBuf<unsigned char> empty, never;
    };
    {
        Owners o;
        if (cudaStreamCreateWithFlags(&o.stream.h, cudaStreamNonBlocking) || cudaEventCreate(&o.ev_a.h) ||
            cudaEventCreateWithFlags(&o.ev_b.h, cudaEventDisableTiming))
            return 1;
        if (o.a.ensure(10) || o.b.ensure(5) || o.empty.ensure(0)) return 2;
        if (!o.empty.p || o.empty.n != 0) return 3;
    }
    return 0;
}

// Moves of every owner, by construction, by assignment and inside a growing std::vector.
int shim_moves() {
    {
        DBuf<double> a;
        if (a.ensure(8)) return 1;
        double *const pa = a.p;
        DBuf<double> b(std::move(a));
        if (a.p || a.n || b.p != pa || b.n != 8) return 2;
        DBuf<double> c;
        if (c.ensure(4)) return 3;
        c = std::move(b);  // c's own allocation goes, b's comes
        if (b.p || b.n || c.p != pa || c.n != 8) return 4;

        std::vector<DBuf<unsigned char>> v(2);
        if (v[0].ensure(3) || v[1].ensure(7)) return 6;
        unsigned char *const p0 = v[0].p;
        v.resize(64);  // reallocates: the elements move
        if (v[0].p != p0 || v[0].n != 3 || v[1].n != 7 || v[63].p) return 7;

        Event e, g;
        if (cudaEventCreate(&e.h) || cudaEventCreate(&g.h)) return 8;
        const cudaEvent_t he = e;
        Event f(std::move(e));
        if (e.h || f != he) return 9;
        g = std::move(f);  // g's own event goes
        if (f.h || g != he) return 10;

        Stream s, t;
        if (cudaStreamCreateWithFlags(&s.h, cudaStreamNonBlocking)) return 11;
        const cudaStream_t hs = s;
        t = std::move(s);
        Stream u(std::move(t));
        if (s.h || t.h || u != hs) return 12;
        std::vector<Event> evs(3);
        for (Event &x : evs)
            if (cudaEventCreate(&x.h)) return 13;
        evs.resize(40);
    }
    return 0;
}

// ensure to 10, to 100 (grows), to 5 and 100 again (no reallocation); returns 0 or the failed check.
int shim_ensure_sizes() {
    DBuf<double> a;
    if (a.ensure(10) || a.n != 10) return 1;
    if (a.ensure(100) || a.n != 100) return 2;
    double *const p = a.p;
    if (a.ensure(5) || a.p != p || a.n != 100) return 3;
    if (a.ensure(100) || a.p != p || a.n != 100) return 4;
    return 0;
}

// A buffer of 10 elements asked for 100 while cudaMalloc fails: returns what ensure returned; *p_null / *n_out report the
// buffer afterwards.
int shim_ensure_fails(int *p_null, long long *n_out) {
    DBuf<double> a;
    if (a.ensure(10)) return -1;
    g_fail_next_malloc = true;
    const int r = a.ensure(100);
    *p_null = a.p == nullptr;
    *n_out = (long long)a.n;
    return r;
}
}
