// device_buffer.cuh -- owners of the engine's device memory, CUDA events and CUDA streams, and the per-thread error text
// (tb200_last_error) they report through.  Each owner frees what it holds when it goes, so a struct of them needs no
// release list; none can be copied, so nothing is freed twice.
#pragma once
#include <string>
#include <utility>

#include <cuda_runtime.h>

#include "../../include/tardis_b200.h"

namespace {

thread_local std::string g_last_error;

int fail(int code, const std::string &msg) {
    g_last_error = msg;
    return code;
}

// At least n elements of T in device memory; grown by ensure (the contents are not kept), freed with the owner.
template <typename T> struct DBuf {
    T *p = nullptr;
    size_t n = 0;
    DBuf() = default;
    DBuf(const DBuf &) = delete;
    DBuf &operator=(const DBuf &) = delete;
    DBuf(DBuf &&o) noexcept : p(std::exchange(o.p, nullptr)), n(std::exchange(o.n, 0)) {}
    DBuf &operator=(DBuf &&o) noexcept {
        if (this != &o) {
            release();
            p = std::exchange(o.p, nullptr);
            n = std::exchange(o.n, 0);
        }
        return *this;
    }
    ~DBuf() { release(); }
    int ensure(size_t count) {
        if (count <= n && p) return TB200_OK;
        if (p) cudaFree(p);
        p = nullptr; n = 0;
        cudaError_t e = cudaMalloc((void **)&p, (count ? count : 1) * sizeof(T));
        if (e != cudaSuccess) return fail(TB200_ERR_CUDA, std::string("cudaMalloc: ") + cudaGetErrorString(e));
        n = count;
        return TB200_OK;
    }
    void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
};

// One CUDA handle, destroyed with the owner.  Created in place through h (cudaEventCreate(&ev.h), ...); converts to the
// raw handle wherever the runtime takes one.
template <typename H, cudaError_t (*destroy)(H)> struct Handle {
    H h = nullptr;
    Handle() = default;
    Handle(const Handle &) = delete;
    Handle &operator=(const Handle &) = delete;
    Handle(Handle &&o) noexcept : h(std::exchange(o.h, nullptr)) {}
    Handle &operator=(Handle &&o) noexcept {
        if (this != &o) {
            if (h) destroy(h);
            h = std::exchange(o.h, nullptr);
        }
        return *this;
    }
    ~Handle() { if (h) destroy(h); }
    operator H() const { return h; }
};

using Event = Handle<cudaEvent_t, cudaEventDestroy>;
using Stream = Handle<cudaStream_t, cudaStreamDestroy>;

}  // namespace
