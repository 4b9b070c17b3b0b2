// common.h — internals shared by the translation units of libb200dsp.so
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstddef>
#include <cstdio>
#include <atomic>
#include <mutex>
#include "b200dsp.h"

#define B200_API extern "C" __attribute__((visibility("default")))

struct B200Device {
    int ordinal = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    int sm_count = 0;
    // rotating copy/compute streams + events for the *_host pipelined entry points
    static constexpr int kPipe = 3;
    cudaStream_t pipe[kPipe] = {nullptr, nullptr, nullptr};
    // scratch owned by the device object (grown on demand, reused by the drop-in host-pointer calls)
    void *scratch = nullptr;
    size_t scratch_bytes = 0;
    void *pinned = nullptr;
    size_t pinned_bytes = 0;
    // Serialises the host-pointer entry points (function tables, b200_sws_scale, *_host): they share `scratch`, `pinned`, `stream`
    // and `pipe[]`, while the reference functions they replace are pure and get called from slice / frame threads concurrently.
    // Recursive: a host entry may call another one (tx -> int32 tx).
    std::recursive_mutex mu;
};
#define B200_LOCK_DEVICE(dev) std::lock_guard<std::recursive_mutex> b200_device_lock_((dev)->mu)

void b200_set_error(const char *fmt, ...);
extern std::atomic<uint64_t> g_b200_launches;
B200Device *b200_default_device();               // lazily opened, nullptr on failure
void *b200_scratch(B200Device *dev, size_t bytes);       // device scratch (>= bytes), nullptr on failure
void *b200_pinned(B200Device *dev, size_t bytes);        // pinned host scratch

#define B200_CUDA_OK(expr)                                                                      \
    do {                                                                                        \
        cudaError_t e_ = (expr);                                                                \
        if (e_ != cudaSuccess) {                                                                \
            b200_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(e_)); \
            return B200_EEXTERNAL;                                                              \
        }                                                                                       \
    } while (0)

#define B200_LAUNCHED() (g_b200_launches.fetch_add(1, std::memory_order_relaxed))

static inline int b200_ceil_div(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

// 2-D copies between a HOST picture with a signed line size (bottom-up / flipped frames have negative ones, which the reference's
// C functions accept: row r lives at base + r * pitch) and a dense device tile.  cudaMemcpy2D takes unsigned pitches only, so a
// negative pitch is copied from the lowest address with |pitch| and the device-side row order reversed: row r of the picture lands
// in (is taken from) device row r either way.
static inline cudaError_t b200_h2d_rows(void *dev, size_t dpitch, const void *host, ptrdiff_t hpitch, size_t w, size_t rows, cudaStream_t st)
{
    if (hpitch >= 0) return cudaMemcpy2DAsync(dev, dpitch, host, (size_t)hpitch, w, rows, cudaMemcpyHostToDevice, st);
    for (size_t r = 0; r < rows; r++) {
        cudaError_t e = cudaMemcpyAsync((uint8_t *)dev + r * dpitch, (const uint8_t *)host + (ptrdiff_t)r * hpitch, w, cudaMemcpyHostToDevice, st);
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}
static inline cudaError_t b200_d2h_rows(void *host, ptrdiff_t hpitch, const void *dev, size_t dpitch, size_t w, size_t rows, cudaStream_t st)
{
    if (hpitch >= 0) return cudaMemcpy2DAsync(host, (size_t)hpitch, dev, dpitch, w, rows, cudaMemcpyDeviceToHost, st);
    for (size_t r = 0; r < rows; r++) {
        cudaError_t e = cudaMemcpyAsync((uint8_t *)host + (ptrdiff_t)r * hpitch, (const uint8_t *)dev + r * dpitch, w, cudaMemcpyDeviceToHost, st);
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}
