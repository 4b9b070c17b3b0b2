// wait_timeouts.h — per-device counters of the bounded waits that ran out, for the frame entries whose kernels wait on one another's
// progress inside one launch (vp9lf.cu, vp9intra.cu, hevcintra.cu, vp8lf.cu).  Each device ordinal gets one small block of device memory for the life of the
// process, made at the first frame call on it, with one int per entry, so each entry's *_timeouts() reports only its own waits.
#pragma once
#include <mutex>
#include <cuda_runtime.h>

enum { B200_WAIT_VP9_LOOPFILTER = 0, B200_WAIT_VP9_INTRA = 1, B200_WAIT_HEVC_INTRA = 2, B200_WAIT_VP8_LOOPFILTER = 3, B200_WAIT_SLOTS = 4 };

// the counter of `slot` on device `ordinal` (the caller has made it current); nullptr when none exists yet and !create, or on failure
inline int *b200_wait_timeouts_word(int ordinal, int slot, bool create)
{
    constexpr int kMaxOrdinals = 64;
    static std::mutex mu;
    static int *words[kMaxOrdinals];
    if (ordinal < 0 || ordinal >= kMaxOrdinals || slot < 0 || slot >= B200_WAIT_SLOTS) return nullptr;
    std::lock_guard<std::mutex> lock(mu);
    if (!words[ordinal] && create) {
        int *w = nullptr;
        const int zero[B200_WAIT_SLOTS] = {};
        if (cudaMalloc(&w, sizeof(zero)) != cudaSuccess) return nullptr;
        if (cudaMemcpy(w, zero, sizeof(zero), cudaMemcpyHostToDevice) != cudaSuccess) { cudaFree(w); return nullptr; }
        words[ordinal] = w;
    }
    return words[ordinal] ? words[ordinal] + slot : nullptr;
}
