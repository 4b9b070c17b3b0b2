// device.cu — device handle (AVHWDeviceContext/AVCUDADeviceContext analogue, libavutil/hwcontext_cuda.h) and helpers
#include "common.h"
#include <cstdarg>
#include <cstring>
#include <mutex>

static thread_local char t_err[512] = "";
std::atomic<uint64_t> g_b200_launches{0};
static B200Device *g_default = nullptr;
static bool g_default_owned = false;
static std::mutex g_mu;

void b200_set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(t_err, sizeof(t_err), fmt, ap);
    va_end(ap);
}

B200_API int b200_abi_version(void) { return B200DSP_ABI_VERSION; }
B200_API const char *b200_last_error(void) { return t_err; }
B200_API uint64_t b200_launch_count(void) { return g_b200_launches.load(); }

B200_API int b200_device_open(B200Device **out, int ordinal, void *cu_stream)
{
    if (!out) return B200_EINVAL;
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) {
        b200_set_error("no CUDA device available (%s)", e == cudaSuccess ? "count 0" : cudaGetErrorString(e));
        return B200_ENODEV;
    }
    if (ordinal < 0 || ordinal >= n) { b200_set_error("device ordinal %d out of range (have %d)", ordinal, n); return B200_EINVAL; }
    B200_CUDA_OK(cudaSetDevice(ordinal));
    B200Device *d = new B200Device();
    d->ordinal = ordinal;
    if (cu_stream) {
        d->stream = (cudaStream_t)cu_stream;
    } else {
        if (cudaStreamCreateWithFlags(&d->stream, cudaStreamNonBlocking) != cudaSuccess) { delete d; return B200_EEXTERNAL; }
        d->own_stream = true;
    }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, ordinal) != cudaSuccess) { delete d; return B200_EEXTERNAL; }
    d->sm_count = prop.multiProcessorCount;
    for (int i = 0; i < B200Device::kPipe; i++)
        if (cudaStreamCreateWithFlags(&d->pipe[i], cudaStreamNonBlocking) != cudaSuccess) { delete d; return B200_EEXTERNAL; }
    *out = d;
    return 0;
}

B200_API void b200_device_close(B200Device *d)
{
    if (!d) return;
    cudaSetDevice(d->ordinal);
    cudaStreamSynchronize(d->stream);
    for (int i = 0; i < B200Device::kPipe; i++)
        if (d->pipe[i]) { cudaStreamSynchronize(d->pipe[i]); cudaStreamDestroy(d->pipe[i]); }
    if (d->scratch) cudaFree(d->scratch);
    if (d->pinned) cudaFreeHost(d->pinned);
    if (d->own_stream) cudaStreamDestroy(d->stream);
    {
        std::lock_guard<std::mutex> lk(g_mu);
        if (g_default == d) { g_default = nullptr; g_default_owned = false; }
    }
    delete d;
}

B200_API int b200_device_sync(B200Device *d)
{
    if (!d) return B200_EINVAL;
    B200_CUDA_OK(cudaStreamSynchronize(d->stream));
    return 0;
}
B200_API int b200_device_ordinal(const B200Device *d) { return d ? d->ordinal : B200_EINVAL; }
B200_API void *b200_device_stream(const B200Device *d) { return d ? (void *)d->stream : nullptr; }
B200_API int b200_device_sm_count(const B200Device *d) { return d ? d->sm_count : B200_EINVAL; }

B200_API int b200_set_default_device(B200Device *d)
{
    std::lock_guard<std::mutex> lk(g_mu);
    g_default = d;
    g_default_owned = false;
    return 0;
}

B200Device *b200_default_device()
{
    std::lock_guard<std::mutex> lk(g_mu);
    if (!g_default) {
        B200Device *d = nullptr;
        if (b200_device_open(&d, 0, nullptr) < 0) return nullptr;
        g_default = d;
        g_default_owned = true;
    }
    return g_default;
}

void *b200_scratch(B200Device *d, size_t bytes)
{
    if (d->scratch_bytes >= bytes) return d->scratch;
    if (d->scratch) {
        // nothing may still read or write the old buffer: the caller's stream and the three pipeline streams (an error return from a
        // *_batch_host call can leave copies in flight there)
        cudaStreamSynchronize(d->stream);
        for (int i = 0; i < B200Device::kPipe; i++) if (d->pipe[i]) cudaStreamSynchronize(d->pipe[i]);
        cudaFree(d->scratch); d->scratch = nullptr; d->scratch_bytes = 0;
    }
    size_t want = bytes + (bytes >> 2) + 4096;
    if (cudaMalloc(&d->scratch, want) != cudaSuccess) { b200_set_error("cudaMalloc(%zu) failed", want); return nullptr; }
    d->scratch_bytes = want;
    return d->scratch;
}

void *b200_pinned(B200Device *d, size_t bytes)
{
    if (d->pinned_bytes >= bytes) return d->pinned;
    if (d->pinned) {
        cudaStreamSynchronize(d->stream);
        for (int i = 0; i < B200Device::kPipe; i++) if (d->pipe[i]) cudaStreamSynchronize(d->pipe[i]);
        cudaFreeHost(d->pinned); d->pinned = nullptr; d->pinned_bytes = 0;
    }
    size_t want = bytes + (bytes >> 2) + 4096;
    if (cudaMallocHost(&d->pinned, want) != cudaSuccess) { b200_set_error("cudaMallocHost(%zu) failed", want); return nullptr; }
    d->pinned_bytes = want;
    return d->pinned;
}

B200_API void *b200_malloc_device(B200Device *d, size_t bytes)
{
    if (!d) return nullptr;
    void *p = nullptr;
    cudaSetDevice(d->ordinal);
    if (cudaMalloc(&p, bytes) != cudaSuccess) { b200_set_error("cudaMalloc(%zu) failed", bytes); return nullptr; }
    return p;
}
B200_API void b200_free_device(B200Device *d, void *p) { if (p) { if (d) cudaSetDevice(d->ordinal); cudaFree(p); } }
B200_API void *b200_malloc_host(size_t bytes)
{
    void *p = nullptr;
    if (cudaMallocHost(&p, bytes) != cudaSuccess) { b200_set_error("cudaMallocHost(%zu) failed", bytes); return nullptr; }
    return p;
}
B200_API void b200_free_host(void *p) { if (p) cudaFreeHost(p); }
B200_API int b200_memcpy_h2d(B200Device *d, void *dst, const void *src, size_t bytes)
{
    if (!d) return B200_EINVAL;
    B200_CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, d->stream));
    return 0;
}
B200_API int b200_memcpy_d2h(B200Device *d, void *dst, const void *src, size_t bytes)
{
    if (!d) return B200_EINVAL;
    B200_CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, d->stream));
    return 0;
}
