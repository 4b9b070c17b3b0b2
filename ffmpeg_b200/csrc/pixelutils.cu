// pixelutils.cu — libavutil's public block SAD (av_pixelutils_get_sad_fn, libavutil/pixelutils.h:31-52) on sm_90a: the me_cmp entry
// with one stride per block that libavfilter's users (vf_deshake, vf_mpdecimate style callers) and external programs reach.
//
// Reference semantics (checker: the pixelutils part of oracle/mecmp_oracle.c), libavutil/pixelutils.c:43-111: square blocks of
// 2, 4, 8, 16 or 32 pixels (w_bits = h_bits = 1 ... 5), sum of |src1 - src2| as an int; any other size has no function (NULL).
#include "common.h"

namespace {

// [device-code pixelutils] (tests/cuda_emu runs this block on the CPU against the checker; comment markers only)
// one thread per (block, row): 32 / size consecutive threads cover consecutive rows of a block; each adds its row into out[block]
__global__ void __launch_bounds__(256)
pixelutils_sad_kernel(int bits, const uint8_t *f1, long long stride1, const uint8_t *f2, long long stride2, const int64_t *off1,
                      const int64_t *off2, long long n, int *out)
{
    const int size = 1 << bits;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long b = t >> bits;
    if (b >= n) return;
    const int row = (int)(t & (size - 1));
    const uint8_t *a = f1 + off1[b] + row * stride1, *c = f2 + off2[b] + row * stride2;
    int sum = 0;
    for (int x = 0; x < size; x++) sum += abs((int)a[x] - (int)c[x]);
    atomicAdd(out + b, sum);
}
// [/device-code pixelutils]

int host_sad(int bits, const uint8_t *src1, ptrdiff_t stride1, const uint8_t *src2, ptrdiff_t stride2)
{
    const int size = 1 << bits;
    const size_t pitch = 32;
    B200HostCall call("av_pixelutils_sad_fn", nullptr, 2 * pitch * 32 + 64);
    uint8_t *d1 = call.scratch, *d2 = call.scratch + pitch * 32;
    int64_t *offs = (int64_t *)(call.scratch + 2 * pitch * 32);
    int *dout = (int *)(offs + 2);
    cudaStream_t st = call.stream;
    call.check(b200_h2d_rows(d1, pitch, src1, stride1, size, size, st), "h2d");
    call.check(b200_h2d_rows(d2, pitch, src2, stride2, size, size, st), "h2d");
    call.check(cudaMemsetAsync(offs, 0, 24, st), "memset");
    pixelutils_sad_kernel<<<1, 32, 0, st>>>(bits, d1, (long long)pitch, d2, (long long)pitch, offs, offs + 1, 1, dout);
    B200_LAUNCHED();
    call.launched();
    int res = 0;
    call.check(cudaMemcpyAsync(&res, dout, 4, cudaMemcpyDeviceToHost, st), "d2h");
    call.sync();
    return res;
}

template <int BITS> int tab_sad(const uint8_t *src1, ptrdiff_t stride1, const uint8_t *src2, ptrdiff_t stride2)
{
    return host_sad(BITS, src1, stride1, src2, stride2);
}

} // namespace

B200_API b200_pixelutils_sad_fn b200_pixelutils_get_sad_fn(int w_bits, int h_bits, int aligned, void *log_ctx)
{
    (void)aligned; (void)log_ctx;
    static const b200_pixelutils_sad_fn tab[5] = { tab_sad<1>, tab_sad<2>, tab_sad<3>, tab_sad<4>, tab_sad<5> };
    if (w_bits < 1 || w_bits > 5 || h_bits < 1 || h_bits > 5) return nullptr;     // pixelutils.c:94-98
    if (w_bits != h_bits) return nullptr;
    if (!b200_default_device()) return nullptr;
    return tab[w_bits - 1];
}

B200_API int b200_pixelutils_sad_batch_device(B200Device *dev, int w_bits, const uint8_t *frame1, ptrdiff_t stride1, const uint8_t *frame2,
                                              ptrdiff_t stride2, const int64_t *off1, const int64_t *off2, int64_t n, int32_t *out)
{
    if (int r = b200_use_device(dev)) return r;
    if (w_bits < 1 || w_bits > 5 || n < 0) return B200_EINVAL;
    if (n == 0) return 0;
    if (!frame1 || !frame2 || !off1 || !off2 || !out) return B200_EINVAL;
    const long long threads = n << w_bits, grid = (threads + 255) / 256;
    if (grid > 0x7fffffffLL) return B200_EINVAL;
    B200_CUDA_OK(cudaMemsetAsync(out, 0, (size_t)n * 4, dev->stream));
    pixelutils_sad_kernel<<<(unsigned)grid, 256, 0, dev->stream>>>(w_bits, frame1, (long long)stride1, frame2, (long long)stride2, off1, off2, n, out);
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}
