// videodsp.cu — libavcodec VideoDSPContext on sm_90a: emulated_edge_mc for 8-bit and 16-bit samples (what ff_videodsp_init(c, bpc)
// installs: the 8-bit template up to 8 bits, the 16-bit one above, libavcodec/videodsp.c:32-62) and the empty prefetch.
//
// Reference semantics reproduced bit-for-bit (checker: oracle/pel_oracle.c):
//   ff_emulated_edge_mc_8 / _16   libavcodec/videodsp_template.c:24-101   a block_w x block_h window at (src_x, src_y) of a w x h picture;
//                                 samples outside the picture replicate the nearest border sample
//
// Batched kernel: a clamped gather, one warp per window, lanes across columns.
#include "common.h"
#include <algorithm>
#include <cstring>

namespace {

constexpr int WARPS = 4;

// P = uint8_t or uint16_t.  geom[4*i..] = block_w, block_h, src_x, src_y in samples; origin[i] = offset of that picture's sample (0, 0)
// from `src`; offsets and line sizes in bytes.
template <typename P>
__global__ void __launch_bounds__(32 * WARPS)
edge_kernel(long long n, uint8_t *buf, const int64_t *buf_off, long long buf_ls, const uint8_t *src, const int64_t *origin,
            long long src_ls, const int32_t *geom, int w, int h)
{
    const long long i = (long long)blockIdx.x * WARPS + (threadIdx.x >> 5);
    if (i >= n) return;
    const int lane = threadIdx.x & 31;
    int4 gm;                                                       // the 8-bit entry requires 16-byte-aligned geom, the 16-bit one does not
    if (sizeof(P) == 1) gm = __ldg(reinterpret_cast<const int4 *>(geom) + i);
    else gm = make_int4(__ldg(geom + 4 * i), __ldg(geom + 4 * i + 1), __ldg(geom + 4 * i + 2), __ldg(geom + 4 * i + 3));
    const int bw = gm.x, bh = gm.y, sx = gm.z, sy = gm.w;
    const uint8_t *pic = src + origin[i];
    uint8_t *out = buf + buf_off[i];
    for (int x = lane; x < bw; x += 32) {
        const int px = min(max(sx + x, 0), w - 1);
        for (int y = 0; y < bh; y++) {
            const int py = min(max(sy + y, 0), h - 1);
            *reinterpret_cast<P *>(out + (long long)y * buf_ls + (int)sizeof(P) * x) =
                __ldg(reinterpret_cast<const P *>(pic + (long long)py * src_ls + (int)sizeof(P) * px));
        }
    }
}

template <typename P>
int launch(cudaStream_t st, long long n, uint8_t *buf, const int64_t *buf_off, long long buf_ls, const uint8_t *src, const int64_t *origin,
           long long src_ls, const int32_t *geom, int w, int h)
{
    const long long blocks = (n + WARPS - 1) / WARPS;
    if (blocks > 0x7fffffffLL) return B200_EINVAL;
    edge_kernel<P><<<(unsigned)blocks, 32 * WARPS, 0, st>>>(n, buf, buf_off, buf_ls, src, origin, src_ls, geom, w, h);
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

// VideoDSPContext.emulated_edge_mc (host pointers): only the part of the picture the window reaches is copied
template <typename P>
void edge_tab(uint8_t *buf, const uint8_t *src, ptrdiff_t buf_linesize, ptrdiff_t src_linesize, int block_w, int block_h,
              int src_x, int src_y, int w, int h)
{
    constexpr int BPS = sizeof(P);                                 // bytes per sample
    if (!w || !h) return;                                          // videodsp_template.c:33-34
    if (block_w <= 0 || block_h <= 0) return;
    // the part of the picture the window can reach after clamping
    const int x0 = std::min(std::max(src_x, 0), w - 1), x1 = std::min(std::max(src_x + block_w - 1, 0), w - 1);
    const int y0 = std::min(std::max(src_y, 0), h - 1), y1 = std::min(std::max(src_y + block_h - 1, 0), h - 1);
    const size_t rw = (size_t)(x1 - x0 + 1) * BPS, rh = (size_t)(y1 - y0 + 1);
    const size_t rp = (rw + 15) & ~(size_t)15, bp = ((size_t)block_w * BPS + 15) & ~(size_t)15;
    B200HostCall call("emulated_edge_mc", nullptr, rp * rh + bp * block_h + 256);
    uint8_t *drect = call.scratch, *dbuf = drect + rp * rh, *meta = dbuf + bp * block_h;
    meta += (16 - ((uintptr_t)meta & 15)) & 15;
    cudaStream_t st = call.stream;
    const uint8_t *pic = src - (ptrdiff_t)src_y * src_linesize - (ptrdiff_t)src_x * BPS;
    call.check(b200_h2d_rows(drect, rp, pic + (ptrdiff_t)y0 * src_linesize + (ptrdiff_t)x0 * BPS, src_linesize, rw, rh, st), "h2d");
    struct { int32_t g[4]; int64_t boff, origin; } m = { { block_w, block_h, src_x, src_y }, 0, -((int64_t)y0 * (int64_t)rp + (int64_t)x0 * BPS) };
    call.check(cudaMemcpyAsync(meta, &m, sizeof(m), cudaMemcpyHostToDevice, st), "h2d meta");
    call.launched(launch<P>(st, 1, dbuf, (const int64_t *)(meta + 16), (long long)bp, drect, (const int64_t *)(meta + 24), (long long)rp,
                            (const int32_t *)meta, w, h));
    call.check(b200_d2h_rows(buf, buf_linesize, dbuf, bp, (size_t)block_w * BPS, (size_t)block_h, st), "d2h");
    call.sync();
}

void prefetch_nop(const uint8_t *, ptrdiff_t, int) {}

} // namespace

B200_API int b200_videodsp_init(B200VideoDSPContext *c, int bpc)
{
    if (!c) return B200_EINVAL;
    if (!b200_default_device()) return B200_ENODEV;
    c->emulated_edge_mc = bpc > 8 ? edge_tab<uint16_t> : edge_tab<uint8_t>;      // videodsp.c:41-45: the 16 bit template above 8
    c->prefetch = prefetch_nop;                                    // videodsp.c:34-36: the C prefetch is an empty function
    return 0;
}

B200_API int b200_emulated_edge_mc_batch_device(B200Device *dev, int64_t n, uint8_t *buf, const int64_t *buf_off,
                                                ptrdiff_t buf_linesize, const uint8_t *src, const int64_t *origin,
                                                ptrdiff_t src_linesize, const int32_t *geom, int w, int h)
{
    if (!dev || n < 0 || !buf || !buf_off || !src || !origin || !geom || w < 0 || h < 0) return B200_EINVAL;
    if (((uintptr_t)geom & 15) != 0) return B200_EINVAL;
    if (n == 0 || !w || !h) return 0;
    if (int r = b200_use_device(dev)) return r;
    return launch<uint8_t>(dev->stream, n, buf, buf_off, buf_linesize, src, origin, src_linesize, geom, w, h);
}

B200_API int b200_emulated_edge_mc_hbd_batch_device(B200Device *dev, int64_t n, uint8_t *buf, const int64_t *buf_off, ptrdiff_t buf_linesize,
                                                    const uint8_t *src, const int64_t *origin, ptrdiff_t src_linesize, const int32_t *geom, int w, int h)
{
    if (!dev || n < 0 || !buf || !buf_off || !src || !origin || !geom || w < 0 || h < 0) return B200_EINVAL;
    if (((buf_linesize | src_linesize) & 1) || ((reinterpret_cast<uintptr_t>(buf) | reinterpret_cast<uintptr_t>(src)) & 1)) return B200_EINVAL;
    if ((uintptr_t)geom & 3) return B200_EINVAL;                   // the kernel reads geom as int32
    if (n == 0 || !w || !h) return 0;
    if (int r = b200_use_device(dev)) return r;
    return launch<uint16_t>(dev->stream, n, buf, buf_off, buf_linesize, src, origin, src_linesize, geom, w, h);
}
