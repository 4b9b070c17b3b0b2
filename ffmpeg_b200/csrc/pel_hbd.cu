// pel_hbd.cu — libavcodec motion compensation for samples above 8 bits (uint16 pixels) on sm_90a: h264qpel for 9, 10, 12 and 14 bit (the
// tables ff_h264qpel_init(c, depth) installs for depth > 8 (libavcodec/h264qpel.c:50-104; h264qpel_template.c instantiated with BIT_DEPTH 9 / 10 / 12 / 14, :30-46).
//
// Reference semantics reproduced bit for bit (checker: the 16-bit qpel part of oracle/pel_oracle.c, pinned on the compiled reference):
//   H264_LOWPASS h / v / hv   libavcodec/h264qpel_template.c:77-305   taps (1,-5,20,20,-5,1); h and v: clip((t + 16) >> 5); hv: the unrounded
//                             horizontal sums over size + 5 rows, then the vertical taps and clip((t + 512) >> 10).  The 10-bit build
//                             offsets the int16 intermediate by -10 * 1023 and takes it out again (:131, :146-160): no value changes.
//   H264_MC mc00 .. mc33      :313-456   which of {full, h-half, v-half, centre} a quarter position averages, (a + b + 1) >> 1
//   put / avg                 :461-465   avg: dst = (dst + value + 1) >> 1;   clip = av_clip_uintp2(v, BIT_DEPTH) (bit_depth_template.c)
// This is the plain version (the 8-bit path in pel.cu carries the tuned kernels): 16-bit content is a small share of H.264 streams.
#include "common.h"
#include "pel_hbd.h"
#include <cstring>

namespace {

constexpr int HB_WARPS = 8;

__device__ __forceinline__ int tap6(int a, int b, int c, int d, int e, int f) { return a - 5 * b + 20 * (c + d) - 5 * e + f; }

struct HbWin {
    const unsigned short *w;           // sample (0, 0) of the block
    long long st;                      // line pitch in samples
    int maxv;
    __device__ __forceinline__ int clip(int v) const { return min(max(v, 0), maxv); }
    __device__ __forceinline__ int F(int x, int y) const { return w[y * st + x]; }
    __device__ __forceinline__ int hraw(int x, int y) const
    {
        const unsigned short *p = w + y * st + x;
        return tap6(p[-2], p[-1], p[0], p[1], p[2], p[3]);
    }
    __device__ __forceinline__ int H(int x, int y) const { return clip((hraw(x, y) + 16) >> 5); }
    __device__ __forceinline__ int V(int x, int y) const
    {
        const unsigned short *p = w + y * st + x;
        return clip((tap6(p[-2 * st], p[-st], p[0], p[st], p[2 * st], p[3 * st]) + 16) >> 5);
    }
    __device__ __forceinline__ int J(int x, int y) const
    {
        return clip((tap6(hraw(x, y - 2), hraw(x, y - 1), hraw(x, y), hraw(x, y + 1), hraw(x, y + 2), hraw(x, y + 3)) + 512) >> 10);
    }
};

// op byte as in b200_h264qpel_batch_device: bit0 avg, bits1-2 size index, bits3-6 position x + 4 y; offsets and stride in BYTES.
// A warp per operation, a lane per pixel (size^2 / 32 rounds); the taps come straight from the reference picture (the window of a
// block stays in L1 for its 8 rounds): no shared memory, no synchronisation, every thread is independent.
// (tests/test_cuda_emu.py runs this whole file, host code included, on the CPU against the checker)
__global__ void __launch_bounds__(32 * HB_WARPS)
qpel_hbd_kernel(long long n, const uint8_t *__restrict__ op, uint8_t *dst, const long long *__restrict__ dst_off, const uint8_t *src,
                const long long *__restrict__ src_off, long long stride, int depth)
{
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long st = stride / 2;
    for (long long i = (long long)blockIdx.x * HB_WARPS + warp; i < n; i += (long long)gridDim.x * HB_WARPS) {
        const int o = op[i], avg = o & 1, ls = 4 - ((o >> 1) & 3), size = 1 << ls, qx = (o >> 3) & 3, qy = (o >> 5) & 3;
        unsigned short *dp = reinterpret_cast<unsigned short *>(dst + dst_off[i]);
        const HbWin W{ reinterpret_cast<const unsigned short *>(src + src_off[i]), st, (1 << depth) - 1 };
        for (int p = lane; p < size * size; p += 32) {
            const int y = p >> ls, x = p & (size - 1);
            int v;
            if (qy == 0)               v = qx == 0 ? W.F(x, y) : qx == 2 ? W.H(x, y) : (W.F(x + (qx == 3), y) + W.H(x, y) + 1) >> 1;
            else if (qx == 0)          v = qy == 2 ? W.V(x, y) : (W.F(x, y + (qy == 3)) + W.V(x, y) + 1) >> 1;
            else if (qx == 2 && qy == 2) v = W.J(x, y);
            else if (qx == 2)          v = (W.H(x, y + (qy == 3)) + W.J(x, y) + 1) >> 1;              // mc21, mc23
            else if (qy == 2)          v = (W.V(x + (qx == 3), y) + W.J(x, y) + 1) >> 1;              // mc12, mc32
            else                       v = (W.H(x, y + (qy == 3)) + W.V(x + (qx == 3), y) + 1) >> 1;   // mc11, mc31, mc13, mc33
            unsigned short *d = dp + y * st + x;
            *d = (unsigned short)(avg ? (*d + v + 1) >> 1 : v);
        }
    }
}

int hbd_launch(cudaStream_t st, int depth, long long n, const uint8_t *op, uint8_t *dst, const long long *doff, const uint8_t *src,
               const long long *soff, long long stride)
{
    if (n <= 0) return 0;
    long long blocks = (n + HB_WARPS - 1) / HB_WARPS;
    if (blocks > 132 * 32) blocks = 132 * 32;        // 32 CTAs per SM of an H100 (132 SMs); the kernel strides over the rest
    qpel_hbd_kernel<<<(unsigned)blocks, 32 * HB_WARPS, 0, st>>>(n, op, dst, doff, src, soff, stride, depth);
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

// h264chroma for 16-bit samples (h264chroma_template.c:27-176 with BIT_DEPTH 16, what ff_h264chroma_init installs for every depth above 8,
// h264chroma.c:45-50): bilinear eighth-pel (A p00 + B p01 + C p10 + D p11 + 32) >> 6 with A = (8-x)(8-y), B = x(8-y), C = (8-x)y, D = xy;
// like the reference the D == 0 / B + C == 0 forms do not read the unused row / column.  op byte: bit0 avg, bits1-2 width index
// (0: 8, 1: 4, 2: 2); h[i] rows; xy[i] = x | y << 3; offsets and stride in BYTES.  A warp per block, a lane per pixel.
__global__ void __launch_bounds__(32 * HB_WARPS)
chroma_hbd_kernel(long long n, const uint8_t *__restrict__ op, const uint8_t *__restrict__ hh, const uint8_t *__restrict__ xy, uint8_t *dst,
                  const long long *__restrict__ dst_off, const uint8_t *src, const long long *__restrict__ src_off, long long stride)
{
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long st = stride / 2;
    for (long long i = (long long)blockIdx.x * HB_WARPS + warp; i < n; i += (long long)gridDim.x * HB_WARPS) {
        const int o = op[i], avg = o & 1, lw = 3 - ((o >> 1) & 3), w = 1 << lw, h = hh[i], x = xy[i] & 7, y = (xy[i] >> 3) & 7;
        const int A = (8 - x) * (8 - y), B = x * (8 - y), C = (8 - x) * y, D = x * y, E = B + C;
        const unsigned short *sp = reinterpret_cast<const unsigned short *>(src + src_off[i]);
        unsigned short *dp = reinterpret_cast<unsigned short *>(dst + dst_off[i]);
        const long long step = C ? st : 1;
        for (int p = lane; p < w * h; p += 32) {
            const int py = p >> lw, px = p & (w - 1);
            const unsigned short *s = sp + py * st + px;
            int v;
            if (D)      v = A * s[0] + B * s[1] + C * s[st] + D * s[st + 1];
            else if (E) v = A * s[0] + E * s[step];
            else        v = A * s[0];
            v = (v + 32) >> 6;
            unsigned short *d = dp + py * st + px;
            *d = (unsigned short)(avg ? (*d + v + 1) >> 1 : v);
        }
    }
}

int chroma_hbd_launch(cudaStream_t st, long long n, const uint8_t *op, const uint8_t *h, const uint8_t *xy, uint8_t *dst, const long long *doff,
                      const uint8_t *src, const long long *soff, long long stride)
{
    if (n <= 0) return 0;
    long long blocks = (n + HB_WARPS - 1) / HB_WARPS;
    if (blocks > 132 * 32) blocks = 132 * 32;        // 32 CTAs per SM of an H100 (132 SMs); the kernel strides over the rest
    chroma_hbd_kernel<<<(unsigned)blocks, 32 * HB_WARPS, 0, st>>>(n, op, h, xy, dst, doff, src, soff, stride);
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

void hbd_die(const char *what)
{
    fprintf(stderr, "libb200dsp: high-bit-depth motion compensation failed: %s (%s)\n", what, b200_last_error());
    abort();
}

// one block through the device for the drop-in tables: only the rectangle the reference function itself reads is copied
template <int DEPTH, int AVG, int SIDX, int POS>
void qpel_hbd_tab(uint8_t *dst, const uint8_t *src, ptrdiff_t stride)
{
    constexpr int X = POS & 3, Y = POS >> 2, size = 16 >> SIDX;
    constexpr int bx = X ? 2 : 0, ax = X ? 3 : 0, by = Y ? 2 : 0, ay = Y ? 3 : 0;
    B200Device *dev = b200_default_device();
    if (!dev) hbd_die("no device");
    if (cudaSetDevice(dev->ordinal) != cudaSuccess) hbd_die("cudaSetDevice");
    const size_t pitch = 64;                                       // 21 samples of 2 bytes
    const int sh = size + 5;
    B200_LOCK_DEVICE(dev);
    uint8_t *scr = (uint8_t *)b200_scratch(dev, pitch * (sh + size) + 256);
    if (!scr) hbd_die("scratch");
    uint8_t *dsrc = scr, *ddst = scr + pitch * sh, *meta = scr + pitch * (sh + size);
    cudaStream_t st = dev->stream;
    if (b200_h2d_rows(dsrc + (2 - by) * pitch + (2 - bx) * 2, pitch, src - by * stride - bx * 2, stride, (size + bx + ax) * 2, size + by + ay, st) != cudaSuccess)
        hbd_die("h2d src");
    if (b200_h2d_rows(ddst, pitch, dst, stride, size * 2, size, st) != cudaSuccess) hbd_die("h2d dst");
    struct { long long doff, soff; uint8_t op; } m = { 0, (long long)(2 * pitch + 4), (uint8_t)(AVG | (SIDX << 1) | (POS << 3)) };
    if (cudaMemcpyAsync(meta, &m, sizeof(m), cudaMemcpyHostToDevice, st) != cudaSuccess) hbd_die("h2d meta");
    if (hbd_launch(st, DEPTH, 1, meta + 16, ddst, (const long long *)meta, dsrc, (const long long *)meta + 1, (long long)pitch) < 0) hbd_die("launch");
    if (b200_d2h_rows(dst, stride, ddst, pitch, size * 2, size, st) != cudaSuccess) hbd_die("d2h");
    if (cudaStreamSynchronize(st) != cudaSuccess) hbd_die("sync");
}

template <int DEPTH, int AVG, int SIDX>
void fill16(b200_qpel_mc_func *t)
{
    t[0] = qpel_hbd_tab<DEPTH, AVG, SIDX, 0>;   t[1] = qpel_hbd_tab<DEPTH, AVG, SIDX, 1>;   t[2] = qpel_hbd_tab<DEPTH, AVG, SIDX, 2>;
    t[3] = qpel_hbd_tab<DEPTH, AVG, SIDX, 3>;   t[4] = qpel_hbd_tab<DEPTH, AVG, SIDX, 4>;   t[5] = qpel_hbd_tab<DEPTH, AVG, SIDX, 5>;
    t[6] = qpel_hbd_tab<DEPTH, AVG, SIDX, 6>;   t[7] = qpel_hbd_tab<DEPTH, AVG, SIDX, 7>;   t[8] = qpel_hbd_tab<DEPTH, AVG, SIDX, 8>;
    t[9] = qpel_hbd_tab<DEPTH, AVG, SIDX, 9>;   t[10] = qpel_hbd_tab<DEPTH, AVG, SIDX, 10>; t[11] = qpel_hbd_tab<DEPTH, AVG, SIDX, 11>;
    t[12] = qpel_hbd_tab<DEPTH, AVG, SIDX, 12>; t[13] = qpel_hbd_tab<DEPTH, AVG, SIDX, 13>; t[14] = qpel_hbd_tab<DEPTH, AVG, SIDX, 14>;
    t[15] = qpel_hbd_tab<DEPTH, AVG, SIDX, 15>;
}
template <int DEPTH>
void fill_ctx(B200H264QpelContext *c)
{
    fill16<DEPTH, 0, 0>(c->put_h264_qpel_pixels_tab[0]); fill16<DEPTH, 0, 1>(c->put_h264_qpel_pixels_tab[1]); fill16<DEPTH, 0, 2>(c->put_h264_qpel_pixels_tab[2]);
    fill16<DEPTH, 1, 0>(c->avg_h264_qpel_pixels_tab[0]); fill16<DEPTH, 1, 1>(c->avg_h264_qpel_pixels_tab[1]); fill16<DEPTH, 1, 2>(c->avg_h264_qpel_pixels_tab[2]);
}

// h264_chroma_mc_func for 16-bit samples: one block through the device; only the rectangle the reference function reads is copied
template <int AVG, int IDX>
void chroma_hbd_tab(uint8_t *dst, const uint8_t *src, ptrdiff_t stride, int h, int x, int y)
{
    if ((unsigned)x > 7 || (unsigned)y > 7) hbd_die("h264chroma: x, y must be in 0..7");     // av_assert2 in the reference
    if (h <= 0) return;
    constexpr int w = 8 >> IDX;
    B200Device *dev = b200_default_device();
    if (!dev) hbd_die("no device");
    if (cudaSetDevice(dev->ordinal) != cudaSuccess) hbd_die("cudaSetDevice");
    const size_t pitch = 32;                                       // 9 samples of 2 bytes
    const int ax = x ? 1 : 0, ay = y ? 1 : 0;
    B200_LOCK_DEVICE(dev);
    uint8_t *scr = (uint8_t *)b200_scratch(dev, pitch * (size_t)(2 * h + 1) + 256);
    if (!scr) hbd_die("scratch");
    uint8_t *dsrc = scr, *ddst = scr + pitch * (size_t)(h + 1), *meta = ddst + pitch * (size_t)h;
    cudaStream_t st = dev->stream;
    if (b200_h2d_rows(dsrc, pitch, src, stride, (size_t)(w + ax) * 2, (size_t)(h + ay), st) != cudaSuccess) hbd_die("h2d src");
    if (b200_h2d_rows(ddst, pitch, dst, stride, (size_t)w * 2, (size_t)h, st) != cudaSuccess) hbd_die("h2d dst");
    struct { long long doff, soff; uint8_t op, h, xy; } m = { 0, 0, (uint8_t)(AVG | (IDX << 1)), (uint8_t)h, (uint8_t)(x | (y << 3)) };
    if (cudaMemcpyAsync(meta, &m, sizeof(m), cudaMemcpyHostToDevice, st) != cudaSuccess) hbd_die("h2d meta");
    if (chroma_hbd_launch(st, 1, meta + 16, meta + 17, meta + 18, ddst, (const long long *)meta, dsrc, (const long long *)meta + 1, (long long)pitch) < 0) hbd_die("launch");
    if (b200_d2h_rows(dst, stride, ddst, pitch, (size_t)w * 2, (size_t)h, st) != cudaSuccess) hbd_die("d2h");
    if (cudaStreamSynchronize(st) != cudaSuccess) hbd_die("sync");
}

} // namespace

bool pel_hbd_fill(B200H264QpelContext *c, int bit_depth)
{
    switch (bit_depth) {
    case 9:  fill_ctx<9>(c);  return true;
    case 10: fill_ctx<10>(c); return true;
    case 12: fill_ctx<12>(c); return true;
    case 14: fill_ctx<14>(c); return true;
    }
    return false;
}

B200_API int b200_h264qpel_hbd_batch_device(B200Device *dev, int bit_depth, int64_t n, const uint8_t *op, uint8_t *dst, const int64_t *dst_off,
                                            const uint8_t *src, const int64_t *src_off, ptrdiff_t stride)
{
    if (!dev || n < 0 || !op || !dst || !dst_off || !src || !src_off) return B200_EINVAL;
    if (bit_depth != 9 && bit_depth != 10 && bit_depth != 12 && bit_depth != 14) return B200_ENOSYS;
    if ((stride & 1) || ((reinterpret_cast<uintptr_t>(dst) | reinterpret_cast<uintptr_t>(src)) & 1)) return B200_EINVAL;
    if (n == 0) return 0;
    B200_CUDA_OK(cudaSetDevice(dev->ordinal));
    return hbd_launch(dev->stream, bit_depth, n, op, dst, (const long long *)dst_off, src, (const long long *)src_off, (long long)stride);
}

void pel_hbd_fill_chroma(B200H264ChromaContext *c)
{
    memset(c, 0, sizeof(*c));                                      // entry [3] stays NULL like the reference's
    c->put_h264_chroma_pixels_tab[0] = chroma_hbd_tab<0, 0>; c->put_h264_chroma_pixels_tab[1] = chroma_hbd_tab<0, 1>; c->put_h264_chroma_pixels_tab[2] = chroma_hbd_tab<0, 2>;
    c->avg_h264_chroma_pixels_tab[0] = chroma_hbd_tab<1, 0>; c->avg_h264_chroma_pixels_tab[1] = chroma_hbd_tab<1, 1>; c->avg_h264_chroma_pixels_tab[2] = chroma_hbd_tab<1, 2>;
}

B200_API int b200_h264chroma_hbd_batch_device(B200Device *dev, int64_t n, const uint8_t *op, const uint8_t *h, const uint8_t *xy, uint8_t *dst,
                                              const int64_t *dst_off, const uint8_t *src, const int64_t *src_off, ptrdiff_t stride)
{
    if (!dev || n < 0 || !op || !h || !xy || !dst || !dst_off || !src || !src_off) return B200_EINVAL;
    if ((stride & 1) || ((reinterpret_cast<uintptr_t>(dst) | reinterpret_cast<uintptr_t>(src)) & 1)) return B200_EINVAL;
    if (n == 0) return 0;
    B200_CUDA_OK(cudaSetDevice(dev->ordinal));
    return chroma_hbd_launch(dev->stream, n, op, h, xy, dst, (const long long *)dst_off, src, (const long long *)src_off, (long long)stride);
}
