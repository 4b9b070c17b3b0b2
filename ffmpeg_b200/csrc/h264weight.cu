// h264weight.cu — libavcodec H.264 explicit weighted prediction on sm_90a for 8, 9, 10, 12 and 14 bit samples: weight_pixels_tab /
// biweight_pixels_tab of H264DSPContext as ff_h264dsp_init(c, depth, ...) installs them (libavcodec/h264dsp.c:103-110).
//
// Reference semantics reproduced bit-for-bit (checker: oracle/pel_oracle.c):
//   weight_h264_pixels{16,8,4,2}_<depth>_c     libavcodec/h264dsp_template.c:30-62    block = clip((block*w + o') >> d)
//   biweight_h264_pixels{16,8,4,2}_<depth>_c   libavcodec/h264dsp_template.c:63-93    dst = clip((src*ws + dst*wd + o'') >> (d+1))
// with o' = (O << d) + (d ? 1 << (d-1) : 0), o'' = ((O + 1) | 1) << d and O = o << (depth - 8), all in 32-bit integers; clip to the
// sample depth.  Samples are uint8 at 8 bits, uint16 above.
//
// Batched kernel: one warp per block, a lane owns 4 consecutive samples of a row (one 4-sample word access when the row is aligned to it).
#include "common.h"
#include <cstring>
#include <type_traits>

namespace {

constexpr int WARPS = 4;

// params per block: p[0] = idx (width 16 >> idx) | height << 8 | log2_denom << 16, p[1] = weight (dst weight for biweight),
//                   p[2] = source weight (biweight only), p[3] = offset.  Offsets and stride in bytes.
// P = uint8_t (depth 8) or uint16_t (9 / 10 / 12 / 14).
template <typename P, bool BI>
__global__ void __launch_bounds__(32 * WARPS)
h264_weight_kernel(long long n, const int32_t *params, uint8_t *dst, const int64_t *dst_off, const uint8_t *src, const int64_t *src_off,
                   long long stride, int depth)
{
    using Word = std::conditional_t<sizeof(P) == 1, unsigned, unsigned long long>;     // 4 samples
    constexpr int BITS = 8 * sizeof(P);
    const long long i = (long long)blockIdx.x * WARPS + (threadIdx.x >> 5);
    if (i >= n) return;
    const int lane = threadIdx.x & 31;
    if (sizeof(P) == 1) depth = 8;
    int4 p;                                                            // the 8-bit entry requires 16-byte-aligned params, the 16-bit one does not
    if (sizeof(P) == 1) p = __ldg(reinterpret_cast<const int4 *>(params) + i);
    else p = make_int4(__ldg(params + 4 * i), __ldg(params + 4 * i + 1), __ldg(params + 4 * i + 2), __ldg(params + 4 * i + 3));
    const int w = 16 >> (p.x & 3), h = (p.x >> 8) & 255, d = (p.x >> 16) & 31, maxv = (1 << depth) - 1;
    const int wd = p.y, ws = p.z, o = (int)((unsigned)p.w << (depth - 8));
    int off;
    if (BI) off = (int)((unsigned)((o + 1) | 1) << d);
    else { off = (int)((unsigned)o << d); if (d) off += 1 << (d - 1); }
    const int sh = BI ? d + 1 : d;
    const long long st = stride / (long long)sizeof(P);
    P *dp = reinterpret_cast<P *>(dst + __ldg(dst_off + i));
    const P *sp = BI ? reinterpret_cast<const P *>(src + __ldg(src_off + i)) : nullptr;
    const int segs = w > 4 ? w >> 2 : 1, npx = w < 4 ? w : 4;          // 4-sample segments per row
    for (int k = lane; k < h * segs; k += 32) {
        const int y = k / segs, x0 = (k - y * segs) * 4;
        P *q = dp + y * st + x0;
        const P *r = BI ? sp + y * st + x0 : nullptr;
        if (npx == 4 && reinterpret_cast<uintptr_t>(q) % sizeof(Word) == 0 && (!BI || reinterpret_cast<uintptr_t>(r) % sizeof(Word) == 0)) {
            const Word a = *reinterpret_cast<const Word *>(q);
            const Word b = BI ? __ldg(reinterpret_cast<const Word *>(r)) : 0;
            Word out = 0;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const int pa = (P)(a >> (BITS * j)), pb = (P)(b >> (BITS * j));
                const int v = BI ? (pb * ws + pa * wd + off) >> sh : (pa * wd + off) >> sh;
                out |= (Word)__vimin_s32_relu(v, maxv) << (BITS * j);
            }
            *reinterpret_cast<Word *>(q) = out;
        } else {
            for (int j = 0; j < npx; j++) {
                const int pa = q[j], pb = BI ? (int)__ldg(r + j) : 0;
                q[j] = (P)__vimin_s32_relu(BI ? (pb * ws + pa * wd + off) >> sh : (pa * wd + off) >> sh, maxv);
            }
        }
    }
}

// src == nullptr: weight in place; else biweight
int launch(cudaStream_t st, int depth, long long n, const int32_t *params, uint8_t *dst, const int64_t *doff, const uint8_t *src,
           const int64_t *soff, long long stride)
{
    const long long blocks = (n + WARPS - 1) / WARPS;
    if (blocks > 0x7fffffffLL) return B200_EINVAL;
    const unsigned g = (unsigned)blocks;
    if (depth == 8 && src) h264_weight_kernel<uint8_t, true><<<g, 32 * WARPS, 0, st>>>(n, params, dst, doff, src, soff, stride, depth);
    else if (depth == 8)   h264_weight_kernel<uint8_t, false><<<g, 32 * WARPS, 0, st>>>(n, params, dst, doff, nullptr, nullptr, stride, depth);
    else if (src)          h264_weight_kernel<uint16_t, true><<<g, 32 * WARPS, 0, st>>>(n, params, dst, doff, src, soff, stride, depth);
    else                   h264_weight_kernel<uint16_t, false><<<g, 32 * WARPS, 0, st>>>(n, params, dst, doff, nullptr, nullptr, stride, depth);
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

// drop-in: one block through the device (host pointers)
template <int DEPTH>
void host_op(bool bi, int idx, uint8_t *dst, const uint8_t *src, ptrdiff_t stride, int height, int log2_denom, int wd, int ws, int offset)
{
    constexpr int BPS = DEPTH > 8 ? 2 : 1;                                // bytes per sample
    const char *feature = "h264 weighted prediction";
    if (height < 0 || height > 255 || log2_denom < 0 || log2_denom > 7) B200HostCall::fail(feature, "unsupported height / log2_denom");
    if (height == 0) return;
    const size_t wb = (size_t)(16 >> idx) * BPS, pitch = 16 * BPS;      // row bytes of the block, of the staging copy
    B200HostCall call(feature, nullptr, 2 * pitch * 256 + 256);
    uint8_t *scr = call.scratch;
    uint8_t *ddst = scr, *dsrc = scr + pitch * 256, *meta = scr + 2 * pitch * 256;
    cudaStream_t st = call.stream;
    call.check(b200_h2d_rows(ddst, pitch, dst, stride, wb, (size_t)height, st), "h2d dst");
    if (bi) call.check(b200_h2d_rows(dsrc, pitch, src, stride, wb, (size_t)height, st), "h2d src");
    struct { int32_t p[4]; int64_t doff, soff; } m = { { idx | (height << 8) | (log2_denom << 16), wd, ws, offset }, 0, 0 };
    call.check(cudaMemcpyAsync(meta, &m, sizeof(m), cudaMemcpyHostToDevice, st), "h2d meta");
    const int64_t *doff = (const int64_t *)(meta + 16), *soff = doff + 1;
    call.launched(launch(st, DEPTH, 1, (const int32_t *)meta, ddst, doff, bi ? dsrc : nullptr, soff, (long long)pitch));
    call.check(b200_d2h_rows(dst, stride, ddst, pitch, wb, (size_t)height, st), "d2h");
    call.sync();
}

template <int DEPTH, int IDX>
void weight_tab(uint8_t *block, ptrdiff_t stride, int height, int log2_denom, int weight, int offset)
{
    host_op<DEPTH>(false, IDX, block, nullptr, stride, height, log2_denom, weight, 0, offset);
}
template <int DEPTH, int IDX>
void biweight_tab(uint8_t *dst, uint8_t *src, ptrdiff_t stride, int height, int log2_denom, int weightd, int weights, int offset)
{
    host_op<DEPTH>(true, IDX, dst, src, stride, height, log2_denom, weightd, weights, offset);
}
template <int D>
void fill(B200H264WeightContext *c)
{
    c->weight_pixels_tab[0] = weight_tab<D, 0>; c->weight_pixels_tab[1] = weight_tab<D, 1>;
    c->weight_pixels_tab[2] = weight_tab<D, 2>; c->weight_pixels_tab[3] = weight_tab<D, 3>;
    c->biweight_pixels_tab[0] = biweight_tab<D, 0>; c->biweight_pixels_tab[1] = biweight_tab<D, 1>;
    c->biweight_pixels_tab[2] = biweight_tab<D, 2>; c->biweight_pixels_tab[3] = biweight_tab<D, 3>;
}

} // namespace

B200_API int b200_h264_weight_init(B200H264WeightContext *c, int bit_depth)
{
    if (!c) return B200_EINVAL;
    if (!b200_default_device()) return B200_ENODEV;
    switch (bit_depth) {
    case 8:  fill<8>(c);  return 0;
    case 9:  fill<9>(c);  return 0;
    case 10: fill<10>(c); return 0;
    case 12: fill<12>(c); return 0;
    case 14: fill<14>(c); return 0;
    }
    return B200_ENOSYS;
}

B200_API int b200_h264_weight_batch_device(B200Device *dev, int64_t n, const int32_t *params, uint8_t *dst, const int64_t *dst_off,
                                           const uint8_t *src, const int64_t *src_off, ptrdiff_t stride)
{
    if (!dev || n < 0 || !params || !dst || !dst_off || (src && !src_off)) return B200_EINVAL;
    if ((uintptr_t)params & 15) return B200_EINVAL;
    if (n == 0) return 0;
    if (int r = b200_use_device(dev)) return r;
    return launch(dev->stream, 8, n, params, dst, dst_off, src, src_off, (long long)stride);
}

B200_API int b200_h264_weight_hbd_batch_device(B200Device *dev, int bit_depth, int64_t n, const int32_t *params, uint8_t *dst, const int64_t *dst_off,
                                               const uint8_t *src, const int64_t *src_off, ptrdiff_t stride)
{
    if (!dev || n < 0 || !params || !dst || !dst_off || (src && !src_off)) return B200_EINVAL;
    if (bit_depth != 9 && bit_depth != 10 && bit_depth != 12 && bit_depth != 14) return B200_ENOSYS;
    if ((stride & 1) || ((reinterpret_cast<uintptr_t>(dst) | reinterpret_cast<uintptr_t>(src)) & 1)) return B200_EINVAL;
    if ((uintptr_t)params & 3) return B200_EINVAL;                     // the kernel reads params as int32
    if (n == 0) return 0;
    if (int r = b200_use_device(dev)) return r;
    return launch(dev->stream, bit_depth, n, params, dst, dst_off, src, src_off, (long long)stride);
}
