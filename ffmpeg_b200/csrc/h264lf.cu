// h264lf.cu — libavcodec's H.264 in-loop deblocking filters on sm_90a for 8, 9, 10, 12 and 14 bit samples: the loop-filter members of
// H264DSPContext as ff_h264dsp_init(c, depth, chroma_format_idc) installs them (libavcodec/h264dsp.h:48-73, libavcodec/h264dsp.c:109-158).
//
// Reference semantics reproduced bit for bit (checker: oracle/h264lf_oracle.c), libavcodec/h264dsp_template.c:
//   :103-152 h264_loop_filter_luma   :166-222 h264_loop_filter_luma_intra   :236-271 h264_loop_filter_chroma   :293-315 ..._chroma_intra
// and the v / h / mbaff / 4:2:2 wrappers around them (:153-165, :223-235, :272-292, :316-340), which only fix the walking direction and
// the number of lines per tc0 entry.  Above 8 bits the samples are uint16: alpha and beta are scaled by << (depth - 8), the luma tc0 by
// * (1 << (depth - 8)), the chroma tc is ((tc0 - 1U) << (depth - 8)) + 1, and results are clipped to the sample depth.  At 8 bits every
// one of these is the identity.
//
// Every line across an edge is independent of the other lines of that edge, so one thread filters one line: it reads p3..q3 and
// writes at most p2..q2.  Edges of one batch must not touch each other's pixels (the decoder's order — vertical edges of a
// macroblock before its horizontal ones, macroblocks in raster order — becomes one batch per independent set, e.g. per anti-diagonal).
#include "common.h"
#include <cstring>

namespace {

// [device-code h264lf] (tests/cuda_emu runs this block on the CPU against the checker; comment markers only)
struct LfShape { int intra, chroma, vert, iters; };
__host__ __device__ __forceinline__ LfShape lf_shape(int kind)
{
    // kind: 0 v_luma, 1 h_luma, 2 h_luma_mbaff, 3-5 their intra forms, 6 v_chroma, 7 h_chroma, 8 h_chroma_mbaff, 9-11 intra forms,
    //       12 / 13 h_chroma / h_chroma_mbaff of 4:2:2, 14 / 15 their intra forms
    LfShape s;
    s.intra = (kind >= 3 && kind <= 5) || (kind >= 9 && kind <= 11) || kind >= 14;
    s.chroma = kind >= 6;
    s.vert = kind == 0 || kind == 3 || kind == 6 || kind == 9;
    s.iters = kind < 6 ? ((kind == 2 || kind == 5) ? 2 : 4)
            : kind < 12 ? ((kind == 8 || kind == 11) ? 1 : 2)
            : ((kind == 12 || kind == 14) ? 4 : 2);
    return s;
}
__device__ __forceinline__ int lf_clip3(int v, int lo, int hi) { return min(max(v, lo), hi); }

// edge e: kinds[e], q0 of its first line at base + off[e] (bytes), alpha[e], beta[e] (the 8-bit table values), tc0 + 4 e; stride in bytes.
// P = uint8_t (depth 8) or uint16_t (9 / 10 / 12 / 14).  One thread per line; 16 thread slots per edge.
template <typename P>
__global__ void __launch_bounds__(128)
h264_loop_filter_kernel(long long nedges, const uint8_t *kinds, uint8_t *base, const int64_t *off, long long stride, const uint8_t *alphas,
                        const uint8_t *betas, const int8_t *tc0s, int depth)
{
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long e = t >> 4;
    const int line = (int)(t & 15);
    if (e >= nedges) return;
    const LfShape S = lf_shape(kinds[e]);
    if (line >= 4 * S.iters) return;
    const long long st = stride / (long long)sizeof(P);
    const long long xs = S.vert ? st : 1, ys = S.vert ? 1 : st;
    P *pix = reinterpret_cast<P *>(base + off[e]) + line * ys;
    if (sizeof(P) == 1) depth = 8;
    const int sh = depth - 8, maxv = (1 << depth) - 1;
    const int alpha = alphas[e] << sh, beta = betas[e] << sh;
    const int p0 = pix[-1 * xs], p1 = pix[-2 * xs], q0 = pix[0], q1 = pix[1 * xs];
    if (!(abs(p0 - q0) < alpha && abs(p1 - p0) < beta && abs(q1 - q0) < beta)) return;
    if (!S.intra) {
        const int raw = tc0s[4 * e + line / S.iters];
        const int t0 = S.chroma ? (int)(((unsigned)raw - 1u) << sh) + 1 : raw * (1 << sh);
        if (S.chroma ? t0 <= 0 : t0 < 0) return;
        int tc = t0;
        if (!S.chroma) {
            const int p2 = pix[-3 * xs], q2 = pix[2 * xs];
            if (abs(p2 - p0) < beta) {
                if (t0) pix[-2 * xs] = (P)(p1 + lf_clip3(((p2 + ((p0 + q0 + 1) >> 1)) >> 1) - p1, -t0, t0));
                tc++;
            }
            if (abs(q2 - q0) < beta) {
                if (t0) pix[xs] = (P)(q1 + lf_clip3(((q2 + ((p0 + q0 + 1) >> 1)) >> 1) - q1, -t0, t0));
                tc++;
            }
        }
        const int delta = lf_clip3((((q0 - p0) * 4) + (p1 - q1) + 4) >> 3, -tc, tc);
        pix[-xs] = (P)lf_clip3(p0 + delta, 0, maxv);
        pix[0] = (P)lf_clip3(q0 - delta, 0, maxv);
        return;
    }
    if (S.chroma) {
        pix[-xs] = (P)((2 * p1 + p0 + q1 + 2) >> 2);
        pix[0] = (P)((2 * q1 + q0 + p1 + 2) >> 2);
        return;
    }
    const int p2 = pix[-3 * xs], q2 = pix[2 * xs];
    if (abs(p0 - q0) < ((alpha >> 2) + 2)) {
        if (abs(p2 - p0) < beta) {
            const int p3 = pix[-4 * xs];
            pix[-1 * xs] = (P)((p2 + 2 * p1 + 2 * p0 + 2 * q0 + q1 + 4) >> 3);
            pix[-2 * xs] = (P)((p2 + p1 + p0 + q0 + 2) >> 2);
            pix[-3 * xs] = (P)((2 * p3 + 3 * p2 + p1 + p0 + q0 + 4) >> 3);
        } else
            pix[-1 * xs] = (P)((2 * p1 + p0 + q1 + 2) >> 2);
        if (abs(q2 - q0) < beta) {
            const int q3 = pix[3 * xs];
            pix[0 * xs] = (P)((p1 + 2 * p0 + 2 * q0 + 2 * q1 + q2 + 4) >> 3);
            pix[1 * xs] = (P)((p0 + q0 + q1 + q2 + 2) >> 2);
            pix[2 * xs] = (P)((2 * q3 + 3 * q2 + q1 + q0 + p0 + 4) >> 3);
        } else
            pix[0 * xs] = (P)((2 * q1 + q0 + p1 + 2) >> 2);
    } else {
        pix[-1 * xs] = (P)((2 * p1 + p0 + q1 + 2) >> 2);
        pix[0 * xs] = (P)((2 * q1 + q0 + p1 + 2) >> 2);
    }
}
// [/device-code h264lf]

int launch(cudaStream_t st, int depth, long long nedges, const uint8_t *kinds, uint8_t *pix, const int64_t *off, long long stride,
           const uint8_t *alpha, const uint8_t *beta, const int8_t *tc0)
{
    const long long threads = nedges * 16, grid = (threads + 127) / 128;
    if (grid > 0x7fffffffLL) return B200_EINVAL;
    if (depth == 8) h264_loop_filter_kernel<uint8_t><<<(unsigned)grid, 128, 0, st>>>(nedges, kinds, pix, off, stride, alpha, beta, tc0, depth);
    else            h264_loop_filter_kernel<uint16_t><<<(unsigned)grid, 128, 0, st>>>(nedges, kinds, pix, off, stride, alpha, beta, tc0, depth);
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

void die(const char *what)
{
    fprintf(stderr, "libb200dsp: h264 loop filter failed: %s (%s)\n", what, b200_last_error());
    abort();
}

// drop-in: one edge through the device (host pointers).  The touched window is 4 samples either side of the edge, 16 lines at most.
template <int DEPTH>
void host_op(int kind, uint8_t *pix, ptrdiff_t stride, int alpha, int beta, const int8_t *tc0)
{
    constexpr int BPS = DEPTH > 8 ? 2 : 1;                                // bytes per sample
    B200Device *dev = b200_default_device();
    if (!dev) die("no device");
    if (cudaSetDevice(dev->ordinal) != cudaSuccess) die("cudaSetDevice");
    const LfShape S = lf_shape(kind);
    const int lines = 4 * S.iters;                                        // the lines this edge has (4 per tc0 entry / iteration group)
    const int w = S.vert ? lines : 8, h = S.vert ? 8 : lines;             // window in samples: vert: `lines` columns x rows -4..3; else columns -4..3 x `lines` rows
    uint8_t *origin = S.vert ? pix - 4 * stride : pix - 4 * BPS;
    const size_t pitch = 16 * BPS;
    B200_LOCK_DEVICE(dev);      // scratch + stream are per device: one host-pointer call at a time (released on return)
    uint8_t *scr = (uint8_t *)b200_scratch(dev, pitch * 16 + 64);
    if (!scr) die("scratch");
    uint8_t *win = scr, *meta = scr + pitch * 16;
    cudaStream_t st = dev->stream;
    if (b200_h2d_rows(win, pitch, origin, stride, (size_t)w * BPS, (size_t)h, st) != cudaSuccess) die("h2d");
    struct { int64_t off; int8_t tc[4]; uint8_t kind, alpha, beta, pad; } m;
    m.off = S.vert ? 4 * (int64_t)pitch : 4 * BPS;
    for (int i = 0; i < 4; i++) m.tc[i] = tc0 ? tc0[i] : 0;
    m.kind = (uint8_t)kind; m.alpha = (uint8_t)alpha; m.beta = (uint8_t)beta; m.pad = 0;
    if (cudaMemcpyAsync(meta, &m, sizeof(m), cudaMemcpyHostToDevice, st) != cudaSuccess) die("h2d meta");
    if (launch(st, DEPTH, 1, meta + 12, win, (const int64_t *)meta, (long long)pitch, meta + 13, meta + 14, (const int8_t *)(meta + 8)) < 0) die("launch");
    if (b200_d2h_rows(origin, stride, win, pitch, (size_t)w * BPS, (size_t)h, st) != cudaSuccess) die("d2h");
    if (cudaStreamSynchronize(st) != cudaSuccess) die("sync");
}

template <int DEPTH, int KIND> void tab_tc(uint8_t *pix, ptrdiff_t stride, int alpha, int beta, int8_t *tc0) { host_op<DEPTH>(KIND, pix, stride, alpha, beta, tc0); }
template <int DEPTH, int KIND> void tab_intra(uint8_t *pix, ptrdiff_t stride, int alpha, int beta) { host_op<DEPTH>(KIND, pix, stride, alpha, beta, nullptr); }

template <int D>
void fill(B200H264LoopFilterContext *c, bool c422)
{
    c->v_loop_filter_luma = tab_tc<D, 0>; c->h_loop_filter_luma = tab_tc<D, 1>; c->h_loop_filter_luma_mbaff = tab_tc<D, 2>;
    c->v_loop_filter_luma_intra = tab_intra<D, 3>; c->h_loop_filter_luma_intra = tab_intra<D, 4>; c->h_loop_filter_luma_mbaff_intra = tab_intra<D, 5>;
    c->v_loop_filter_chroma = tab_tc<D, 6>;
    c->h_loop_filter_chroma = c422 ? tab_tc<D, 12> : tab_tc<D, 7>;
    c->h_loop_filter_chroma_mbaff = c422 ? tab_tc<D, 13> : tab_tc<D, 8>;
    c->v_loop_filter_chroma_intra = tab_intra<D, 9>;
    c->h_loop_filter_chroma_intra = c422 ? tab_intra<D, 14> : tab_intra<D, 10>;
    c->h_loop_filter_chroma_mbaff_intra = c422 ? tab_intra<D, 15> : tab_intra<D, 11>;
}

} // namespace

B200_API int b200_h264_loop_filter_init(B200H264LoopFilterContext *c, int bit_depth, int chroma_format_idc)
{
    if (!c) return B200_EINVAL;
    if (!b200_default_device()) return B200_ENODEV;
    const bool c422 = chroma_format_idc > 1;                             // h264dsp.c:116-132
    switch (bit_depth) {
    case 8:  fill<8>(c, c422);  return 0;
    case 9:  fill<9>(c, c422);  return 0;
    case 10: fill<10>(c, c422); return 0;
    case 12: fill<12>(c, c422); return 0;
    case 14: fill<14>(c, c422); return 0;
    }
    return B200_ENOSYS;
}

B200_API int b200_h264_loop_filter_batch_device(B200Device *dev, int64_t nedges, const uint8_t *kinds, uint8_t *pix, const int64_t *pix_off,
                                                ptrdiff_t stride, const uint8_t *alpha, const uint8_t *beta, const int8_t *tc0)
{
    if (!dev) dev = b200_default_device();
    if (!dev) return B200_ENODEV;
    if (nedges < 0 || stride < 0) return B200_EINVAL;
    if (nedges == 0) return 0;
    if (!kinds || !pix || !pix_off || !alpha || !beta || !tc0) return B200_EINVAL;
    B200_CUDA_OK(cudaSetDevice(dev->ordinal));
    return launch(dev->stream, 8, nedges, kinds, pix, pix_off, (long long)stride, alpha, beta, tc0);
}

B200_API int b200_h264_loop_filter_hbd_batch_device(B200Device *dev, int bit_depth, int64_t nedges, const uint8_t *kinds, uint8_t *pix,
                                                    const int64_t *pix_off, ptrdiff_t stride, const uint8_t *alpha, const uint8_t *beta, const int8_t *tc0)
{
    if (!dev) dev = b200_default_device();
    if (!dev) return B200_ENODEV;
    if (nedges < 0 || stride < 0 || (stride & 1)) return B200_EINVAL;
    if (bit_depth != 9 && bit_depth != 10 && bit_depth != 12 && bit_depth != 14) return B200_ENOSYS;
    if (nedges == 0) return 0;
    if (!kinds || !pix || !pix_off || !alpha || !beta || !tc0 || ((uintptr_t)pix & 1)) return B200_EINVAL;
    B200_CUDA_OK(cudaSetDevice(dev->ordinal));
    return launch(dev->stream, bit_depth, nedges, kinds, pix, pix_off, (long long)stride, alpha, beta, tc0);
}
