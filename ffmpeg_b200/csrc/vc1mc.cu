// vc1mc.cu — VC-1 / WMV3 inter prediction on sm_90a: put_ / avg_vc1_mspel_pixels_tab[2][16] and put_ / avg_no_rnd_vc1_chroma_pixels_tab
// of VC1DSPContext (libavcodec/vc1dsp.h:60-67) as ff_vc1dsp_init fills them (vc1dsp.c:962-1017), and a one-call-per-frame device entry
// that runs the decoder's progressive sequence of ff_vc1_mc_1mv, ff_vc1_mc_4mv_luma, ff_vc1_mc_4mv_chroma and ff_vc1_interp_mc
// (vc1_mc.c:172-836, :1004-1230) with the edge emulation, range reduction and intensity compensation fused into the reads.
//
// Reference semantics reproduced bit for bit (checker: oracle/vc1dsp_oracle.c):
//   mspel     vc1dsp.c:542-723, restated in mspel_px: the 1-D passes round with 32 (8 at the half phase) minus rnd horizontally and
//             minus 1 - rnd vertically; the 2-D pass filters vertically into int16 with shift (s[h] + s[v]) >> 1 and (1 << (shift - 1))
//             + rnd - 1, then horizontally with 64 - rnd and >> 7; dxy 0 is the plain copy
//   hpel      hpeldsp.c put_ / put_no_rnd_ / avg_ / avg_no_rnd_pixels: (a + b + 1 - rnd) >> 1, (a + b + c + d + 2 - rnd) >> 2
//   chroma    h264chroma put_ / avg_h264_chroma_mc8 (+ 32) for rnd 0, vc1dsp.c:780-877 no_rnd (+ 28) for rnd 1
//   avg       (dst + x + 1) >> 1 after the clip, in every family
// The bilinear hpel / chroma arithmetic is kept here (hpel_px, chroma_px) rather than taken from pel.cu, whose device functions are
// shaped around its own op layouts and 16-byte row loads.
//
// Frame kernel: one warp per op, four per CTA, each warp with its own shared memory and no CTA-wide barrier.  Per source the warp
// evaluates the decoder's edge test, stages the footprint the member reads (columns and rows -1 .. n + 1 only in a direction it
// filters) — through clamped coordinates with range reduction and the IC LUT of the window row's source-row parity where the test
// fires, straight from the plane where it does not — for a 1MV op the luma and both chroma windows in the same pass, then computes
// four output samples per item and stores them as 4-byte words (averaged with what the first source wrote for src[1]).  The drop-in
// members stage what the reference function reads in the device scratch and run vc1_mc_member_kernel, which uses the same sample functions.
#include "common.h"
#include <cstring>

namespace {

constexpr int kWarps = 4;
constexpr int kLumaPitch = 20, kLumaRows = 19;             // 17 + 2 mspel
constexpr int kChromaPitch = 12, kChromaRows = 9;
constexpr int kWarpSmem = kLumaPitch * kLumaRows + 2 * kChromaPitch * kChromaRows + 12;   // 608 bytes, a multiple of 16
constexpr int kMaxRefs = 2;
constexpr long long kChunkOps = 1LL << 20;                  // ops per launch

// vc1_mspel_{ver,hor}_filter_16bits / vc1_mspel_filter taps at -1, 0, 1, 2 for modes 0..3 (vc1dsp.c:547-583)
__constant__ int c_mspel_taps[4][4] = { { 0, 0, 0, 0 }, { -4, 53, 18, -3 }, { -1, 9, 9, -1 }, { -3, 18, 53, -4 } };

__device__ __forceinline__ int clip8(int v) { return min(max(v, 0), 255); }
__device__ __forceinline__ int avg2(int d, int v) { return (d + v + 1) >> 1; }

__device__ __forceinline__ int mspel_taps(const uint8_t *s, int step, int mode)
{
    const int *c = c_mspel_taps[mode];
    return c[0] * s[-step] + c[1] * s[0] + c[2] * s[step] + c[3] * s[2 * step];
}

// put_vc1_mspel_pixels_tab[*][hm + 4 vm] at the sample s (row pitch p), before the clip
__device__ __forceinline__ int mspel_px(const uint8_t *s, int p, int hm, int vm, int rnd)
{
    if (hm && vm) {
        const int shift = ((hm == 2 ? 1 : 5) + (vm == 2 ? 1 : 5)) >> 1, r = (1 << (shift - 1)) + rnd - 1;
        int t[4];
#pragma unroll
        for (int k = 0; k < 4; k++) t[k] = (int16_t)((mspel_taps(s + k - 1, p, vm) + r) >> shift);
        const int *c = c_mspel_taps[hm];
        return (c[0] * t[0] + c[1] * t[1] + c[2] * t[2] + c[3] * t[3] + 64 - rnd) >> 7;
    }
    if (vm) return (mspel_taps(s, p, vm) + (vm == 2 ? 8 : 32) - (1 - rnd)) >> (vm == 2 ? 4 : 6);
    if (hm) return (mspel_taps(s, 1, hm) + (hm == 2 ? 8 : 32) - rnd) >> (hm == 2 ? 4 : 6);
    return s[0];
}

// hpeldsp put_pixels_tab (rnd 0) / put_no_rnd_pixels_tab (rnd 1) at dxy = x half + 2 y half
__device__ __forceinline__ int hpel_px(const uint8_t *s, int p, int dxy, int rnd)
{
    switch (dxy) {
    case 1: return (s[0] + s[1] + 1 - rnd) >> 1;
    case 2: return (s[0] + s[p] + 1 - rnd) >> 1;
    case 3: return (s[0] + s[1] + s[p] + s[p + 1] + 2 - rnd) >> 2;
    }
    return s[0];
}

// eighth-sample bilinear chroma at (x, y) 0..7: bias 32 (h264chroma) or 28 (the VC-1 no_rnd form)
__device__ __forceinline__ int chroma_px(const uint8_t *s, int p, int x, int y, int bias)
{
    return ((8 - x) * (8 - y) * s[0] + x * (8 - y) * s[1] + (8 - x) * y * s[p] + x * y * s[p + 1] + bias) >> 6;
}

__device__ __forceinline__ uint32_t avg_word(uint32_t d, uint32_t w)
{
    uint32_t o = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) o |= (uint32_t)avg2((d >> (8 * k)) & 0xFF, (w >> (8 * k)) & 0xFF) << (8 * k);
    return o;
}

struct McArgs {
    const B200Vc1McOp *ops;
    long long nops;
    uint8_t *dst[3];
    long long ls_y, ls_uv;
    int mbw, mbh, H, V, nrefs;
    B200Vc1McRef refs[kMaxRefs];
};

// the device-side guard: an op it refuses writes nothing
__device__ __forceinline__ bool op_ok(const B200Vc1McOp &op, const McArgs &a)
{
    const int kind = op.kind, nsrc = op.flags & B200_VC1_MC_AVG ? 2 : 1;
    if (kind > B200_VC1_MC_CHROMA8 || (nsrc == 2 && kind != B200_VC1_MC_1MV)) return false;
#pragma unroll
    for (int s = 0; s < 2; s++) {
        const B200Vc1McSrc &S = op.src[s];
        if (s < nsrc && (S.ref >= a.nrefs || S.mx > 3 || S.my > 3 || S.uvmx > 3 || S.uvmy > 3)) return false;
    }
    const int n = kind == B200_VC1_MC_1MV ? 16 : 8, w = kind == B200_VC1_MC_CHROMA8 ? 8 * a.mbw : 16 * a.mbw;
    const int h = kind == B200_VC1_MC_CHROMA8 ? 8 * a.mbh : 16 * a.mbh;
    return op.dst_x >= 0 && op.dst_y >= 0 && !(op.dst_x & 7) && !(op.dst_y & 7) && op.dst_x + n <= w && op.dst_y + n <= h;
}

// the decoder's edge test for source s of op (vc1_mc.c:299-302 ff_vc1_mc_1mv, :1066-1068 ff_vc1_interp_mc, :563-566
// ff_vc1_mc_4mv_luma, :735-738 ff_vc1_mc_4mv_chroma); the comparisons are unsigned as there
__device__ __forceinline__ bool edge_fires(const B200Vc1McOp &op, const B200Vc1McSrc &S, int s, int ms, const B200Vc1McRef &R, int H, int V)
{
    if (R.rangeredfrm || R.use_ic) return true;
    if (op.kind == B200_VC1_MC_1MV) {
        const int xm = s ? 1 : ms;
        return H < 22 || V < 22 || (unsigned)(S.x - xm) > (unsigned)(H - S.mx - 16 - 3 * xm) || (unsigned)(S.y - 1) > (unsigned)(V - S.my - 19);
    }
    if (op.kind == B200_VC1_MC_LUMA8)
        return H < 13 || V < 23 || (unsigned)(S.x - ms) > (unsigned)(H - S.mx - 8 - 2 * ms) || (unsigned)(S.y - ms) > (unsigned)(V - S.my - 8 - 2 * ms);
    return H < 18 || V < 18 || (unsigned)S.uvx > (unsigned)((H >> 1) - 9) || (unsigned)S.uvy > (unsigned)((V >> 1) - 9);
}

// one window sample: source (yy, xx) of plane `base`, clamped with range reduction and the LUT of the source row's parity where the
// edge test fired
__device__ __forceinline__ uint8_t window_sample(const uint8_t *base, long long ls, int yy, int xx, int W, int Hh, bool fire, int rr,
                                                 const uint8_t (*lut)[256])
{
    if (!fire) return base[(long long)yy * ls + xx];
    int v = base[(long long)min(max(yy, 0), Hh - 1) * ls + min(max(xx, 0), W - 1)];
    if (rr) v = ((v - 128) >> 1) + 128;
    if (lut) v = lut[yy & 1][v];
    return (uint8_t)v;
}

__global__ void __launch_bounds__(32 * kWarps) vc1_mc_kernel(McArgs a)
{
    extern __shared__ uint32_t vc1_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long i = (long long)blockIdx.x * kWarps + warp;
    if (i >= a.nops) return;
    const B200Vc1McOp op = a.ops[i];
    if (!op_ok(op, a)) return;                                            // warp-uniform
    uint8_t *wy = reinterpret_cast<uint8_t *>(vc1_smem) + warp * kWarpSmem, *wu = wy + kLumaRows * kLumaPitch;
    uint8_t *wv = wu + kChromaRows * kChromaPitch;
    const int ms = op.flags & B200_VC1_MC_MSPEL ? 1 : 0, rnd = op.flags & B200_VC1_MC_RND ? 1 : 0;
    const bool luma = op.kind != B200_VC1_MC_CHROMA8, chroma = op.kind != B200_VC1_MC_LUMA8;
    const int n = op.kind == B200_VC1_MC_1MV ? 16 : 8, nl = luma ? n * n / 4 : 0, q = n / 4;
    const int cx = op.kind == B200_VC1_MC_CHROMA8 ? op.dst_x : op.dst_x / 2, cy = op.kind == B200_VC1_MC_CHROMA8 ? op.dst_y : op.dst_y / 2;
    const int nsrc = op.flags & B200_VC1_MC_AVG ? 2 : 1;
    for (int s = 0; s < nsrc; s++) {
        const B200Vc1McSrc S = a.ops[i].src[s];                          // from memory: a dynamic index into op would live on the stack
        const B200Vc1McRef &R = a.refs[S.ref];
        const bool fire = edge_fires(op, S, s, ms, R, a.H, a.V);
        if (luma) {                                                        // window (r, c) is source (y - ms + r, x - ms + c)
            const int c0 = ms && S.mx ? 0 : ms, c1 = ms ? (S.mx ? n + 3 : n + 1) : n + ((S.mx & 2) ? 1 : 0);
            const int r0 = ms && S.my ? 0 : ms, r1 = ms ? (S.my ? n + 3 : n + 1) : n + ((S.my & 2) ? 1 : 0);
            const int cols = c1 - c0, rows = r1 - r0, X = S.x - ms, Y = S.y - ms;
            for (int e = lane; e < rows * cols; e += 32) {
                const int r = r0 + e / cols, c = c0 + e % cols;
                wy[r * kLumaPitch + c] = window_sample(R.y, R.ls_y, Y + r, X + c, a.H, a.V, fire, R.rangeredfrm, R.use_ic ? R.luty : nullptr);
            }
        }
        if (chroma) {                                                      // window (r, c) is source (uvy + r, uvx + c)
            const int cols = 8 + (S.uvmx ? 1 : 0), rows = 8 + (S.uvmy ? 1 : 0);
            for (int e = lane; e < 2 * rows * cols; e += 32) {
                const int p = e >= rows * cols, f = e - p * rows * cols, r = f / cols, c = f % cols;
                (p ? wv : wu)[r * kChromaPitch + c] = window_sample(p ? R.v : R.u, R.ls_uv, S.uvy + r, S.uvx + c, a.H >> 1, a.V >> 1, fire,
                                                                    R.rangeredfrm, R.use_ic ? R.lutuv : nullptr);
            }
        }
        __syncwarp();
        for (int e = lane; e < nl + (chroma ? 32 : 0); e += 32) {
            uint32_t word = 0;
            uint8_t *d;
            if (e < nl) {
                const int y = e / q, x0 = (e - y * q) * 4;
                const uint8_t *src = wy + (y + ms) * kLumaPitch + x0 + ms;
                const int dxy = (S.my & 2) | ((S.mx & 2) >> 1);
#pragma unroll
                for (int k = 0; k < 4; k++)
                    word |= (uint32_t)(ms ? clip8(mspel_px(src + k, kLumaPitch, S.mx, S.my, rnd)) : hpel_px(src + k, kLumaPitch, dxy, rnd)) << (8 * k);
                d = a.dst[0] + (long long)(op.dst_y + y) * a.ls_y + op.dst_x + x0;
            } else {
                const int f = e - nl, p = f >> 4, y = (f & 15) >> 1, x0 = (f & 1) * 4;
                const uint8_t *src = (p ? wv : wu) + y * kChromaPitch + x0;
#pragma unroll
                for (int k = 0; k < 4; k++)
                    word |= (uint32_t)chroma_px(src + k, kChromaPitch, S.uvmx << 1, S.uvmy << 1, rnd ? 28 : 32) << (8 * k);
                d = a.dst[1 + p] + (long long)(cy + y) * a.ls_uv + cx + x0;
            }
            uint32_t *dw = reinterpret_cast<uint32_t *>(d);
            *dw = s ? avg_word(*dw, word) : word;
        }
        __syncwarp();
    }
}

cudaError_t launch(McArgs a, cudaStream_t st)
{
    const long long nops = a.nops;
    const B200Vc1McOp *ops = a.ops;
    for (long long b = 0; b < nops; b += kChunkOps) {
        a.ops = ops + b;
        a.nops = nops - b < kChunkOps ? nops - b : kChunkOps;
        const unsigned grid = (unsigned)((a.nops + kWarps - 1) / kWarps);
        vc1_mc_kernel<<<grid, 32 * kWarps, kWarps * kWarpSmem, st>>>(a);
        B200_LAUNCHED();
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// ---- drop-in members (host pointers): the samples the reference function reads are copied into a dense device window whose sample
// (1, 1) is the block's (0, 0), and for avg the destination block; one CTA computes the block with the frame kernel's sample functions
// and the block is copied back.
constexpr int kMemberPitch = 32;

__global__ void vc1_mc_member_kernel(const uint8_t *win, uint8_t *dst, int w, int h, int chroma, int hx, int vy, int rnd, int avg)
{
    for (int e = threadIdx.x; e < w * h; e += blockDim.x) {
        const int y = e / w, x = e - y * w;
        const uint8_t *s = win + (y + 1) * kMemberPitch + x + 1;
        int v = chroma ? chroma_px(s, kMemberPitch, hx, vy, 28) : clip8(mspel_px(s, kMemberPitch, hx, vy, rnd));
        if (avg) v = avg2(dst[y * kMemberPitch + x], v);
        dst[y * kMemberPitch + x] = (uint8_t)v;
    }
}

// footprint: columns c0 .. c1 - 1 and rows r0 .. r1 - 1 relative to the block's (0, 0)
void member_host(const char *what, uint8_t *dst, ptrdiff_t stride, const uint8_t *src, int w, int h, int chroma, int hx, int vy, int rnd,
                 int avg, int c0, int c1, int r0, int r1)
{
    const size_t wbytes = ((size_t)kMemberPitch * (r1 - r0 + 2) + 255) & ~(size_t)255, dbytes = (size_t)kMemberPitch * h;
    B200HostCall call(what, nullptr, wbytes + dbytes);
    uint8_t *dwin = call.scratch, *ddst = dwin + wbytes;
    cudaStream_t st = call.stream;
    call.check(b200_h2d_rows(dwin + (1 + r0) * kMemberPitch + 1 + c0, kMemberPitch, src + r0 * stride + c0, stride, (size_t)(c1 - c0),
                             (size_t)(r1 - r0), st), "h2d window");
    if (avg) call.check(b200_h2d_rows(ddst, kMemberPitch, dst, stride, (size_t)w, (size_t)h, st), "h2d dst");
    vc1_mc_member_kernel<<<1, 256, 0, st>>>(dwin, ddst, w, h, chroma, hx, vy, rnd, avg);
    B200_LAUNCHED();
    call.launched();
    call.check(b200_d2h_rows(dst, stride, ddst, kMemberPitch, (size_t)w, (size_t)h, st), "d2h");
    call.sync();
}

// put_ / avg_vc1_mspel_pixels_tab[size][HM + 4 VM]: n x n, reads columns -1 .. n + 1 only when HM filters and rows only when VM does
template <int N, int HM, int VM, int AVG>
void m_mspel(uint8_t *dst, const uint8_t *src, ptrdiff_t stride, int rnd)
{
    member_host("vc1 mspel member", dst, stride, src, N, N, 0, HM, VM, rnd, AVG, HM ? -1 : 0, HM ? N + 2 : N, VM ? -1 : 0, VM ? N + 2 : N);
}

// put_ / avg_no_rnd_vc1_chroma_pixels_tab[size]: W x h, reads (W + 1) x (h + 1)
template <int W, int AVG>
void m_chroma(uint8_t *dst, const uint8_t *src, ptrdiff_t stride, int h, int x, int y)
{
    if (h < 0 || h > 4096 || x < 0 || x > 7 || y < 0 || y > 7) {
        b200_set_error("vc1 chroma member: h %d outside 0..4096 or (x, y) = (%d, %d) outside 0..7", h, x, y);
        return;
    }
    if (!h) return;
    member_host("vc1 chroma member", dst, stride, src, W, h, 1, x, y, 0, AVG, 0, W + 1, 0, h + 1);
}

template <int N, int D>
void fill_dxy(B200VC1DSPContext *c, int i)
{
    c->put_vc1_mspel_pixels_tab[i][D] = m_mspel<N, (D & 3), (D >> 2), 0>;
    c->avg_vc1_mspel_pixels_tab[i][D] = m_mspel<N, (D & 3), (D >> 2), 1>;
    if constexpr (D < 15) fill_dxy<N, D + 1>(c, i);
}

} // namespace

void b200_vc1_fill_transforms(B200VC1DSPContext *c);                   // vc1idct.cu

B200_API int b200_vc1_dsp_init(B200VC1DSPContext *c)
{
    if (!c) { b200_set_error("vc1 dsp init: NULL context"); return B200_EINVAL; }
    if (!b200_default_device()) return B200_ENODEV;
    memset(c, 0, sizeof(*c));                                            // overlap, loop filter, sprite, start-code members: NULL
    fill_dxy<16, 0>(c, 0);
    fill_dxy<8, 0>(c, 1);
    c->put_no_rnd_vc1_chroma_pixels_tab[0] = m_chroma<8, 0>;
    c->avg_no_rnd_vc1_chroma_pixels_tab[0] = m_chroma<8, 1>;
    c->put_no_rnd_vc1_chroma_pixels_tab[1] = m_chroma<4, 0>;
    c->avg_no_rnd_vc1_chroma_pixels_tab[1] = m_chroma<4, 1>;
    b200_vc1_fill_transforms(c);
    return 0;
}

B200_API int b200_vc1_mc_frame_device(B200Device *dev, int nrefs, const B200Vc1McRef *refs, uint8_t *const dst[3], ptrdiff_t ls_y,
                                      ptrdiff_t ls_uv, int mb_width, int mb_height, int h_edge_pos, int v_edge_pos, int64_t nops,
                                      const B200Vc1McOp *ops)
{
    if (nops < 0 || nrefs < 1 || nrefs > kMaxRefs || mb_width < 1 || mb_height < 1 || mb_width > 2047 || mb_height > 2047 ||
        h_edge_pos < 1 || v_edge_pos < 1 || h_edge_pos > 32767 || v_edge_pos > 32767) {
        b200_set_error("vc1 mc frame: negative nops, nrefs outside 1..2, a macroblock count outside 1..2047 or an edge position outside 1..32767");
        return B200_EINVAL;
    }
    if (nops == 0) return 0;
    if (!refs || !ops || !dst || ((uintptr_t)ops & 3)) { b200_set_error("vc1 mc frame: NULL or misaligned refs / ops / dst"); return B200_EINVAL; }
    if ((ls_y & 3) || (ls_uv & 3)) { b200_set_error("vc1 mc frame: line size not a multiple of 4"); return B200_EINVAL; }
    for (int p = 0; p < 3; p++)
        if (!dst[p] || ((uintptr_t)dst[p] & 3)) { b200_set_error("vc1 mc frame: plane %d NULL or not 4-byte aligned", p); return B200_EINVAL; }
    McArgs a;
    memset(&a, 0, sizeof(a));
    for (int r = 0; r < nrefs; r++) {
        if (!refs[r].y || !refs[r].u || !refs[r].v) { b200_set_error("vc1 mc frame: reference %d has a NULL plane", r); return B200_EINVAL; }
        if (refs[r].interlaced) { b200_set_error("vc1 mc frame: reference %d is interlaced (not implemented)", r); return B200_ENOSYS; }
        a.refs[r] = refs[r];
    }
    if (int r = b200_use_device(dev)) return r;
    a.ops = ops;
    a.nops = (long long)nops;
    for (int p = 0; p < 3; p++) a.dst[p] = dst[p];
    a.ls_y = (long long)ls_y;
    a.ls_uv = (long long)ls_uv;
    a.mbw = mb_width;
    a.mbh = mb_height;
    a.H = h_edge_pos;
    a.V = v_edge_pos;
    a.nrefs = nrefs;
    B200_CUDA_OK(launch(a, dev->stream));
    return 0;
}
