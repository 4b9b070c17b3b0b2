// hevcsao.cu — HEVC sample adaptive offset on sm_90a: the SAO members of HEVCDSPContext (libavcodec/hevc/dsp.h:47-125:
// sao_band_filter[5], sao_edge_filter[5], sao_edge_restore[2], hevc/dsp.c:217-228) as ff_hevc_dsp_init fills them for 8, 9, 10 and
// 12 bit samples, and a one-pass plane entry that applies SAO to a whole luma or chroma plane out of place from a grid of CTB records.
//
// Reference semantics reproduced bit for bit (checker: oracle/hevcsao_oracle.c), h26x/h2656_sao_template.c and the decoder's
// sao_filter_CTB (hevc/filter.c:269-478):
//   band   clip(s + offset_val[k + 1]) where k = ((s >> (depth - 5)) - band_position) & 31 is below 4, else s.
//   edge   d = sign(s - a) + sign(s - b) for the class's two neighbours a, b; clip(s + offset_val[{1, 2, 0, 3, 4}[2 + d]]).  The
//          neighbours are always deblocked samples: sao_filter_CTB reads them from the frame before a neighbouring CTB is filtered and
//          from its saved copies (sao_pixel_buffer_h / _v) after, so the result does not depend on the order of the CTBs and the
//          plane can be filtered out of place in one pass.
//   then sao_edge_restore[0 / 1] overwrites picture-border samples with clip(s + offset_val[0]) and, for [1], puts s back along slice
//   and tile edges that may not be filtered, and restore_tqb_pixels puts s back in PCM / transquant-bypass blocks.
// sao_outcome() below replays the writes of sao_edge_restore_0 / _1 for one sample, in the reference's order (last write wins), and
// is shared by the kernel and the host-side restore members.
//
// Plane kernel: a thread owns a run of 4 samples in each of 4 rows (a run never straddles a CTB: a CTB is at least 8 samples wide
// and tall), reads its CTB record and the 6 x 6 window around the runs through the read-only path in one round trip (each row's run
// as one word where aligned), decides each sample and stores each run as one 4- or 8-byte word where the row is aligned.
// Every sample is read from HBM once and written once; the neighbour reads hit L1 / L2.
#include "common.h"
#include <cstring>
#include <type_traits>

namespace {

enum { SAO_FILTER = 0, SAO_BORDER = 1, SAO_SRC = 2 };

constexpr int kRun = 4, kRows = 4, kBX = 32, kBY = 8;   // a thread: kRun samples x kRows rows

// The last write sao_edge_restore_0 (r1 false) or sao_edge_restore_1 (r1 true) makes to sample (x, y) of a W x H block, or
// SAO_FILTER when it leaves the edge filter's value.  b = borders[0..3] as bits 0..3 (left, top, right, bottom); f = the edge flags in
// B200HevcSaoCtb.flags bits (VERT_L ... DIAG_BL), read only when r1.  Any eo: the reference compares it with the four classes only.
__host__ __device__ __forceinline__ int sao_outcome(int x, int y, int W, int H, int eo, unsigned b, unsigned f, bool r1)
{
    int o = SAO_FILTER, init_x = 0, init_y = 0, w = W, h = H;
    if (eo != 1) {
        if (b & 1) { if (x == 0 && y < h) o = SAO_BORDER; init_x = 1; }
        if (b & 4) { if (x == w - 1 && y < h) o = SAO_BORDER; w--; }
    }
    if (eo != 0) {
        if (b & 2) { if (y == 0 && x >= init_x && x < w) o = SAO_BORDER; init_y = r1; }
        if (b & 8) { if (y == h - 1 && x >= init_x && x < w) o = SAO_BORDER; h--; }
    }
    if (!r1) return o;
    const int sul = !(f & B200_HEVC_SAO_DIAG_TL) && eo == 2 && !(b & 1) && !(b & 2);
    const int sur = !(f & B200_HEVC_SAO_DIAG_TR) && eo == 3 && !(b & 2) && !(b & 4);
    const int slr = !(f & B200_HEVC_SAO_DIAG_BR) && eo == 2 && !(b & 4) && !(b & 8);
    const int sll = !(f & B200_HEVC_SAO_DIAG_BL) && eo == 3 && !(b & 1) && !(b & 8);
    if ((f & B200_HEVC_SAO_VERT_L) && eo != 1 && x == 0 && y >= init_y + sul && y < h - sll) o = SAO_SRC;
    if ((f & B200_HEVC_SAO_VERT_R) && eo != 1 && x == w - 1 && y >= init_y + sur && y < h - slr) o = SAO_SRC;
    if ((f & B200_HEVC_SAO_HORIZ_T) && eo != 0 && y == 0 && x >= init_x + sul && x < w - sur) o = SAO_SRC;
    if ((f & B200_HEVC_SAO_HORIZ_B) && eo != 0 && y == h - 1 && x >= init_x + sll && x < w - slr) o = SAO_SRC;
    if ((f & B200_HEVC_SAO_DIAG_TL) && eo == 2 && x == 0 && y == 0) o = SAO_SRC;
    if ((f & B200_HEVC_SAO_DIAG_TR) && eo == 3 && x == w - 1 && y == 0) o = SAO_SRC;
    if ((f & B200_HEVC_SAO_DIAG_BR) && eo == 2 && x == w - 1 && y == h - 1) o = SAO_SRC;
    if ((f & B200_HEVC_SAO_DIAG_BL) && eo == 3 && x == 0 && y == h - 1) o = SAO_SRC;
    return o;
}

__host__ __device__ __forceinline__ int clip_pix(int v, int maxv) { return v < 0 ? 0 : v > maxv ? maxv : v; }

// off[i] without a dynamically indexed local array (which would live in local memory)
__device__ __forceinline__ int pick(const int (&off)[5], int i)
{
    return i == 0 ? off[0] : i == 1 ? off[1] : i == 2 ? off[2] : i == 3 ? off[3] : off[4];
}

struct SaoArgs {
    uint8_t *dst;
    const uint8_t *src;
    long long dstride, sstride;                              // bytes
    const B200HevcSaoCtb *ctb;
    long long cstride;                                       // records
    const uint8_t *keep;
    long long kstride;
    int width, height, depth, lcw, lch, hs, vs, log2_ctb, log2_pu, ncx, ncy;
};

template <typename P>
__device__ __forceinline__ int ld(const SaoArgs &a, int x, int y)
{
    x = x < 0 ? 0 : x >= a.width ? a.width - 1 : x;          // clamped: such reads only feed samples that take another outcome
    y = y < 0 ? 0 : y >= a.height ? a.height - 1 : y;
    return __ldg(reinterpret_cast<const P *>(a.src + (long long)y * a.sstride) + x);
}

// samples x0 - 1 .. x0 + kRun of row y into w[0 .. kRun + 1] (clamped to the plane); the kRun samples from x0 as one word where the run
// is whole, inside the row range and aligned
template <typename P>
__device__ __forceinline__ void ld_run(const SaoArgs &a, int x0, int y, int n, int (&w)[kRun + 2])
{
    const int yc = y < 0 ? 0 : y >= a.height ? a.height - 1 : y;
    const P *row = reinterpret_cast<const P *>(a.src + (long long)yc * a.sstride);
    w[0] = ld<P>(a, x0 - 1, yc);
    w[kRun + 1] = ld<P>(a, x0 + kRun, yc);
    if (n == kRun && ((uintptr_t)(row + x0) % (kRun * sizeof(P))) == 0) {
        if (sizeof(P) == 1) {
            const uint32_t v = __ldg(reinterpret_cast<const uint32_t *>(row + x0));
#pragma unroll
            for (int k = 0; k < kRun; k++) w[k + 1] = (v >> (8 * k)) & 0xFF;
        } else {
            const uint2 v = __ldg(reinterpret_cast<const uint2 *>(row + x0));
            w[1] = v.x & 0xFFFF; w[2] = v.x >> 16; w[3] = v.y & 0xFFFF; w[4] = v.y >> 16;
        }
    } else {
#pragma unroll
        for (int k = 0; k < kRun; k++) w[k + 1] = ld<P>(a, x0 + k, yc);
    }
}

// one row of a thread's run: up / mid / dn = samples x0 - 1 .. x0 + kRun of rows y - 1, y, y + 1
template <typename P>
__device__ __forceinline__ void sao_row(const SaoArgs &a, const B200HevcSaoCtb &r, const int (&off)[5], int i, int j, int x0, int n, int y,
                                        const int (&up)[kRun + 2], const int (&mid)[kRun + 2], const int (&dn)[kRun + 2])
{
    const int maxv = (1 << a.depth) - 1;
    int c[kRun], v[kRun];
#pragma unroll
    for (int k = 0; k < kRun; k++) c[k] = v[k] = mid[k + 1];
    const bool edge = r.type == B200_HEVC_SAO_EDGE && r.cls <= 3;
    if (r.type == B200_HEVC_SAO_BAND) {
#pragma unroll
        for (int k = 0; k < kRun; k++) {
            const int bk = ((c[k] >> (a.depth - 5)) - r.cls) & 31;
            v[k] = bk < 4 ? clip_pix(c[k] + pick(off, bk + 1), maxv) : c[k];
        }
    } else if (edge) {
        const int cx = i << a.lcw, cy = j << a.lch;      // CTB origin in the plane
        const int W = min(1 << a.lcw, a.width - cx), H = min(1 << a.lch, a.height - cy);
        const unsigned b = (i == 0) | (j == 0) << 1 | (i == a.ncx - 1) << 2 | (j == a.ncy - 1) << 3;
        unsigned f = r.flags & B200_HEVC_SAO_RESTORE ? r.flags : 0;
        if (b & 1) f &= ~(B200_HEVC_SAO_VERT_L | B200_HEVC_SAO_DIAG_TL | B200_HEVC_SAO_DIAG_BL);
        if (b & 2) f &= ~(B200_HEVC_SAO_HORIZ_T | B200_HEVC_SAO_DIAG_TL | B200_HEVC_SAO_DIAG_TR);
        if (b & 4) f &= ~(B200_HEVC_SAO_VERT_R | B200_HEVC_SAO_DIAG_TR | B200_HEVC_SAO_DIAG_BR);
        if (b & 8) f &= ~(B200_HEVC_SAO_HORIZ_B | B200_HEVC_SAO_DIAG_BR | B200_HEVC_SAO_DIAG_BL);
        const int eo = r.cls;
        // only samples within two of the CTB's sides can take another outcome than the filter (sao_edge_restore writes rows 0,
        // H - 2, H - 1 and columns 0, W - 2, W - 1): the run's interior samples skip the replay
        const int lx = x0 - cx, ly = y - cy;
        const bool inner = ly > 0 && ly < H - 2 && lx > 0 && lx + kRun - 1 < W - 2;
#pragma unroll
        for (int k = 0; k < kRun; k++) {
            if (k < n) {
                const int o = inner ? SAO_FILTER : sao_outcome(lx + k, ly, W, H, eo, b, f, (r.flags & B200_HEVC_SAO_RESTORE) != 0);
                // neighbours a / b of the class (hevc: horizontal, vertical, 135 and 45 degrees), window column k + 1 = the sample
                const int sa = eo == 0 ? mid[k] : eo == 1 ? up[k + 1] : eo == 2 ? up[k] : up[k + 2];
                const int sb = eo == 0 ? mid[k + 2] : eo == 1 ? dn[k + 1] : eo == 2 ? dn[k + 2] : dn[k];
                const int d = (c[k] > sa) - (c[k] < sa) + (c[k] > sb) - (c[k] < sb);
                const int idx = d == -2 ? 1 : d == -1 ? 2 : d == 0 ? 0 : d == 1 ? 3 : 4;
                if (o == SAO_BORDER) v[k] = clip_pix(c[k] + off[0], maxv);
                else if (o == SAO_FILTER) v[k] = clip_pix(c[k] + pick(off, idx), maxv);
            }
        }
    }
    if (a.keep && (edge || r.type == B200_HEVC_SAO_BAND)) {
        // restore_tqb_pixels with the luma CTB origin and the component's CTB size: PU px covers the sample when it lies below
        // (X + W) >> log2_pu, W the component width (the reference's quirk for subsampled chroma)
        const int X = i << a.log2_ctb, Y = j << a.log2_ctb;
        const int W = min(1 << a.lcw, a.width - (i << a.lcw)), H = min(1 << a.lch, a.height - (j << a.lch));
        const int ly = y - (j << a.lch), py = (Y + (ly << a.vs)) >> a.log2_pu;
        if (py < (Y + H) >> a.log2_pu) {
            const uint8_t *kr = a.keep + (long long)py * a.kstride;
#pragma unroll
            for (int k = 0; k < kRun; k++) {
                const int px = (X + ((x0 + k - (i << a.lcw)) << a.hs)) >> a.log2_pu;
                if (k < n && px < (X + W) >> a.log2_pu && __ldg(kr + px)) v[k] = c[k];
            }
        }
    }
    P *d = reinterpret_cast<P *>(a.dst + (long long)y * a.dstride) + x0;
    if (n == kRun && ((uintptr_t)d % (kRun * sizeof(P))) == 0) {
        if (sizeof(P) == 1) *reinterpret_cast<uint32_t *>(d) = (uint32_t)v[0] | (uint32_t)v[1] << 8 | (uint32_t)v[2] << 16 | (uint32_t)v[3] << 24;
        else *reinterpret_cast<uint2 *>(d) = make_uint2((uint32_t)v[0] | (uint32_t)v[1] << 16, (uint32_t)v[2] | (uint32_t)v[3] << 16);
    } else {
#pragma unroll
        for (int k = 0; k < kRun; k++)
            if (k < n) d[k] = (P)v[k];
    }
}

template <typename P>
__global__ void __launch_bounds__(kBX * kBY) hevc_sao_kernel(SaoArgs a)
{
    const int x0 = (int)(blockIdx.x * kBX + threadIdx.x) * kRun;
    if (x0 >= a.width) return;
    const int n = a.width - x0 < kRun ? a.width - x0 : kRun;
    const int i = x0 >> a.lcw;
    for (int y0 = (int)(blockIdx.y * kBY + threadIdx.y) * kRows; y0 < a.height; y0 += (int)(gridDim.y * kBY) * kRows) {
        const int j = y0 >> a.lch;                           // the kRows rows lie in one CTB row (CTBs are >= 8 rows, y0 = 0 mod 4)
        // the record and the kRows + 2 rows of the window are loaded together (none depends on another): one memory round trip
        const uint4 raw = __ldg(reinterpret_cast<const uint4 *>(a.ctb + (long long)j * a.cstride + i));
        int win[kRows + 2][kRun + 2];
#pragma unroll
        for (int q = 0; q < kRows + 2; q++) ld_run<P>(a, x0, y0 - 1 + q, n, win[q]);
        B200HevcSaoCtb r;
        memcpy(&r, &raw, sizeof(r));
        const int off[5] = { r.offset_val[0], r.offset_val[1], r.offset_val[2], r.offset_val[3], r.offset_val[4] };
#pragma unroll
        for (int q = 0; q < kRows; q++)
            if (y0 + q < a.height) sao_row<P>(a, r, off, i, j, x0, n, y0 + q, win[q], win[q + 1], win[q + 2]);
    }
}

bool depth_ok(int d) { return d == 8 || d == 9 || d == 10 || d == 12; }

cudaError_t launch(const SaoArgs &a, cudaStream_t st)
{
    const int runs = (a.width + kRun - 1) / kRun;
    const int gy = (a.height + kBY * kRows - 1) / (kBY * kRows);
    const dim3 grid((unsigned)((runs + kBX - 1) / kBX), (unsigned)(gy < 65535 ? gy : 65535)), block(kBX, kBY);
    if (a.depth == 8) hevc_sao_kernel<uint8_t><<<grid, block, 0, st>>>(a);
    else hevc_sao_kernel<uint16_t><<<grid, block, 0, st>>>(a);
    B200_LAUNCHED();
    return cudaGetLastError();
}

SaoArgs plane_args(int depth, uint8_t *dst, long long dstride, const uint8_t *src, long long sstride, int width, int height, int log2_ctb,
                   int hs, int vs, const B200HevcSaoCtb *ctb, long long cstride, const uint8_t *keep, long long kstride, int log2_pu)
{
    SaoArgs a;
    a.dst = dst; a.src = src; a.dstride = dstride; a.sstride = sstride;
    a.ctb = ctb; a.cstride = cstride; a.keep = keep; a.kstride = kstride;
    a.width = width; a.height = height; a.depth = depth;
    a.lcw = log2_ctb - hs; a.lch = log2_ctb - vs; a.hs = hs; a.vs = vs; a.log2_ctb = log2_ctb; a.log2_pu = log2_pu;
    a.ncx = (width + (1 << a.lcw) - 1) >> a.lcw;
    a.ncy = (height + (1 << a.lch) - 1) >> a.lch;
    return a;
}

// ---- band and edge members (host pointers): the block is staged into a scratch plane and run through the plane kernel with
// 64-sample CTBs, so the filter arithmetic exists once.  Band: a w x h plane, one BAND CTB.  Edge: a (w + 2) x (h + 2) plane with
// the block at (1, 1), every CTB EDGE with no flags: the block's samples are never on a CTB's picture border, so all of them take
// the edge filter, and only the ring the class reads is staged.
constexpr int kPitch = 80;                                   // scratch rows, in samples (>= 66)
constexpr size_t kRec = 256;                                 // scratch bytes for the records (4 x 16)

void member_run(int depth, bool band, uint8_t *dst, ptrdiff_t dst_stride, const uint8_t *src, ptrdiff_t src_stride, const int16_t *off,
                int cls, int w, int h)
{
    const int bps = depth > 8 ? 2 : 1;
    const size_t pitch = (size_t)kPitch * bps, plane = pitch * kPitch;
    B200HostCall call("hevc sao", nullptr, kRec + 2 * plane);
    uint8_t *scr = call.scratch;
    cudaStream_t st = call.stream;
    uint8_t *ssrc = scr + kRec, *sdst = scr + kRec + plane;
    B200HevcSaoCtb rec[4];
    memset(rec, 0, sizeof(rec));
    for (int k = 0; k < 4; k++) {
        for (int m = 0; m < 5; m++) rec[k].offset_val[m] = off[m];
        rec[k].type = band ? B200_HEVC_SAO_BAND : B200_HEVC_SAO_EDGE;
        rec[k].cls = (uint8_t)(band ? cls & 31 : cls);
    }
    call.check(cudaMemcpyAsync(scr, rec, sizeof(rec), cudaMemcpyHostToDevice, st), "h2d records");
    const int pw = band ? w : w + 2, ph = band ? h : h + 2, o = band ? 0 : 1;
    // rows / columns of the host block staged: edge classes read only their neighbours' ring
    const int r0 = band || cls == 0 ? 0 : -1, r1 = band || cls == 0 ? h : h + 1;
    const int c0 = band || cls == 1 ? 0 : -1, c1 = band || cls == 1 ? w : w + 1;
    call.check(b200_h2d_rows(ssrc + (size_t)(r0 + o) * pitch + (size_t)(c0 + o) * bps, pitch, src + (ptrdiff_t)r0 * src_stride + (ptrdiff_t)c0 * bps,
                             src_stride, (size_t)(c1 - c0) * bps, (size_t)(r1 - r0), st),
               "h2d block");
    const SaoArgs a = plane_args(depth, sdst, (long long)pitch, ssrc, (long long)pitch, pw, ph, 6, 0, 0, (const B200HevcSaoCtb *)scr, 2,
                                 nullptr, 0, 2);
    call.check(launch(a, st), "launch");
    call.check(b200_d2h_rows(dst, dst_stride, sdst + (size_t)o * pitch + (size_t)o * bps, pitch, (size_t)w * bps, (size_t)h, st), "d2h block");
    call.sync();
}

template <int D>
void m_band(uint8_t *dst, const uint8_t *src, ptrdiff_t stride_dst, ptrdiff_t stride_src, const int16_t *off, int left_class, int w, int h)
{
    if (w < 1 || h < 1 || w > 64 || h > 64) { b200_set_error("hevc sao_band_filter: %dx%d is outside 1..64", w, h); return; }
    member_run(D, true, dst, stride_dst, src, stride_src, off, left_class, w, h);
}

template <int D>
void m_edge(uint8_t *dst, const uint8_t *src, ptrdiff_t stride_dst, const int16_t *off, int eo, int w, int h)
{
    if (w < 1 || h < 1 || w > 64 || h > 64) { b200_set_error("hevc sao_edge_filter: %dx%d is outside 1..64", w, h); return; }
    if (eo < 0 || eo > 3) { b200_set_error("hevc sao_edge_filter: eo_class %d is not 0..3", eo); return; }
    member_run(D, false, dst, stride_dst, src, 2 * 64 + 64, off, eo, w, h);
}

// ---- restore members: host only (at most four lines of at most 64 samples), the kernel's per-sample classification
template <int D, bool R1>
void m_restore(uint8_t *dst, const uint8_t *src, ptrdiff_t stride_dst, ptrdiff_t stride_src, const struct SAOParams *sp, const int *borders,
               int w, int h, int c_idx, const uint8_t *vert_edge, const uint8_t *horiz_edge, const uint8_t *diag_edge)
{
    typedef typename std::conditional<D == 8, uint8_t, uint16_t>::type P;
    if (c_idx < 0 || c_idx > 2) { b200_set_error("hevc sao_edge_restore: c_idx %d is not 0..2", c_idx); return; }
    if (w < 1 || h < 1 || w > 64 || h > 64) { b200_set_error("hevc sao_edge_restore: %dx%d is outside 1..64", w, h); return; }
    const B200SAOParams *sao = reinterpret_cast<const B200SAOParams *>(sp);
    const int off0 = sao->offset_val[c_idx][0], eo = sao->eo_class[c_idx], maxv = (1 << D) - 1;
    const unsigned b = (borders[0] ? 1u : 0u) | (borders[1] ? 2u : 0u) | (borders[2] ? 4u : 0u) | (borders[3] ? 8u : 0u);
    unsigned f = 0;
    if (R1) {
        f = (vert_edge[0] ? B200_HEVC_SAO_VERT_L : 0) | (vert_edge[1] ? B200_HEVC_SAO_VERT_R : 0) | (horiz_edge[0] ? B200_HEVC_SAO_HORIZ_T : 0) |
            (horiz_edge[1] ? B200_HEVC_SAO_HORIZ_B : 0) | (diag_edge[0] ? B200_HEVC_SAO_DIAG_TL : 0) | (diag_edge[1] ? B200_HEVC_SAO_DIAG_TR : 0) |
            (diag_edge[2] ? B200_HEVC_SAO_DIAG_BR : 0) | (diag_edge[3] ? B200_HEVC_SAO_DIAG_BL : 0);
    }
    // the writes fall on rows 0, h - 2, h - 1 and columns 0, w - 2, w - 1 (h - 2 / w - 2 after a border took the last line)
    for (int y = 0; y < h; y++) {
        const bool ring_row = y == 0 || y >= h - 2;
        for (int x = 0; x < w; x++) {
            if (!ring_row && x != 0 && x < w - 2) { x = w - 3; continue; }
            const int o = sao_outcome(x, y, w, h, eo, b, f, R1);
            if (o == SAO_FILTER) continue;
            const int s = reinterpret_cast<const P *>(src + (ptrdiff_t)y * stride_src)[x];
            reinterpret_cast<P *>(dst + (ptrdiff_t)y * stride_dst)[x] = (P)(o == SAO_BORDER ? clip_pix(s + off0, maxv) : s);
        }
    }
}

// hevc/dsp.c:217-228: the five band members are one function, as are the five edge members
template <int D>
void fill(B200HEVCDSPContext *c)
{
    for (int k = 0; k < 5; k++) {
        c->sao_band_filter[k] = m_band<D>;
        c->sao_edge_filter[k] = m_edge<D>;
    }
    c->sao_edge_restore[0] = m_restore<D, false>;
    c->sao_edge_restore[1] = m_restore<D, true>;
}

} // namespace

B200_API int b200_hevc_dsp_init_sao(B200HEVCDSPContext *c, int bit_depth)
{
    if (!c) return B200_EINVAL;
    if (!depth_ok(bit_depth)) return B200_ENOSYS;
    if (!b200_default_device()) return B200_ENODEV;
    switch (bit_depth) {
    case 8:  fill<8>(c); break;
    case 9:  fill<9>(c); break;
    case 10: fill<10>(c); break;
    default: fill<12>(c); break;
    }
    return 0;
}

B200_API int b200_hevc_sao_plane_device(B200Device *dev, int bit_depth, uint8_t *dst, ptrdiff_t dst_stride, const uint8_t *src,
                                        ptrdiff_t src_stride, int width, int height, int log2_ctb_size, int hshift, int vshift,
                                        const B200HevcSaoCtb *ctb, int64_t ctb_stride, const uint8_t *keep, int64_t keep_stride,
                                        int log2_min_pu_size)
{
    if (!dst || !src || !ctb) { b200_set_error("hevc sao plane: NULL pointer"); return B200_EINVAL; }
    if (!depth_ok(bit_depth)) { b200_set_error("hevc sao plane: bit depth %d is not 8, 9, 10 or 12", bit_depth); return B200_EINVAL; }
    if (width < 1 || height < 1) { b200_set_error("hevc sao plane: %dx%d is empty", width, height); return B200_EINVAL; }
    if (log2_ctb_size < 4 || log2_ctb_size > 6) { b200_set_error("hevc sao plane: log2_ctb_size %d is not 4..6", log2_ctb_size); return B200_EINVAL; }
    if ((hshift != 0 && hshift != 1) || (vshift != 0 && vshift != 1)) {
        b200_set_error("hevc sao plane: shifts %d, %d are not 0 or 1", hshift, vshift);
        return B200_EINVAL;
    }
    const int bps = bit_depth > 8 ? 2 : 1;
    const ptrdiff_t row = (ptrdiff_t)width * bps;
    if (dst_stride < row || src_stride < row || dst_stride % bps || src_stride % bps) {
        b200_set_error("hevc sao plane: stride shorter than a row or not a whole number of samples");
        return B200_EINVAL;
    }
    if ((uintptr_t)dst % bps || (uintptr_t)src % bps || (uintptr_t)ctb % 16) {
        b200_set_error("hevc sao plane: dst / src not aligned to a sample or ctb not aligned to 16 bytes");
        return B200_EINVAL;
    }
    const int cw = (1 << log2_ctb_size) >> hshift;
    if (ctb_stride < (width + cw - 1) / cw) { b200_set_error("hevc sao plane: ctb_stride shorter than the CTB row"); return B200_EINVAL; }
    if (keep && (log2_min_pu_size < 2 || log2_min_pu_size > log2_ctb_size - 1 ||
                 keep_stride < (((int64_t)width << hshift) >> log2_min_pu_size))) {
        b200_set_error("hevc sao plane: log2_min_pu_size %d or keep_stride %lld does not fit the plane", log2_min_pu_size, (long long)keep_stride);
        return B200_EINVAL;
    }
    const uintptr_t d0 = (uintptr_t)dst, d1 = d0 + (uintptr_t)((height - 1) * (int64_t)dst_stride + row);
    const uintptr_t s0 = (uintptr_t)src, s1 = s0 + (uintptr_t)((height - 1) * (int64_t)src_stride + row);
    if (d0 < s1 && s0 < d1) { b200_set_error("hevc sao plane: dst and src overlap (the entry works out of place)"); return B200_EINVAL; }
    if (int r = b200_use_device(dev)) return r;
    const SaoArgs a = plane_args(bit_depth, dst, (long long)dst_stride, src, (long long)src_stride, width, height, log2_ctb_size, hshift,
                                 vshift, ctb, (long long)ctb_stride, keep, (long long)keep_stride, log2_min_pu_size);
    B200_CUDA_OK(launch(a, dev->stream));
    return 0;
}
