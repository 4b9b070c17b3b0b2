// pel.cu — libavcodec h264qpel (8 bit), h264chroma (8 bit) and hpeldsp motion-compensation interpolation on sm_90a (C ABI: "h264qpel / hpeldsp").
//
// Reference semantics reproduced bit-for-bit (checker: oracle/pel_oracle.c):
//   H264_LOWPASS / H264_MC / op_put, op_avg   libavcodec/h264qpel_template.c:77-465
//   PIXOP2, rnd_avg32 / no_rnd_avg32          libavcodec/hpeldsp.c:38-333, libavcodec/rnd_avg.h:31-39
//
// Batched kernel: one warp per operation.  The warp first stages the (size+5) x (size+5) source window in shared
// memory (coalesced row reads through the read-only path), for positions that need the centre sample it builds the
// unrounded horizontal 6-tap sums once (size+5 rows of int16), and then every lane produces its pixels from shared
// memory.  The 6-tap is never recomputed per output pixel and the reference block is read from HBM exactly once.
#include "common.h"
#include "pel_hbd.h"
#include <algorithm>
#include <cstring>
#include <cstdlib>

namespace {

__device__ __forceinline__ int clip8(int v) { return __vimin_s32_relu(v, 255); }

constexpr int QW = 48;                 // window pitch in bytes (12 words: the 8-byte row segments of a half-warp fall in 16 distinct
                                       // bank pairs); only bytes 0..31 are used, block pixel (0,0) sits at byte 8 of window row 2
constexpr int QX = 8;                  // so that every 8-pixel segment of a row starts 8-byte aligned in shared memory
constexpr int WARPS = 4;

// Shared memory per warp is held at 7456 bytes, which leaves room for 7 CTAs (28 warps) per SM.  The data below needs 5776 bytes, with
// which 9 CTAs fit, and the kernel then ran 8 % slower (H100 SXM at a 400 W limit: 1.37 instead of 1.49 G blocks/s in bench.py).
constexpr int QPEL_WARP_SMEM = 7456;
struct __align__(16) QpelSmem {
    uint8_t win[21 * QW];              // source rows -2 .. size+2; source column x is at byte QX + x (x = -2 .. size+2)
    short hraw[21 * 16];               // unrounded horizontal 6-tap sums for the same rows, block columns 0 .. 15
    uint8_t ring[4][16 + 21 * 48];     // raw 16-byte chunks of QD windows in flight (cp.async), window row r at ring[slot][16 + r * 48]
                                       // (16 bytes of slack: the re-alignment may read the word in front of a row)
    uint8_t pad[QPEL_WARP_SMEM - 21 * QW - 21 * 16 * 2 - 4 * (16 + 21 * 48)];   // unused: see QPEL_WARP_SMEM
};
static_assert(sizeof(QpelSmem) == QPEL_WARP_SMEM, "QpelSmem must keep the footprint that sets the kernel's occupancy");

// ---- packed arithmetic helpers --------------------------------------------------------------------------------------
// The 6-tap (1,-5,20,20,-5,1) is evaluated with the integer dot-product instructions: IDP.4A for the horizontal filter
// (u8 pixels x s8 taps, 4 taps per instruction), IDP.2A for the vertical ones (two rows interleaved by PRMT, s16 tap pair
// x u8 pixels for V; s16 sums x s8 tap pair for the centre sample).  Every component of a quarter-pel position ends up as
// two packed u8x4 words, so the (a + b + 1) >> 1 combinations are byte-SIMD averages.
__device__ __forceinline__ int dp4a_us(unsigned a, int b, int c)      // c + sum_k a.u8[k] * b.s8[k]
{ int d; asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ int dp2a_lo_su(int a, unsigned b, int c)   // c + a.s16[0]*b.u8[0] + a.s16[1]*b.u8[1]
{ int d; asm("dp2a.lo.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ int dp2a_hi_su(int a, unsigned b, int c)   // c + a.s16[0]*b.u8[2] + a.s16[1]*b.u8[3]
{ int d; asm("dp2a.hi.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ int dp2a_lo_ss(unsigned a, int b, int c)   // c + a.s16[0]*b.s8[0] + a.s16[1]*b.s8[1]
{ int d; asm("dp2a.lo.s32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }

constexpr int TAP4_A = 0x1414FB01;     // s8 (1, -5, 20, 20)
constexpr int TAP4_B = 0x000001FB;     // s8 (-5, 1, 0, 0)
__host__ __device__ constexpr int tap2_16(int j) { return j == 0 ? (int)0xFFFB0001 : j == 1 ? 0x00140014 : 0x0001FFFB; }   // s16 pairs (1,-5) (20,20) (-5,1)
__host__ __device__ constexpr int tap2_8(int j)  { return j == 0 ? 0x0000FB01 : j == 1 ? 0x00001414 : 0x000001FB; }        // s8 pairs, same taps

// 8 packed bytes of a window row: block columns x0+dx .. x0+dx+7 (dx = 0 or 1)
__device__ __forceinline__ uint2 row8p(const uint8_t *row, int x0, int dx)
{
    const unsigned *w = reinterpret_cast<const unsigned *>(row + QX + x0);
    unsigned w0 = w[0], w1 = w[1];
    if (dx) { const unsigned w2 = w[2]; w0 = __funnelshift_r(w0, w1, 8); w1 = __funnelshift_r(w1, w2, 8); }
    return make_uint2(w0, w1);
}
// unrounded horizontal 6-tap sums (+ init) for block columns x0 .. x0+7 of window row `row`
__device__ __forceinline__ void hsum8(const uint8_t *row, int x0, int init, int *o)
{
    const unsigned *w = reinterpret_cast<const unsigned *>(row + QX + x0 - 4);     // A[0] = columns x0-4 .. x0-1
    const unsigned A[5] = { w[0], w[1], w[2], w[3], w[4] };
    unsigned S[12];                                                                  // S[i] = columns x0-2+i .. x0+1+i
#pragma unroll
    for (int i = 0; i < 12; i++) {
        const int b = 2 + i;
        S[i] = (b & 3) ? __funnelshift_r(A[b >> 2], A[(b >> 2) + 1], (b & 3) * 8) : A[b >> 2];
    }
#pragma unroll
    for (int i = 0; i < 8; i++) o[i] = dp4a_us(S[i + 4], TAP4_B, dp4a_us(S[i], TAP4_A, init));
}
// one vertical tap pair over two rows of 8 packed pixels
__device__ __forceinline__ void vfold(int k2, const uint2 &r0, const uint2 &r1, int *acc)
{
    unsigned lo = __byte_perm(r0.x, r1.x, 0x5140), hi = __byte_perm(r0.x, r1.x, 0x7362);
    acc[0] = dp2a_lo_su(k2, lo, acc[0]); acc[1] = dp2a_hi_su(k2, lo, acc[1]); acc[2] = dp2a_lo_su(k2, hi, acc[2]); acc[3] = dp2a_hi_su(k2, hi, acc[3]);
    lo = __byte_perm(r0.y, r1.y, 0x5140); hi = __byte_perm(r0.y, r1.y, 0x7362);
    acc[4] = dp2a_lo_su(k2, lo, acc[4]); acc[5] = dp2a_hi_su(k2, lo, acc[5]); acc[6] = dp2a_lo_su(k2, hi, acc[6]); acc[7] = dp2a_hi_su(k2, hi, acc[7]);
}
// clip8(v[k] >> SH) for 8 values -> two packed words
template <int SH>
__device__ __forceinline__ uint2 clip_pack8(const int *v)
{
    unsigned c[8];
#pragma unroll
    for (int k = 0; k < 8; k++) c[k] = (unsigned)clip8(v[k] >> SH);
    uint2 o;
    o.x = __byte_perm(__byte_perm(c[0], c[1], 0x1140), __byte_perm(c[2], c[3], 0x1140), 0x5410);
    o.y = __byte_perm(__byte_perm(c[4], c[5], 0x1140), __byte_perm(c[6], c[7], 0x1140), 0x5410);
    return o;
}

// The kernel is latency-bound if every operation waits for its descriptor, then its window, then (avg) its
// destination.  Each warp therefore walks QK consecutive operations and software-pipelines them: while operation t is
// computed, the windows of the next QD - 1 operations are already in flight (below), every descriptor of the warp has been
// fetched, and the destination row of t (avg) was requested before the shared-memory staging started.
constexpr int QK = 32;               // operations per warp (one descriptor per lane): the start-up round trips (descriptors, first windows) are paid once per 32 blocks

struct QMeta { int o; long long soff, doff; };
__device__ __forceinline__ QMeta load_meta(const uint8_t *op, const int64_t *src_off, const int64_t *dst_off, long long i, long long n)
{
    QMeta m; m.o = -1; m.soff = 0; m.doff = 0;
    if (i < n) { m.o = __ldg(op + i); m.soff = __ldg(src_off + i); m.doff = __ldg(dst_off + i); }
    return m;
}
// Windows in flight.  With one window per warp in flight the kernel is bound by memory latency, so the raw 16-byte chunks go
// global -> shared with cp.async into a ring of QD windows per warp (no registers held while they fly), QD - 1 operations ahead of
// the one being computed; the lane that copied a row re-aligns it out of the ring when its turn comes.
constexpr int QD = 4;
__device__ __forceinline__ void q_cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void q_cp_wait() { asm volatile("cp.async.wait_group %0;" :: "n"(N) : "memory"); }
// request window row `lane` (source row lane - 2, columns -2 .. size + 2) of one operation: the one to three aligned 16-byte words
// that contain at least one needed byte; always closes a group, so that the group count is the operation count.
//   first = address of the row's column -2; rl = shared address of this lane's row in the ring slot
__device__ __forceinline__ void issue_window(unsigned rl, uintptr_t first, int wdim, int lane, bool valid)
{
    if (valid && lane < wdim) {
        const uint8_t *q = reinterpret_cast<const uint8_t *>(first & ~(uintptr_t)15);
        const int nv = (int)(((first & 15) + wdim + 15) >> 4);
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(rl), "l"(q) : "memory");
        if (nv > 1) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(rl + 16), "l"(q + 16) : "memory");
        if (nv > 2) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(rl + 32), "l"(q + 32) : "memory");
    }
    q_cp_commit();
}
// the lane's own row out of the ring, block column 0 moved to byte QX of the window row;
// sh = low four bits of the row's first address, raw = the lane's row in the ring slot
__device__ __forceinline__ void stage_from_ring(QpelSmem &s, const unsigned *raw, unsigned sh, int wdim, int lane)
{
    if (lane >= wdim) return;
    const int ws = (int)((sh + 2) >> 2) - 1;                     // window word j = raw bytes sh + 4j - 6 .. sh + 4j - 3; ws in -1 .. 3
    const unsigned fs = ((sh + 2) & 3) * 8;
    unsigned x[7];
#pragma unroll
    for (int i = 0; i < 7; i++) x[i] = raw[ws + i];              // word -1 (slack / previous row) and words never copied only feed columns nobody reads
    uint4 *row = reinterpret_cast<uint4 *>(&s.win[lane * QW]);
    row[0] = make_uint4(0u, __funnelshift_r(x[0], x[1], fs), __funnelshift_r(x[1], x[2], fs), __funnelshift_r(x[2], x[3], fs));
    row[1] = make_uint4(__funnelshift_r(x[3], x[4], fs), __funnelshift_r(x[4], x[5], fs), __funnelshift_r(x[5], x[6], fs), 0u);
}

// Lane l works on one 8-pixel (4 for size 4) row segment: row l>>1, half l&1 for 16x16.
__global__ void __launch_bounds__(32 * WARPS)
qpel_kernel(long long n, const uint8_t *op, uint8_t *dst, const int64_t *dst_off, const uint8_t *src,
            const int64_t *src_off, long long stride)
{
    __shared__ QpelSmem sm[WARPS];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long first_op = ((long long)blockIdx.x * WARPS + warp) * QK;
    if (first_op >= n) return;
    QpelSmem &s = sm[warp];
    // lane k (< QK) owns the descriptor of the warp's operation k; everybody gets it by shuffle when the operation is issued / computed
    const QMeta mine_m = load_meta(op, src_off, dst_off, first_op + lane, lane < QK ? n : 0);
    const long long rowoff = (long long)(lane - 2) * stride - 2;                          // this lane's window row, column -2, from the block's (0, 0)
    const uintptr_t srcb = reinterpret_cast<uintptr_t>(src) + (uintptr_t)rowoff;
    const unsigned ring0 = (unsigned)__cvta_generic_to_shared(&s.ring[0][16 + lane * 48]);
    constexpr unsigned RING_SLOT = (unsigned)sizeof(s.ring[0]);
#pragma unroll
    for (int k = 0; k < QD - 1; k++) {                                                   // QD - 1 windows ahead
        const int ok = __shfl_sync(0xffffffffu, mine_m.o, k);
        const long long sk = __shfl_sync(0xffffffffu, mine_m.soff, k);
        issue_window(ring0 + k * RING_SLOT, srcb + (uintptr_t)sk, (16 >> ((ok >> 1) & 3)) + 5, lane, ok >= 0);
    }
    for (int t = 0; t < QK; t++) {
        const int o = __shfl_sync(0xffffffffu, mine_m.o, t);
        if (o < 0) break;                                                                // past the end (warp-uniform)
        const long long soff0 = __shfl_sync(0xffffffffu, mine_m.soff, t);
        const long long doff0 = __shfl_sync(0xffffffffu, mine_m.doff, t);
        {
            const int ka = t + QD - 1, kk = ka < QK ? ka : QK - 1;
            const int oa = __shfl_sync(0xffffffffu, mine_m.o, kk);
            const long long sa = __shfl_sync(0xffffffffu, mine_m.soff, kk);
            issue_window(ring0 + (ka & (QD - 1)) * RING_SLOT, srcb + (uintptr_t)sa, (16 >> ((oa >> 1) & 3)) + 5, lane, ka < QK && oa >= 0);
        }

        const int avg = o & 1, sidx = (o >> 1) & 3, size = 16 >> sidx, qx = (o >> 3) & 3, qy = (o >> 5) & 3;
        uint8_t *dp = dst + doff0;
        const int wdim = size + 5;
        int npx = 8, segs = 2, y = lane >> 1, x0 = (lane & 1) << 3;
        bool mine = true;
        if (size != 16) {                                                                // 8 x 8 and 4 x 4: one segment per row
            npx = size < 8 ? size : 8; segs = 1;
            mine = lane < size; y = lane; x0 = 0;
        }
        // size index 3 names no table of the reference: the op writes nothing.  It still waits for its window (issued above like any
        // other), so that the ring slot is free before the look-ahead of a later op is copied into it.
        if (sidx == 3) mine = false;
        uint8_t *d = dp + (long long)y * stride + x0;
        const bool vec = npx == 8 && ((reinterpret_cast<uintptr_t>(d)) & 7) == 0;
        uint2 pv = make_uint2(0, 0);
        if (mine && avg && vec) pv = *reinterpret_cast<const uint2 *>(d);                // destination row requested early

        q_cp_wait<QD - 1>();                                                             // this operation's chunks have landed (own copies)
        stage_from_ring(s, reinterpret_cast<const unsigned *>(&s.ring[t & (QD - 1)][16 + lane * 48]),
                        ((unsigned)srcb + (unsigned)soff0) & 15u, wdim, lane);
        __syncwarp();
        const bool need_j = (qx == 2 && qy != 0) || (qy == 2 && qx != 0);                // positions built from the centre sample
        if (need_j) {
            for (int k = lane; k < wdim * segs; k += 32) {
                const int r = k / segs, xx = (k - r * segs) * 8;
                int h[8];
                hsum8(&s.win[r * QW], xx, 0, h);
                uint4 pk;
                pk.x = __byte_perm(h[0], h[1], 0x5410); pk.y = __byte_perm(h[2], h[3], 0x5410);
                pk.z = __byte_perm(h[4], h[5], 0x5410); pk.w = __byte_perm(h[6], h[7], 0x5410);
                *reinterpret_cast<uint4 *>(&s.hraw[r * 16 + xx]) = pk;
            }
            __syncwarp();
        }
        if (mine) {
            // the one or two samples each quarter position averages (h264qpel_template.c:313-456): F full-pel, H horizontal
            // half, V vertical half, J centre.  acc collects them; two samples -> (a + b + 1) >> 1.
            const bool useF = (qy == 0 && qx != 2) || (qx == 0 && (qy & 1));
            const bool useH = qx != 0 && qy != 2;
            const bool useV = qy != 0 && qx != 2;
            uint2 res = make_uint2(0, 0);
            bool have = false;
            auto add = [&](const uint2 &c) {
                if (have) { res.x = __vavgu4(res.x, c.x); res.y = __vavgu4(res.y, c.y); }
                else { res = c; have = true; }
            };
            if (useF) add(row8p(&s.win[(y + 2 + (qy == 3)) * QW], x0, qx == 3));
            if (useH) {
                int h[8];
                hsum8(&s.win[(y + 2 + (qy == 3)) * QW], x0, 16, h);
                add(clip_pack8<5>(h));
            }
            if (useV) {
                const int dx = qx == 3;
                int a8[8];
#pragma unroll
                for (int k = 0; k < 8; k++) a8[k] = 16;
#pragma unroll
                for (int j = 0; j < 3; j++)
                    vfold(tap2_16(j), row8p(&s.win[(y + 2 * j) * QW], x0, dx), row8p(&s.win[(y + 2 * j + 1) * QW], x0, dx), a8);
                add(clip_pack8<5>(a8));
            }
            if (need_j) {
                int j6[8];
#pragma unroll
                for (int k = 0; k < 8; k++) j6[k] = 512;
#pragma unroll
                for (int j = 0; j < 3; j++) {
                    const uint4 pa = *reinterpret_cast<const uint4 *>(&s.hraw[(y + 2 * j) * 16 + x0]);
                    const uint4 pb = *reinterpret_cast<const uint4 *>(&s.hraw[(y + 2 * j + 1) * 16 + x0]);
                    const unsigned wa[4] = { pa.x, pa.y, pa.z, pa.w }, wb[4] = { pb.x, pb.y, pb.z, pb.w };
#pragma unroll
                    for (int k = 0; k < 4; k++) {
                        j6[2 * k]     = dp2a_lo_ss(__byte_perm(wa[k], wb[k], 0x5410), tap2_8(j), j6[2 * k]);
                        j6[2 * k + 1] = dp2a_lo_ss(__byte_perm(wa[k], wb[k], 0x7632), tap2_8(j), j6[2 * k + 1]);
                    }
                }
                add(clip_pack8<10>(j6));
            }
            if (vec) {
                if (avg) { res.x = __vavgu4(res.x, pv.x); res.y = __vavgu4(res.y, pv.y); }
                *reinterpret_cast<uint2 *>(d) = res;
            } else {
                for (int k = 0; k < npx; k++) {
                    const int v = (int)__byte_perm(k < 4 ? res.x : res.y, 0, 0x4440 | (k & 3));
                    d[k] = (uint8_t)(avg ? (d[k] + v + 1) >> 1 : v);
                }
            }
        }
        __syncwarp();                                                                    // shared window is reused by the next operation
    }
    q_cp_wait<0>();                                                                      // nothing of this warp's is in flight when it leaves
}

// hpel: one warp per operation, direct global reads (at most 4 taps per pixel, rows are contiguous)
__global__ void __launch_bounds__(32 * WARPS)
hpel_kernel(long long n, const uint8_t *op, const uint8_t *hh, uint8_t *dst, const int64_t *dst_off, const uint8_t *src,
            const int64_t *src_off, long long stride)
{
    const long long i = (long long)blockIdx.x * WARPS + (threadIdx.x >> 5);
    if (i >= n) return;
    const int lane = threadIdx.x & 31;
    const int o = op[i], h = hh[i];
    const int tab = o & 3, sidx = (o >> 2) & 3, xy = (o >> 4) & 3, w = 16 >> sidx;
    if ((tab == 2 && sidx >= 2) || (tab == 3 && sidx >= 1)) return;   // entries the reference leaves NULL (hpeldsp.c:337-352): write nothing
    const int no_rnd = tab >= 2;
    const int avg = (tab & 1) && !(sidx == 3 && xy == 3);        // avg_pixels2_xy2 stores without averaging (hpeldsp.c:134-166)
    const uint8_t *sp = src + src_off[i];
    uint8_t *dp = dst + dst_off[i];
    for (int k = lane; k < w * h; k += 32) {
        const int y = k / w, x = k - y * w;
        const uint8_t *p = sp + (long long)y * stride + x;
        int v;
        switch (xy) {
        case 0:  v = __ldg(p); break;
        case 1:  v = (__ldg(p) + __ldg(p + 1) + 1 - no_rnd) >> 1; break;
        case 2:  v = (__ldg(p) + __ldg(p + stride) + 1 - no_rnd) >> 1; break;
        default: v = (__ldg(p) + __ldg(p + 1) + __ldg(p + stride) + __ldg(p + stride + 1) + 2 - no_rnd) >> 2; break;
        }
        uint8_t *d = dp + (long long)y * stride + x;
        *d = (uint8_t)(avg ? (*d + v + 1) >> 1 : v);
    }
}

// h264chroma: bilinear eighth-pel (h264chroma_template.c:27-176).  8 lanes per operation, lane r owns row r (and r+8 of a
// 16-row block).  A row is fetched as the one or two aligned 8-byte words that hold bytes the reference itself reads (x == 0
// never touches the column right of the block, y == 0 never the row below it) and normalised to block column 0 with funnel
// shifts; the row below comes from the next lane by shuffle.  (A*t0 + B*t1 + C*b0 + D*b1 + 32) >> 6 is evaluated with
// coefficients scaled by 4, so that the result is byte 1 of the sum: two IDP.2A per pixel and no shifts.
constexpr int CH_LANES = 8;
struct ChRow { unsigned r0, r1, r2; };
__device__ __forceinline__ ChRow chroma_row(const uint8_t *p, int nbytes, bool on)
{
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    const unsigned sh = (unsigned)(a & 7);
    const uint2 *q = reinterpret_cast<const uint2 *>(a & ~(uintptr_t)7);
    uint2 v0 = make_uint2(0, 0), v1 = make_uint2(0, 0);
    if (on) {
        v0 = __ldg(q);
        if (sh + nbytes > 8) v1 = __ldg(q + 1);
    }
    const bool up = sh & 4;
    const unsigned t0 = up ? v0.y : v0.x, t1 = up ? v1.x : v0.y, t2 = up ? v1.y : v1.x, t3 = up ? 0u : v1.y;
    const unsigned fs = (sh & 3) * 8;
    ChRow o;
    o.r0 = __funnelshift_r(t0, t1, fs); o.r1 = __funnelshift_r(t1, t2, fs); o.r2 = __funnelshift_r(t2, t3, fs);
    return o;
}
// CK operations per 8-lane group, with every global load of the CK windows (descriptors first, then window rows and, for avg,
// destination rows) issued before the first result is computed: with one window per 8 lanes the kernel waits on three dependent
// round trips to memory per operation.  CK = 2 at 8 CTAs per SM is the largest batch that fits in 64 registers without spilling.
constexpr int CK = 2, CK_MINB = 8;
__global__ void __launch_bounds__(32 * WARPS, CK_MINB)
chroma_kernel(long long n, const uint8_t *op, const uint8_t *hh, const uint8_t *xy, uint8_t *dst, const int64_t *dst_off,
              const uint8_t *src, const int64_t *src_off, long long stride)
{
    const int lane = threadIdx.x & 31, grp = lane >> 3, sub = lane & (CH_LANES - 1);
    // persistent warps: batch b = 4 * CK consecutive operations; the descriptors of the next batch are requested before this one is
    // worked on, so only the window loads are left on the critical path of a batch
    const long long nwarps = (long long)gridDim.x * WARPS, nbatch = (n + 4 * CK - 1) / (4 * CK);
    long long b = (long long)blockIdx.x * WARPS + (threadIdx.x >> 5);
    if (b >= nbatch) return;
    int nmeta[CK];
    long long nso[CK], ndof[CK];
    auto fetch = [&](long long bb) {
#pragma unroll
        for (int j = 0; j < CK; j++) {
            const long long gi = bb * (4 * CK) + 4 * j + grp;
            const bool ok = bb < nbatch && gi < n;
            const long long i = ok ? gi : n - 1;
            nmeta[j] = (int)__ldg(op + i) | (int)__ldg(hh + i) << 8 | (int)__ldg(xy + i) << 16 | (ok ? 1 << 24 : 0);
            nso[j] = __ldg(src_off + i); ndof[j] = __ldg(dst_off + i);
        }
    };
    fetch(b);
    for (; b < nbatch; b += nwarps) {
    int o[CK], h[CK], pq[CK];
    long long so[CK], dof[CK];
    bool valid[CK];
#pragma unroll
    for (int j = 0; j < CK; j++) {
        o[j] = nmeta[j] & 255; h[j] = (nmeta[j] >> 8) & 255; pq[j] = (nmeta[j] >> 16) & 255;
        valid[j] = ((nmeta[j] >> 24) & 1) && ((o[j] >> 1) & 3) != 3;                  // width index 3 is the reference's NULL entry: write nothing
        so[j] = nso[j]; dof[j] = ndof[j];
    }
    fetch(b + nwarps);
    int hm = 0;
#pragma unroll
    for (int j = 0; j < CK; j++) hm = max(hm, valid[j] ? h[j] : 0);
    const int hmax = __reduce_max_sync(0xffffffffu, hm);
    for (int y0 = 0; y0 < hmax; y0 += CH_LANES) {
        const int y = y0 + sub;
        ChRow t[CK], bl[CK];
        uint2 pv[CK];
        bool mine[CK], vec[CK];
        // every load of the CK windows
#pragma unroll
        for (int j = 0; j < CK; j++) {
            const int fx = pq[j] & 7, fy = (pq[j] >> 3) & 7, w = 8 >> ((o[j] >> 1) & 3);
            const int nbytes = w + (fx != 0);
            mine[j] = valid[j] && y < h[j];
            const uint8_t *rowp = src + so[j] + (long long)y * stride;
            t[j] = chroma_row(rowp, nbytes, mine[j]);
            const bool last = sub == CH_LANES - 1 || y == h[j] - 1;      // the row below is not held by the next lane
            bl[j] = chroma_row(rowp + stride, nbytes, mine[j] && last && fy != 0);
            const uint8_t *d = dst + dof[j] + (long long)y * stride;
            vec[j] = w == 8 && (reinterpret_cast<uintptr_t>(d) & 7) == 0;
            pv[j] = make_uint2(0, 0);
            if (mine[j] && vec[j] && (o[j] & 1)) pv[j] = *reinterpret_cast<const uint2 *>(d);
        }
#pragma unroll
        for (int j = 0; j < CK; j++) {
            const int fx = pq[j] & 7, fy = (pq[j] >> 3) & 7, avg = o[j] & 1, w = 8 >> ((o[j] >> 1) & 3);
            const int kab = 4 * ((8 - fx) * (8 - fy)) | (4 * (fx * (8 - fy))) << 16;      // s16 pairs (4A, 4B) and (4C, 4D)
            const int kcd = 4 * ((8 - fx) * fy) | (4 * (fx * fy)) << 16;
            ChRow b;
            b.r0 = __shfl_down_sync(0xffffffffu, t[j].r0, 1, CH_LANES); b.r1 = __shfl_down_sync(0xffffffffu, t[j].r1, 1, CH_LANES);
            b.r2 = __shfl_down_sync(0xffffffffu, t[j].r2, 1, CH_LANES);
            if (sub == CH_LANES - 1 || y == h[j] - 1) b = bl[j];
            if (!mine[j]) continue;
            const ChRow &tt = t[j];
            const unsigned ta = __funnelshift_r(tt.r0, tt.r1, 8), tb = __funnelshift_r(tt.r1, tt.r2, 8);
            const unsigned ba = __funnelshift_r(b.r0, b.r1, 8), bb = __funnelshift_r(b.r1, b.r2, 8);
            int v[8];
            v[0] = dp2a_lo_su(kcd, b.r0, dp2a_lo_su(kab, tt.r0, 128)); v[1] = dp2a_lo_su(kcd, ba, dp2a_lo_su(kab, ta, 128));
            v[2] = dp2a_hi_su(kcd, b.r0, dp2a_hi_su(kab, tt.r0, 128)); v[3] = dp2a_hi_su(kcd, ba, dp2a_hi_su(kab, ta, 128));
            v[4] = dp2a_lo_su(kcd, b.r1, dp2a_lo_su(kab, tt.r1, 128)); v[5] = dp2a_lo_su(kcd, bb, dp2a_lo_su(kab, tb, 128));
            v[6] = dp2a_hi_su(kcd, b.r1, dp2a_hi_su(kab, tt.r1, 128)); v[7] = dp2a_hi_su(kcd, bb, dp2a_hi_su(kab, tb, 128));
            unsigned w0 = __byte_perm(__byte_perm(v[0], v[1], 0x5151), __byte_perm(v[2], v[3], 0x5151), 0x5410);
            unsigned w1 = __byte_perm(__byte_perm(v[4], v[5], 0x5151), __byte_perm(v[6], v[7], 0x5151), 0x5410);
            uint8_t *d = dst + dof[j] + (long long)y * stride;
            if (vec[j]) {
                if (avg) { w0 = __vavgu4(pv[j].x, w0); w1 = __vavgu4(pv[j].y, w1); }
                *reinterpret_cast<uint2 *>(d) = make_uint2(w0, w1);
            } else if (w >= 4 && (reinterpret_cast<uintptr_t>(d) & 3) == 0) {
                unsigned *d4 = reinterpret_cast<unsigned *>(d);
                d4[0] = avg ? __vavgu4(d4[0], w0) : w0;
                if (w == 8) d4[1] = avg ? __vavgu4(d4[1], w1) : w1;
            } else {
                for (int k = 0; k < w; k++) {
                    const int px = (int)__byte_perm(k < 4 ? w0 : w1, 0, 0x4440 | (k & 3));
                    d[k] = (uint8_t)(avg ? (d[k] + px + 1) >> 1 : px);
                }
            }
        }
    }
    }
}

// The dot-product form is the one qpel path: the filter arithmetic is a minority of the instructions per block, the rest is per-block
// scaffolding (descriptor shuffles, window re-alignment, destination addressing, stores), so moving the filters to the tensor cores
// does not pay.  Windows arrive by cp.async rather than TMA: small 2-D boxes (one 48 x 21-byte box per operation) are bound by the
// copy engine's per-row requests, not by the LSU they bypass.
int qpel_launch(cudaStream_t st, int64_t n, const uint8_t *op, uint8_t *dst, const int64_t *dst_off, const uint8_t *src,
                const int64_t *src_off, ptrdiff_t stride)
{
    const long long blocks = (n + WARPS * QK - 1) / (WARPS * QK);
    if (blocks > 0x7fffffffLL) return B200_EINVAL;
    qpel_kernel<<<(unsigned)blocks, 32 * WARPS, 0, st>>>(n, op, dst, dst_off, src, src_off, stride);
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

// persistent warps: one per batch of 4 * CK operations, at most CK_MINB CTAs per SM (sms = the device's SM count)
int chroma_launch(cudaStream_t st, int sms, int64_t n, const uint8_t *op, const uint8_t *h, const uint8_t *xy, uint8_t *dst,
                  const int64_t *dst_off, const uint8_t *src, const int64_t *src_off, ptrdiff_t stride)
{
    const long long nbatch = (n + 4 * CK - 1) / (4 * CK), want = (nbatch + WARPS - 1) / WARPS, cap = (long long)sms * CK_MINB;
    chroma_kernel<<<(unsigned)(want < cap ? want : cap), 32 * WARPS, 0, st>>>(n, op, h, xy, dst, dst_off, src, src_off, stride);
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

enum HostKind { HOST_QPEL, HOST_HPEL, HOST_CHROMA };
constexpr const char *kFeature = "motion compensation";

// one block through the device for the drop-in tables.  Only the source rectangle the reference function itself reads is
// copied from the caller's buffer (bx/ax columns left/right, by/ay rows above/below the block).
void host_op(HostKind kind, int o, int h, int w, uint8_t *dst, const uint8_t *src, ptrdiff_t stride,
             int bx, int ax, int by, int ay, int fxy = 0)
{
    const int before = kind == HOST_QPEL ? 2 : 0, after = kind == HOST_QPEL ? 3 : 1;   // the window the kernels may touch
    const int sh = h + before + after;
    const size_t pitch = 32;
    B200HostCall call(kFeature, nullptr, pitch * (sh + h) + 256);
    uint8_t *scr = call.scratch;
    uint8_t *dsrc = scr, *ddst = scr + pitch * sh;
    uint8_t *meta = scr + pitch * (sh + h);           // op, h, offsets
    cudaStream_t st = call.stream;
    call.check(b200_h2d_rows(dsrc + (before - by) * pitch + (before - bx), pitch, src - by * stride - bx, stride, w + bx + ax, h + by + ay, st),
               "h2d src");
    call.check(b200_h2d_rows(ddst, pitch, dst, stride, w, h, st), "h2d dst");
    struct { int64_t doff, soff; uint8_t op, h, xy; } m = { 0, (int64_t)(before * pitch + before), (uint8_t)o, (uint8_t)h, (uint8_t)fxy };
    call.check(cudaMemcpyAsync(meta, &m, sizeof(m), cudaMemcpyHostToDevice, st), "h2d meta");
    const int64_t *doff = (const int64_t *)meta, *soff = doff + 1;
    const uint8_t *dop = meta + 16, *dh = meta + 17, *dxy = meta + 18;
    // dst and src live in one buffer with the same pitch, like the reference's single stride
    int err = 0;
    if (kind == HOST_QPEL)        err = qpel_launch(st, 1, dop, ddst, doff, dsrc, soff, pitch);
    else if (kind == HOST_CHROMA) err = chroma_launch(st, call.dev->sm_count, 1, dop, dh, dxy, ddst, doff, dsrc, soff, pitch);
    else { hpel_kernel<<<1, 32 * WARPS, 0, st>>>(1, dop, dh, ddst, doff, dsrc, soff, (long long)pitch); B200_LAUNCHED(); }
    call.launched(err);
    call.check(b200_d2h_rows(dst, stride, ddst, pitch, w, h, st), "d2h");
    call.sync();
}

template <int AVG, int SIDX, int POS>
void qpel_tab(uint8_t *dst, const uint8_t *src, ptrdiff_t stride)
{
    constexpr int X = POS & 3, Y = POS >> 2;           // h264qpel_template.c: mc{x}{y} filters horizontally iff x, vertically iff y
    host_op(HOST_QPEL, AVG | (SIDX << 1) | (POS << 3), 16 >> SIDX, 16 >> SIDX, dst, src, stride, X ? 2 : 0, X ? 3 : 0, Y ? 2 : 0, Y ? 3 : 0);
}
template <int TAB, int SIDX, int XY>
void hpel_tab(uint8_t *block, const uint8_t *pixels, ptrdiff_t line_size, int h)
{
    host_op(HOST_HPEL, TAB | (SIDX << 2) | (XY << 4), h, 16 >> SIDX, block, pixels, line_size, 0, XY & 1, 0, XY >> 1);
}
template <int AVG, int IDX>
void chroma_tab(uint8_t *dst, const uint8_t *src, ptrdiff_t stride, int h, int x, int y)
{
    if ((unsigned)x > 7 || (unsigned)y > 7) B200HostCall::fail(kFeature, "h264chroma: x, y must be in 0..7");     // av_assert2 in the reference
    host_op(HOST_CHROMA, AVG | (IDX << 1), h, 8 >> IDX, dst, src, stride, 0, x ? 1 : 0, 0, y ? 1 : 0, x | (y << 3));
}

template <int AVG, int SIDX>
void fill_qpel(b200_qpel_mc_func *t)
{
    t[0] = qpel_tab<AVG, SIDX, 0>;   t[1] = qpel_tab<AVG, SIDX, 1>;   t[2] = qpel_tab<AVG, SIDX, 2>;   t[3] = qpel_tab<AVG, SIDX, 3>;
    t[4] = qpel_tab<AVG, SIDX, 4>;   t[5] = qpel_tab<AVG, SIDX, 5>;   t[6] = qpel_tab<AVG, SIDX, 6>;   t[7] = qpel_tab<AVG, SIDX, 7>;
    t[8] = qpel_tab<AVG, SIDX, 8>;   t[9] = qpel_tab<AVG, SIDX, 9>;   t[10] = qpel_tab<AVG, SIDX, 10>; t[11] = qpel_tab<AVG, SIDX, 11>;
    t[12] = qpel_tab<AVG, SIDX, 12>; t[13] = qpel_tab<AVG, SIDX, 13>; t[14] = qpel_tab<AVG, SIDX, 14>; t[15] = qpel_tab<AVG, SIDX, 15>;
}
template <int TAB, int SIDX>
void fill_hpel(b200_op_pixels_func *t)
{
    t[0] = hpel_tab<TAB, SIDX, 0>; t[1] = hpel_tab<TAB, SIDX, 1>; t[2] = hpel_tab<TAB, SIDX, 2>; t[3] = hpel_tab<TAB, SIDX, 3>;
}

} // namespace

B200_API int b200_h264qpel_init(B200H264QpelContext *c, int bit_depth)
{
    if (!c) return B200_EINVAL;
    if (bit_depth != 8 && bit_depth != 9 && bit_depth != 10 && bit_depth != 12 && bit_depth != 14) return B200_ENOSYS;   // h264qpel.c:87-103
    if (!b200_default_device()) return B200_ENODEV;
    if (bit_depth != 8) { pel_hbd_fill(c, bit_depth); return 0; }  // uint16 samples (pel_hbd.cu)
    fill_qpel<0, 0>(c->put_h264_qpel_pixels_tab[0]); fill_qpel<0, 1>(c->put_h264_qpel_pixels_tab[1]); fill_qpel<0, 2>(c->put_h264_qpel_pixels_tab[2]);
    fill_qpel<1, 0>(c->avg_h264_qpel_pixels_tab[0]); fill_qpel<1, 1>(c->avg_h264_qpel_pixels_tab[1]); fill_qpel<1, 2>(c->avg_h264_qpel_pixels_tab[2]);
    return 0;
}

B200_API int b200_hpeldsp_init(B200HpelDSPContext *c, int flags)
{
    (void)flags;
    if (!c) return B200_EINVAL;
    if (!b200_default_device()) return B200_ENODEV;
    memset(c, 0, sizeof(*c));
    fill_hpel<0, 0>(c->put_pixels_tab[0]); fill_hpel<0, 1>(c->put_pixels_tab[1]); fill_hpel<0, 2>(c->put_pixels_tab[2]); fill_hpel<0, 3>(c->put_pixels_tab[3]);
    fill_hpel<1, 0>(c->avg_pixels_tab[0]); fill_hpel<1, 1>(c->avg_pixels_tab[1]); fill_hpel<1, 2>(c->avg_pixels_tab[2]); fill_hpel<1, 3>(c->avg_pixels_tab[3]);
    fill_hpel<2, 0>(c->put_no_rnd_pixels_tab[0]); fill_hpel<2, 1>(c->put_no_rnd_pixels_tab[1]);
    fill_hpel<3, 0>(c->avg_no_rnd_pixels_tab);
    return 0;
}

B200_API int b200_h264chroma_init(B200H264ChromaContext *c, int bit_depth)
{
    if (!c) return B200_EINVAL;
    if (!b200_default_device()) return B200_ENODEV;
    if (bit_depth > 8 && bit_depth <= 16) { pel_hbd_fill_chroma(c); return 0; }       // h264chroma.c:45-50: the 16 bit template (pel_hbd.cu)
    memset(c, 0, sizeof(*c));                                      // entry [3] stays NULL like the reference's
    c->put_h264_chroma_pixels_tab[0] = chroma_tab<0, 0>; c->put_h264_chroma_pixels_tab[1] = chroma_tab<0, 1>; c->put_h264_chroma_pixels_tab[2] = chroma_tab<0, 2>;
    c->avg_h264_chroma_pixels_tab[0] = chroma_tab<1, 0>; c->avg_h264_chroma_pixels_tab[1] = chroma_tab<1, 1>; c->avg_h264_chroma_pixels_tab[2] = chroma_tab<1, 2>;
    return 0;
}

B200_API int b200_h264chroma_batch_device(B200Device *dev, int64_t n, const uint8_t *op, const uint8_t *h, const uint8_t *xy,
                                          uint8_t *dst, const int64_t *dst_off, const uint8_t *src, const int64_t *src_off,
                                          ptrdiff_t stride)
{
    if (!dev || n < 0 || !op || !h || !xy || !dst || !dst_off || !src || !src_off) return B200_EINVAL;
    if (n == 0) return 0;
    if (int r = b200_use_device(dev)) return r;
    return chroma_launch(dev->stream, dev->sm_count, n, op, h, xy, dst, dst_off, src, src_off, stride);
}

B200_API int b200_h264qpel_batch_device(B200Device *dev, int64_t n, const uint8_t *op, uint8_t *dst, const int64_t *dst_off,
                                        const uint8_t *src, const int64_t *src_off, ptrdiff_t stride)
{
    if (!dev || n < 0 || !op || !dst || !dst_off || !src || !src_off) return B200_EINVAL;
    if (n == 0) return 0;
    if (int r = b200_use_device(dev)) return r;
    return qpel_launch(dev->stream, n, op, dst, dst_off, src, src_off, stride);
}

// HOST buffers: a stream of frames, each with its own reference picture, destination picture and list of motion-compensation
// operations (what a decoder holding its pictures in host memory hands over once per frame).  Frame f occupies
// [f * frame_bytes, (f + 1) * frame_bytes) of `src` and of `dst`; its operations are op_begin[f] .. op_begin[f + 1] - 1, with offsets
// counted from the start of `dst` / `src` like the device entry point, and must stay inside frame f.  Frames are cut into chunks that
// rotate over the device's three pipeline streams: H2D of the chunk's reference and destination pictures and operation lists, the
// kernel, D2H of the destination pictures.
B200_API int b200_h264qpel_frames_host(B200Device *dev, int nframes, int64_t frame_bytes, const int64_t *op_begin, const uint8_t *op,
                                       uint8_t *dst, const int64_t *dst_off, const uint8_t *src, const int64_t *src_off, ptrdiff_t stride)
{
    if (!dev || nframes < 0 || frame_bytes <= 0 || !op_begin || !op || !dst || !dst_off || !src || !src_off) return B200_EINVAL;
    if (nframes == 0) return 0;
    B200_CUDA_OK(cudaSetDevice(dev->ordinal));
    int64_t ops_total = op_begin[nframes] - op_begin[0];
    for (int f = 0; f < nframes; f++) if (op_begin[f + 1] < op_begin[f]) return B200_EINVAL;
    const int64_t ops_per_frame = (ops_total + nframes - 1) / nframes;
    const size_t perFrame = 2 * (size_t)frame_bytes + (size_t)ops_per_frame * 17 + 64;
    int chunk = (int)(((size_t)64 << 20) / perFrame);
    if (chunk < 1) chunk = 1;
    if (chunk > nframes) chunk = nframes;
    int64_t max_ops = 0;                                            // operations of the busiest chunk
    for (int f0 = 0; f0 < nframes; f0 += chunk) max_ops = std::max(max_ops, op_begin[std::min(nframes, f0 + chunk)] - op_begin[f0]);
    const size_t n8 = (((size_t)max_ops * 8) + 255) & ~(size_t)255;
    const size_t pics = ((2 * (size_t)frame_bytes * chunk) + 255) & ~(size_t)255;
    const size_t slotBytes = pics + 2 * n8 + (((size_t)max_ops + 255) & ~(size_t)255);
    const int K = B200Device::kPipe;
    B200_LOCK_DEVICE(dev);
    uint8_t *scr = (uint8_t *)b200_scratch(dev, slotBytes * K);
    if (!scr) return B200_ENOMEM;
    B200_CUDA_OK(cudaStreamSynchronize(dev->stream));
    int slot = 0;
    for (int f0 = 0; f0 < nframes; f0 += chunk, slot = (slot + 1) % K) {
        const int nf = nframes - f0 < chunk ? nframes - f0 : chunk;
        cudaStream_t st = dev->pipe[slot];
        uint8_t *base = scr + (size_t)slot * slotBytes;
        uint8_t *dsrc = base, *ddst = base + (size_t)frame_bytes * chunk;
        int64_t *ddo = (int64_t *)(base + pics), *dso = (int64_t *)(base + pics + n8);
        uint8_t *dop = base + pics + 2 * n8;
        const int64_t o0 = op_begin[f0], n = op_begin[f0 + nf] - o0;
        B200_CUDA_OK(cudaMemcpyAsync(dsrc, src + (size_t)f0 * frame_bytes, (size_t)nf * frame_bytes, cudaMemcpyHostToDevice, st));
        B200_CUDA_OK(cudaMemcpyAsync(ddst, dst + (size_t)f0 * frame_bytes, (size_t)nf * frame_bytes, cudaMemcpyHostToDevice, st));
        if (n > 0) {
            B200_CUDA_OK(cudaMemcpyAsync(ddo, dst_off + o0, (size_t)n * 8, cudaMemcpyHostToDevice, st));
            B200_CUDA_OK(cudaMemcpyAsync(dso, src_off + o0, (size_t)n * 8, cudaMemcpyHostToDevice, st));
            B200_CUDA_OK(cudaMemcpyAsync(dop, op + o0, (size_t)n, cudaMemcpyHostToDevice, st));
            // the lists keep their offsets from the start of the whole buffers: hand the kernel bases moved back by the chunk's origin
            const int r = qpel_launch(st, n, dop, ddst - (size_t)f0 * frame_bytes, ddo, dsrc - (size_t)f0 * frame_bytes, dso, stride);
            if (r) return r;
        }
        B200_CUDA_OK(cudaMemcpyAsync(dst + (size_t)f0 * frame_bytes, ddst, (size_t)nf * frame_bytes, cudaMemcpyDeviceToHost, st));
    }
    for (int i = 0; i < K; i++) B200_CUDA_OK(cudaStreamSynchronize(dev->pipe[i]));
    return 0;
}

B200_API int b200_hpel_batch_device(B200Device *dev, int64_t n, const uint8_t *op, const uint8_t *h, uint8_t *dst,
                                    const int64_t *dst_off, const uint8_t *src, const int64_t *src_off, ptrdiff_t stride)
{
    if (!dev || n < 0 || !op || !h || !dst || !dst_off || !src || !src_off) return B200_EINVAL;
    if (n == 0) return 0;
    if (int r = b200_use_device(dev)) return r;
    const long long blocks = (n + WARPS - 1) / WARPS;
    if (blocks > 0x7fffffffLL) return B200_EINVAL;
    hpel_kernel<<<(unsigned)blocks, 32 * WARPS, 0, dev->stream>>>(n, op, h, dst, dst_off, src, src_off, stride);
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}
