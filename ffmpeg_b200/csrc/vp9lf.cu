// vp9lf.cu — the VP9 loop filter on sm_90a: the loop_filter_8[3][2], loop_filter_16[2] and loop_filter_mix2[2][2][2] members of
// VP9DSPContext (libavcodec/vp9dsp.h:40-122) as vp9dsp_loopfilter_init fills them for 8, 10 and 12 bit samples (vp9dsp_template.c:
// 1780-1967), and a frame entry that runs ff_vp9_loopfilter_sb (vp9lpf.c:179-203) over every superblock of a frame in one launch.
//
// Reference semantics reproduced bit for bit (checker: oracle/vp9lf_oracle.c):
//   filter     one line of p7..p0 q0..q7 across an edge, E, I, H shifted by depth - 8, F = 1 << (depth - 8): lf_line below restates
//              loop_filter (vp9dsp_template.c:1780-1889)
//   dispatch   filter_plane_cols / filter_plane_rows (vp9lpf.c:27-177) restated per line and per column as col_edge / row_edge below,
//              with the driver's quirks: in the column pass the second 8 lines' mask leaves out its 16-wide bit unless the first 8
//              lines are 16-wide too, and a 16-wide pair then filters both halves with the first half's level; with ss_h the level
//              column is k & ~1; the inner 4-wide edges ([3]) only where the direction is not subsampled; in the row pass the pair is
//              bits k and k + 1 + ss_h, and an inner row edge is reached only while the row's [0..2] masks have a bit at or above it
//   order      per superblock in raster order and per plane, all column edges, then all row edges
//
// The order is part of the result: an edge writes up to 7 samples on each side and the next edge along the line reads them, and
// superblock (r, c)'s first row edge reads rows that (r - 1, c + 1)'s 16-wide column edge has changed.  Frame-wide "all columns, then
// all rows" (hevcdbk.cu's model) or a slope-1 wavefront give different pictures.  So superblock (r, c) of a plane runs after (r, c - 1)
// and (r - 1, c + 1): a wavefront of slope 2 with a critical path of sb_cols + 2 (sb_rows - 1) superblocks.
//
// Frame kernel: one CTA per (plane, superblock row), 3 sb_rows of them.  A CTA takes its row from an atomicAdd ticket (planes
// interleaved), so every row it waits on belongs to a CTA that is already running: no deadlock whatever else shares the GPU.  It walks
// its row left to right with the superblock in shared memory (an 8-sample halo on the left, the previous superblock slid over, and on
// the top, read from global memory after the wait; the superblock itself is read before it, since no other CTA writes it first).
// Before superblock c it waits until its plane's row r - 1 has published min(c + 2, sb_cols) finished superblocks (acquire loads), and
// it publishes its own count after its stores (fence, release store).
// Every wait is bounded by about one second of %globaltimer: a scheduling mistake ends with wrong samples, never with a hung GPU, and
// each wait that runs out is counted in a per-device word that b200_vp9_loopfilter_timeouts() reads back.
// The column pass gives each thread one line and the row pass one column; each walks its edges in the driver's order.
#include "common.h"
#include "wait_timeouts.h"
#include <cstring>

namespace {

constexpr int kThreads = 64;                                 // one line / column of a luma superblock per thread
constexpr int kTile = 72;                                    // 8 halo + 64 samples
constexpr int kPitch = 74;                                   // tile row in uint16: an odd number of words (a warp down a column is conflict-free)
constexpr unsigned long long kWaitNs = 1000000000ull;        // bound of one wait
constexpr int kBatch = 12;                                   // global loads of a thread in flight

struct LfArgs {
    uint8_t *plane[3];
    long long ls[3];                                         // bytes
    const B200Vp9Filter *lflvl;
    long long lstride;                                       // records
    int *sync;                                               // [0] ticket, [1 + p sb_rows + r] superblocks finished in row r of plane p
    int *timeouts;                                           // waits that ran out, counted for the device (b200_vp9_loopfilter_timeouts)
    int cols, rows, sb_cols, sb_rows, ss_h, ss_v, depth;
    uint8_t lim[64], mblim[64];
};

// ---- inter-CTA progress
__device__ __forceinline__ int ld_acquire(const int *p)
{
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release(int *p, int v)
{
    asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long globaltimer()
{
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// ---- end of inter-CTA progress

// one line across an edge, v[0..15] = p7..p0 q0..q7 (v[8] = q0); width 4 / 8 read v[4..11], width 16 all of it
__device__ __forceinline__ void lf_line(int (&v)[16], int wd, int E, int I, int H, int depth)
{
    const int sh = depth - 8, F = 1 << sh, maxv = (1 << depth) - 1, lim = (1 << (depth - 1)) - 1;
    E <<= sh;
    I <<= sh;
    H <<= sh;
    const int p3 = v[4], p2 = v[5], p1 = v[6], p0 = v[7], q0 = v[8], q1 = v[9], q2 = v[10], q3 = v[11];
    const bool fm = abs(p3 - p2) <= I && abs(p2 - p1) <= I && abs(p1 - p0) <= I && abs(q1 - q0) <= I && abs(q2 - q1) <= I &&
                    abs(q3 - q2) <= I && abs(p0 - q0) * 2 + (abs(p1 - q1) >> 1) <= E;
    if (!fm) return;
    const bool flat8in = wd >= 8 && abs(p3 - p0) <= F && abs(p2 - p0) <= F && abs(p1 - p0) <= F && abs(q1 - q0) <= F &&
                         abs(q2 - q0) <= F && abs(q3 - q0) <= F;
    bool flat8out = false;
    if (wd >= 16) {
        flat8out = true;
#pragma unroll
        for (int k = 0; k < 4; k++) flat8out = flat8out && abs(v[k] - p0) <= F && abs(v[12 + k] - q0) <= F;
    }
    if (flat8out && flat8in) {
        // output k (1..14) = (sum of the 15 taps centred on k, the ends repeated, + tap k once more + 8) >> 4
        int o[16];
#pragma unroll
        for (int k = 1; k < 15; k++) {
            int s = v[k] + 8;
#pragma unroll
            for (int d = -7; d <= 7; d++) s += v[min(max(k + d, 0), 15)];
            o[k] = s >> 4;
        }
#pragma unroll
        for (int k = 1; k < 15; k++) v[k] = o[k];
    } else if (flat8in) {
        v[5] = (p3 + p3 + p3 + 2 * p2 + p1 + p0 + q0 + 4) >> 3;
        v[6] = (p3 + p3 + p2 + 2 * p1 + p0 + q0 + q1 + 4) >> 3;
        v[7] = (p3 + p2 + p1 + 2 * p0 + q0 + q1 + q2 + 4) >> 3;
        v[8] = (p2 + p1 + p0 + 2 * q0 + q1 + q2 + q3 + 4) >> 3;
        v[9] = (p1 + p0 + q0 + 2 * q1 + q2 + q3 + q3 + 4) >> 3;
        v[10] = (p0 + q0 + q1 + 2 * q2 + q3 + q3 + q3 + 4) >> 3;
    } else {
        const bool hev = abs(p1 - p0) > H || abs(q1 - q0) > H;
        int f = hev ? min(max(p1 - q1, -lim - 1), lim) : 0;
        f = min(max(3 * (q0 - p0) + f, -lim - 1), lim);
        const int f1 = min(f + 4, lim) >> 3, f2 = min(f + 3, lim) >> 3;
        v[7] = min(max(p0 + f2, 0), maxv);
        v[8] = min(max(q0 - f1, 0), maxv);
        if (!hev) {
            const int g = (f1 + 1) >> 1;
            v[6] = min(max(p1 + g, 0), maxv);
            v[9] = min(max(q1 - g, 0), maxv);
        }
    }
}

// samples at s[k * step], k = -r..r-1 (r = 8 for width 16, else 4), filtered as one line; only what the width may write is stored
template <typename S>
__device__ __forceinline__ void lf_apply(S *s, int step, int wd, int E, int I, int H, int depth)
{
    int v[16];
    const int r = wd == 16 ? 8 : 4, w = wd == 16 ? 7 : wd == 8 ? 3 : 2;
#pragma unroll
    for (int k = 0; k < 16; k++) v[k] = (k >= 8 - r && k < 8 + r) ? (int)s[(k - 8) * step] : 0;
    lf_line(v, wd, E, I, H, depth);
#pragma unroll
    for (int k = 0; k < 16; k++)
        if (k >= 8 - w && k < 8 + w) s[(k - 8) * step] = (S)v[k];
}

struct Edge { int wd, L; };                                  // wd 0: no edge

// filter_plane_cols for one line in 8-line group g of the superblock at mask bit k: the main edge (inner = false, at k * (8 >> ss_h))
// or the inner 4-wide edge (inner = true, 4 samples further; only without ss_h).  m = the plane's column masks, lvl = level[].
__device__ __forceinline__ Edge col_edge(const uint8_t (*m)[4], const uint8_t *lvl, int g, int k, int ss_h, int ss_v, bool inner)
{
    const int m1 = (g & ~1) << ss_v, m2 = m1 + (1 << ss_v), x = 1 << k, lc = ss_h ? (k & ~1) : k;
    const uint8_t *h1 = m[m1], *h2 = m[m2];
    const int L1 = lvl[m1 * 8 + lc] & 63, L2 = lvl[m2 * 8 + lc] & 63;
    if (inner) {
        if (g & 1) return { (h2[3] & x) ? 4 : 0, L2 };
        return { (h1[3] & x) ? 4 : 0, L1 };
    }
    if (!(g & 1)) return { (h1[0] & x) ? 16 : (h1[1] & x) ? 8 : (h1[2] & x) ? 4 : 0, L1 };
    if (h1[0] & x) return { (h2[0] & x) ? 16 : 0, L1 };      // loop_filter_16 with the first half's level, or the first half alone
    if ((h2[1] | h2[2]) & x) return { (h2[1] & x) ? 8 : 4, L2 };
    return { 0, 0 };
}

// filter_plane_rows for one column in 8-column half `half` of the 16-column pair whose first bit is a, mask row y: main edge at row
// y * (8 >> ss_v) or the inner edge 4 rows below (only without ss_v)
__device__ __forceinline__ Edge row_edge(const uint8_t (*m)[4], const uint8_t *lvl, int y, int a, int half, int ss_h, int ss_v, bool inner)
{
    const uint8_t *v = m[y];
    const int vm = v[0] | v[1] | v[2];
    if (!(vm >> a)) return { 0, 0 };                         // the driver's x loop has ended before this pair
    const int b = a + 1 + ss_h, xa = 1 << a, xb = 1 << b, lr = ss_v ? (y & ~1) : y;
    const int La = lvl[lr * 8 + a] & 63, Lb = lvl[lr * 8 + b] & 63;
    if (inner) {
        if (half) return { (v[3] & xb) ? 4 : 0, Lb };
        return { (v[3] & xa) ? 4 : 0, La };
    }
    if (!half) return { (v[0] & xa) ? 16 : (v[1] & xa) ? 8 : (v[2] & xa) ? 4 : 0, La };
    if (v[0] & xa) return { (v[0] & xb) ? 16 : 0, La };
    if (vm & xb) return { (v[1] & xb) ? 8 : 4, Lb };
    return { 0, 0 };
}

template <typename P>
__global__ void __launch_bounds__(kThreads) vp9_lf_kernel(const __grid_constant__ LfArgs a)
{
    __shared__ uint16_t t[kTile][kPitch];                    // [8 + row][8 + column] of the superblock
    __shared__ uint8_t rec[192];                             // the record, bits outside the picture cleared
    __shared__ int s_ticket;
    const int tid = threadIdx.x;
    if (tid == 0) s_ticket = atomicAdd(a.sync, 1);
    __syncthreads();
    const int p = s_ticket % 3, r = s_ticket / 3;
    if (r >= a.sb_rows) return;
    for (int i = tid; i < kTile * kPitch; i += kThreads) (&t[0][0])[i] = 0;   // tile cells outside the area hold defined values
    const int ssh = p ? a.ss_h : 0, ssv = p ? a.ss_v : 0, mi = p ? (a.ss_h | a.ss_v) : 0;
    const int W = p ? ((a.cols * 8 >> ssh) + 7) & ~7 : a.cols * 8, H = p ? ((a.rows * 8 >> ssv) + 7) & ~7 : a.rows * 8;
    const int sbw = 64 >> ssh, sbh = 64 >> ssv, y0 = r * sbh;
    uint8_t *base = a.plane[p];
    const long long ls = a.ls[p];
    const int *prev = a.sync + 1 + (long long)p * a.sb_rows + r - 1;
    int *mine = a.sync + 1 + (long long)p * a.sb_rows + r;
    auto at = [&](int y, int x) { return reinterpret_cast<P *>(base + (long long)y * ls) + x; };
    const uint8_t *lvl = rec;
    const uint8_t (*cm)[4] = reinterpret_cast<const uint8_t (*)[4]>(rec + 64 + mi * 64);
    const uint8_t (*rm)[4] = reinterpret_cast<const uint8_t (*)[4]>(rec + 64 + mi * 64 + 32);
    // rows [ty0, ty0 + nrows) of the tile's superblock columns from global memory, clipped to the plane's area, with kBatch loads of a
    // thread in flight at once (one round trip per batch rather than per sample)
    auto load = [&](int x0, int ty0, int nrows) {
        const int n = nrows * sbw;
        for (int i0 = tid; i0 < n; i0 += kThreads * kBatch) {
            P v[kBatch];
#pragma unroll
            for (int u = 0; u < kBatch; u++) {
                const int i = i0 + u * kThreads, y = y0 - 8 + ty0 + i / sbw, x = x0 + i % sbw;
                if (i < n && y >= 0 && y < H && x < W) v[u] = __ldcg(at(y, x));
            }
#pragma unroll
            for (int u = 0; u < kBatch; u++) {
                const int i = i0 + u * kThreads, y = y0 - 8 + ty0 + i / sbw, x = x0 + i % sbw;
                if (i < n && y >= 0 && y < H && x < W) t[ty0 + i / sbw][8 + i % sbw] = v[u];
            }
        }
    };
    for (int c = 0; c < a.sb_cols; c++) {
        const int x0 = c * sbw;
        // the previous superblock's last 8 columns become the left halo
        if (c > 0)
            for (int i = tid; i < 8 * sbh; i += kThreads) t[8 + i / 8][i % 8] = t[8 + i / 8][sbw + i % 8];
        if (tid < 192 / 4) {
            // byte loads: the records carry no alignment beyond a byte (B200Vp9Filter is uint8_t throughout)
            const uint8_t *f = reinterpret_cast<const uint8_t *>(a.lflvl + (long long)r * a.lstride + c) + 4 * tid;
            unsigned w = f[0] | (unsigned)f[1] << 8 | (unsigned)f[2] << 16 | (unsigned)f[3] << 24;
            if (tid >= 16) {                                  // mask word j = [ch][dir][row]: rows and columns outside the picture cleared,
                const int j = tid - 16, row = j & 7;          // and the 16-wide chroma edges that would cross into the next superblock
                const unsigned keep = r * 8 + row < a.rows ? (a.cols - c * 8 >= 8 ? 0xFFu : (1u << max(a.cols - c * 8, 0)) - 1) : 0u;
                w &= keep * 0x01010101u;
                if (j == 16 + row && a.ss_h) w &= ~0x80u;
                if (j == 24 + 7 && a.ss_v) w &= ~0xFFu;
            }
            reinterpret_cast<unsigned *>(rec)[tid] = w;
        }
        __syncthreads();
        // the superblock itself: no other CTA writes it before this one is done, so it is read before the wait
        load(x0, 8, sbh);
        if (r > 0 && tid == 0) {
            const int need = min(c + 2, a.sb_cols);
            if (ld_acquire(prev) < need) {
                const unsigned long long t0 = globaltimer();
                unsigned ns = 32;
                while (ld_acquire(prev) < need && globaltimer() - t0 < kWaitNs) {
                    __nanosleep(ns);
                    ns = min(ns * 2, 1024u);
                }
                if (ld_acquire(prev) < need) atomicAdd(a.timeouts, 1);
            }
        }
        __syncthreads();
        // the top halo: rows the superblocks (r - 1, c) and (r - 1, c + 1) have finished
        if (r > 0) load(x0, 0, 8);
        __syncthreads();
        // column edges: a thread per line
        if (tid < sbh && y0 + tid < H) {
            const int g = tid >> 3;
            uint16_t *row = t[8 + tid];
            for (int k = 0; k < 8; k++) {
                const Edge e = col_edge(cm, lvl, g, k, ssh, ssv, false);
                if (e.wd && (c || k)) lf_apply(row + 8 + k * (8 >> ssh), 1, e.wd, a.mblim[e.L], a.lim[e.L], e.L >> 4, a.depth);
                if (!ssh) {
                    const Edge e4 = col_edge(cm, lvl, g, k, ssh, ssv, true);
                    if (e4.wd) lf_apply(row + 8 + k * 8 + 4, 1, 4, a.mblim[e4.L], a.lim[e4.L], e4.L >> 4, a.depth);
                }
            }
        }
        __syncthreads();
        // row edges: a thread per column
        if (tid < sbw && x0 + tid < W) {
            const int half = (tid >> 3) & 1, pa = (tid >> 4) * (2 << ssh);
            uint16_t *col = &t[8][8 + tid];
            for (int y = 0; y < 8; y++) {
                const Edge e = row_edge(rm, lvl, y, pa, half, ssh, ssv, false);
                if (e.wd && (r || y)) lf_apply(col + y * (8 >> ssv) * kPitch, kPitch, e.wd, a.mblim[e.L], a.lim[e.L], e.L >> 4, a.depth);
                if (!ssv) {
                    const Edge e4 = row_edge(rm, lvl, y, pa, half, ssh, ssv, true);
                    if (e4.wd) lf_apply(col + (y * 8 + 4) * kPitch, kPitch, 4, a.mblim[e4.L], a.lim[e4.L], e4.L >> 4, a.depth);
                }
            }
        }
        __syncthreads();
        // store the superblock with the halo samples it may have changed (left: column edge at x0; top: row edge at y0)
        for (int i = tid; i < (sbh + 8) * (sbw + 8); i += kThreads) {
            const int ty = i / (sbw + 8), tx = i % (sbw + 8), y = y0 - 8 + ty, x = x0 + tx - 8;
            if ((ty < 8 && tx < 8) || y < 0 || y >= H || x < 0 || x >= W) continue;
            *at(y, x) = (P)t[ty][tx];
        }
        __threadfence();
        __syncthreads();
        if (tid == 0) st_release(mine, c + 1);
    }
}

bool depth_ok(int d) { return d == 8 || d == 10 || d == 12; }

// ---- drop-in members (host pointers): the footprint of each 8-line half (dst[-4..3] across for widths 4 / 8, dst[-8..7] for 16) goes
// to a 16 x 16 device scratch laid out like the host's (dir 0: line l is scratch row l, q0 at column 8; dir 1: across-offset k is
// scratch row 8 + k, line l column l); one CTA filters the lines with lf_apply, and the samples the width may write come back.
struct MemberArgs {
    uint8_t *scr;
    int dir, depth;
    int wd[2], E[2], I[2], H[2];                             // lines 0..7, lines 8..15 (wd 0: none)
};

template <typename P>
__global__ void __launch_bounds__(16) vp9_lf_member_kernel(const __grid_constant__ MemberArgs m)
{
    const int l = threadIdx.x, h = l >> 3;
    if (!m.wd[h]) return;
    P *s = reinterpret_cast<P *>(m.scr) + (m.dir ? 8 * 16 + l : l * 16 + 8);
    lf_apply(s, m.dir ? 16 : 1, m.wd[h], m.E[h], m.I[h], m.H[h], m.depth);
}

void member_host(int depth, int dir, int wd1, int wd2, uint8_t *dst, ptrdiff_t stride, int E1, int I1, int H1, int E2, int I2, int H2)
{
    const int bps = depth > 8 ? 2 : 1;
    const size_t dpitch = 16 * (size_t)bps;
    B200HostCall call("vp9 loop filter", nullptr, 16 * dpitch);
    uint8_t *scr = call.scratch;
    cudaStream_t st = call.stream;
    const int wd[2] = { wd1, wd2 };
    // the block of lines 8h..8h+7 and across-offsets -n..n-1: host address, scratch address, bytes per copied row, rows
    auto copy = [&](int h, int n, bool up) {
        uint8_t *hs = dst + (dir ? -(ptrdiff_t)n * stride + (ptrdiff_t)(8 * h) * bps : (ptrdiff_t)(8 * h) * stride - (ptrdiff_t)n * bps);
        uint8_t *ds = scr + (dir ? (size_t)(8 - n) * dpitch + (size_t)(8 * h) * bps : (size_t)(8 * h) * dpitch + (size_t)(8 - n) * bps);
        const size_t w = (dir ? 8 : 2 * (size_t)n) * bps, rows = dir ? 2 * (size_t)n : 8;
        return up ? b200_h2d_rows(ds, dpitch, hs, stride, w, rows, st) : b200_d2h_rows(hs, stride, ds, dpitch, w, rows, st);
    };
    for (int h = 0; h < 2; h++)
        if (wd[h]) call.check(copy(h, wd[h] == 16 ? 8 : 4, true), "h2d edge");
    const MemberArgs m = { scr, dir, depth, { wd1, wd2 }, { E1, E2 }, { I1, I2 }, { H1, H2 } };
    if (depth == 8) vp9_lf_member_kernel<uint8_t><<<1, 16, 0, st>>>(m);
    else vp9_lf_member_kernel<uint16_t><<<1, 16, 0, st>>>(m);
    B200_LAUNCHED();
    call.launched();
    for (int h = 0; h < 2; h++)
        if (wd[h]) call.check(copy(h, wd[h] == 16 ? 7 : wd[h] == 8 ? 3 : 2, false), "d2h edge");
    call.sync();
}

template <int D, int WD, int DIR>
void m_lf8(uint8_t *dst, ptrdiff_t stride, int E, int I, int H) { member_host(D, DIR, 4 << WD, 0, dst, stride, E, I, H, 0, 0, 0); }
template <int D, int DIR>
void m_lf16(uint8_t *dst, ptrdiff_t stride, int E, int I, int H) { member_host(D, DIR, 16, 16, dst, stride, E, I, H, E, I, H); }
template <int D, int A, int B, int DIR>
void m_mix2(uint8_t *dst, ptrdiff_t stride, int E, int I, int H)
{
    member_host(D, DIR, 4 << A, 4 << B, dst, stride, E & 0xff, I & 0xff, H & 0xff, E >> 8, I >> 8, H >> 8);
}

// vp9dsp_template.c:1947-1967
template <int D>
void fill(B200VP9DSPContext *c)
{
    c->loop_filter_8[0][0] = m_lf8<D, 0, 0>;
    c->loop_filter_8[0][1] = m_lf8<D, 0, 1>;
    c->loop_filter_8[1][0] = m_lf8<D, 1, 0>;
    c->loop_filter_8[1][1] = m_lf8<D, 1, 1>;
    c->loop_filter_8[2][0] = m_lf8<D, 2, 0>;
    c->loop_filter_8[2][1] = m_lf8<D, 2, 1>;
    c->loop_filter_16[0] = m_lf16<D, 0>;
    c->loop_filter_16[1] = m_lf16<D, 1>;
    c->loop_filter_mix2[0][0][0] = m_mix2<D, 0, 0, 0>;
    c->loop_filter_mix2[0][0][1] = m_mix2<D, 0, 0, 1>;
    c->loop_filter_mix2[0][1][0] = m_mix2<D, 0, 1, 0>;
    c->loop_filter_mix2[0][1][1] = m_mix2<D, 0, 1, 1>;
    c->loop_filter_mix2[1][0][0] = m_mix2<D, 1, 0, 0>;
    c->loop_filter_mix2[1][0][1] = m_mix2<D, 1, 0, 1>;
    c->loop_filter_mix2[1][1][0] = m_mix2<D, 1, 1, 0>;
    c->loop_filter_mix2[1][1][1] = m_mix2<D, 1, 1, 1>;
}

} // namespace

B200_API int b200_vp9_dsp_init_loopfilter(B200VP9DSPContext *c, int bit_depth)
{
    if (!c) return B200_EINVAL;
    if (!depth_ok(bit_depth)) return B200_ENOSYS;
    if (!b200_default_device()) return B200_ENODEV;
    switch (bit_depth) {
    case 8:  fill<8>(c); break;
    case 10: fill<10>(c); break;
    default: fill<12>(c); break;
    }
    return 0;
}

B200_API int b200_vp9_loopfilter_frame_device(B200Device *dev, int bit_depth, int ss_h, int ss_v, int width, int height,
                                              uint8_t *const planes[3], ptrdiff_t ls_y, ptrdiff_t ls_uv, const B200Vp9Filter *lflvl,
                                              int64_t lflvl_stride, const uint8_t lim_lut[64], const uint8_t mblim_lut[64])
{
    if (!planes || !planes[0] || !planes[1] || !planes[2] || !lflvl || !lim_lut || !mblim_lut) {
        b200_set_error("vp9 loop filter frame: NULL pointer");
        return B200_EINVAL;
    }
    if (!depth_ok(bit_depth)) { b200_set_error("vp9 loop filter frame: bit depth %d is not 8, 10 or 12", bit_depth); return B200_EINVAL; }
    if ((ss_h != 0 && ss_h != 1) || (ss_v != 0 && ss_v != 1)) { b200_set_error("vp9 loop filter frame: ss_h / ss_v not 0 or 1"); return B200_EINVAL; }
    if (width < 1 || height < 1) { b200_set_error("vp9 loop filter frame: %dx%d picture", width, height); return B200_EINVAL; }
    const int bps = bit_depth > 8 ? 2 : 1;
    const int cols = (width + 7) >> 3, rows = (height + 7) >> 3, sb_cols = (cols + 7) >> 3, sb_rows = (rows + 7) >> 3;
    const long long wy = (long long)cols * 8 * bps, wuv = (long long)((((cols * 8) >> ss_h) + 7) & ~7) * bps;
    if (ls_y < wy || ls_uv < wuv || ls_y % bps || ls_uv % bps) {
        b200_set_error("vp9 loop filter frame: stride shorter than a plane row or not a whole number of samples");
        return B200_EINVAL;
    }
    for (int p = 0; p < 3; p++)
        if ((uintptr_t)planes[p] % bps) { b200_set_error("vp9 loop filter frame: plane %d not aligned to a sample", p); return B200_EINVAL; }
    if (lflvl_stride < sb_cols) { b200_set_error("vp9 loop filter frame: lflvl_stride %lld below %d", (long long)lflvl_stride, sb_cols); return B200_EINVAL; }
    if (int r = b200_use_device(dev)) return r;
    B200_LOCK_DEVICE(dev);
    int *timeouts = b200_wait_timeouts_word(dev->ordinal, B200_WAIT_VP9_LOOPFILTER, true);
    if (!timeouts) { b200_set_error("vp9 loop filter frame: no timeout counter for device %d", dev->ordinal); return B200_ENOMEM; }
    const size_t sync_bytes = sizeof(int) * (1 + 3 * (size_t)sb_rows);
    int *sync = (int *)b200_scratch(dev, sync_bytes);
    if (!sync) return B200_ENOMEM;
    LfArgs a;
    memset(&a, 0, sizeof(a));
    for (int p = 0; p < 3; p++) a.plane[p] = planes[p];
    a.ls[0] = ls_y;
    a.ls[1] = a.ls[2] = ls_uv;
    a.lflvl = lflvl;
    a.lstride = lflvl_stride;
    a.sync = sync;
    a.timeouts = timeouts;
    a.cols = cols;
    a.rows = rows;
    a.sb_cols = sb_cols;
    a.sb_rows = sb_rows;
    a.ss_h = ss_h;
    a.ss_v = ss_v;
    a.depth = bit_depth;
    memcpy(a.lim, lim_lut, 64);
    memcpy(a.mblim, mblim_lut, 64);
    B200_CUDA_OK(cudaMemsetAsync(sync, 0, sync_bytes, dev->stream));
    const unsigned grid = 3u * (unsigned)sb_rows;
    if (bit_depth == 8) vp9_lf_kernel<uint8_t><<<grid, kThreads, 0, dev->stream>>>(a);
    else vp9_lf_kernel<uint16_t><<<grid, kThreads, 0, dev->stream>>>(a);
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

B200_API int b200_vp9_loopfilter_timeouts(B200Device *dev, int64_t *count)
{
    if (!count) { b200_set_error("vp9 loop filter timeouts: NULL pointer"); return B200_EINVAL; }
    if (int r = b200_use_device(dev)) return r;
    B200_CUDA_OK(cudaStreamSynchronize(dev->stream));
    int v = 0;
    int *w = b200_wait_timeouts_word(dev->ordinal, B200_WAIT_VP9_LOOPFILTER, false);
    if (w) B200_CUDA_OK(cudaMemcpy(&v, w, sizeof(int), cudaMemcpyDeviceToHost));
    *count = v;
    return 0;
}
