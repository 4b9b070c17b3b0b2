// vp8lf.cu — the VP8 / VP7 loop filter on sm_90a: the ten loop-filter members of VP8DSPContext (libavcodec/vp8dsp.h:46-64) as
// ff_vp8dsp_init / ff_vp7dsp_init fill them (vp8dsp.c:263-457, :702-713, :733-744), and a frame entry that runs the decoder's
// filter_mb_row (vp8.c:2523-2574) over every macroblock row of a frame in one launch.
//
// Reference semantics reproduced bit for bit (checker: oracle/vp8lf_oracle.c):
//   line       p3..q3 across an edge; VP8 simple limit 2 |p0 - q0| + (|p1 - q1| >> 1) <= E, VP7 |p0 - q0| <= E; the normal limit adds
//              every neighbour difference p3..q3 <= I; high edge variance |p1 - p0| > H or |q1 - q0| > H
//   common     a = clip_int8(3 (q0 - p0) [+ clip_int8(p1 - q1) for the 4-tap form]); f1 = min(a + 4, 127) >> 3, f2 = VP8 min(a + 3, 127)
//              >> 3, VP7 f1 - ((a & 7) == 4); p0 + f2, q0 - f1, and without the 4-tap form p1 / q1 by (f1 + 1) >> 1, clipped to 0..255
//   mbedge     w = clip_int8(clip_int8(p1 - q1) + 3 (q0 - p0)); p2..q2 moved by (9 w + 63) >> 7, (18 w + 63) >> 7, (27 w + 63) >> 7
//   members    MB edge: hev ? common 4-tap : mbedge; inner: hev ? common 4-tap : common 2-tap; simple: common 4-tap
// lf_line below is that arithmetic, once, used by the members' kernel and by the frame kernel.
//
// Frame: per macroblock in raster order filter_mb (vp8.c:2181-2266) or filter_mb_simple (:2268-2299): the left MB edge (mb_x > 0), the
// inner column edges (VP8 here, VP7 last), the top MB edge (mb_y > 0), the inner row edges.  Whole-frame filtering is exact: the
// decoder filters row r - 1 before it decodes row r, but row r's intra prediction reads the unfiltered top border that
// backup_mb_border / xchg_mb_border saved (vp8.c:1701-1706, :2556-2561), and its left neighbours unfiltered too, so filtering the fully
// reconstructed frame once gives the single-threaded decoder's picture.
//
// The order is part of the result: MB (r, c)'s top edge reads rows 16 r - 4 .. 16 r - 1 of columns 16 c .. 16 c + 15, of which
// (r - 1, c + 1)'s left edge has changed columns 16 c + 13 .. 16 c + 15 (8 samples to a block in chroma).  So (r, c) runs after (r, c - 1)
// and (r - 1, c + 1): a wavefront of slope 2 (the decoder's own check_thread_pos(.., mb_x + 1 + mb_width + 3, mb_y - 1)) with a critical
// path of mb_width + 2 (mb_height - 1) macroblocks.
//
// Frame kernel: one warp per macroblock row, all three planes.  Lanes 0..15 take luma, 16..23 U, 24..31 V: one line each in the column
// pass, one column each in the row pass.  The warp takes its row from an atomicAdd ticket, so every row it waits on belongs to a warp that
// is already running.  The MB sits in shared memory with a 4-sample left halo (the previous MB slid over) and a 4-sample top halo (read
// from global memory after the wait; the MB itself is read before it, since no other warp writes it first).  Before MB c the warp waits
// until row r - 1 has published min(c + 2, mb_width) finished MBs (acquire loads, __nanosleep backoff, bounded by about one second of
// %globaltimer; a wait that runs out is counted in a per-device word read back by b200_vp8_loopfilter_timeouts()), and after its stores,
// the halo samples it changed included, it publishes its own count (fence, release store).
#include "common.h"
#include "wait_timeouts.h"
#include <cstring>

namespace {

constexpr int kY = 20, kC = 12;                              // tile side: 4 halo + 16 (luma) / 8 (chroma) samples
constexpr unsigned long long kWaitNs = 1000000000ull;        // bound of one wait

enum { LF_MBEDGE = 0, LF_INNER = 1, LF_SIMPLE = 2 };         // member kinds

struct LfArgs {
    uint8_t *plane[3];
    long long ls[3];                                         // bytes
    const uint8_t *f;                                        // B200Vp8FilterStrength records, 3 bytes each
    long long fstride;                                       // records
    int *sync;                                               // [0] ticket, [1 + r] MBs finished in row r
    int *timeouts;                                           // waits that ran out, counted for the device (b200_vp8_loopfilter_timeouts)
    int mbw, mbh, vp7, simple, keyframe;
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

__device__ __forceinline__ int clip_s8(int v) { return min(max(v, -128), 127); }
__device__ __forceinline__ int clip_u8(int v) { return min(max(v, 0), 255); }

// filter_common on v[2..5] = p1 p0 q0 q1
__device__ __forceinline__ void lf_common(int (&v)[8], bool four_tap, bool vp7)
{
    const int p1 = v[2], p0 = v[3], q0 = v[4], q1 = v[5];
    int a = 3 * (q0 - p0);
    if (four_tap) a += clip_s8(p1 - q1);
    a = clip_s8(a);
    const int f1 = min(a + 4, 127) >> 3;
    const int f2 = vp7 ? f1 - ((a & 7) == 4) : min(a + 3, 127) >> 3;
    v[3] = clip_u8(p0 + f2);
    v[4] = clip_u8(q0 - f1);
    if (!four_tap) {
        const int g = (f1 + 1) >> 1;
        v[2] = clip_u8(p1 + g);
        v[5] = clip_u8(q1 - g);
    }
}

// one line across an edge, v[0..7] = p3..q3 (the simple kind reads only v[2..5])
__device__ __forceinline__ void lf_line(int (&v)[8], int kind, int E, int I, int H, bool vp7)
{
    const int p3 = v[0], p2 = v[1], p1 = v[2], p0 = v[3], q0 = v[4], q1 = v[5], q2 = v[6], q3 = v[7];
    if (vp7 ? abs(p0 - q0) > E : 2 * abs(p0 - q0) + (abs(p1 - q1) >> 1) > E) return;
    if (kind == LF_SIMPLE) {
        lf_common(v, true, vp7);
        return;
    }
    if (abs(p3 - p2) > I || abs(p2 - p1) > I || abs(p1 - p0) > I || abs(q3 - q2) > I || abs(q2 - q1) > I || abs(q1 - q0) > I) return;
    if (abs(p1 - p0) > H || abs(q1 - q0) > H) {
        lf_common(v, true, vp7);
        return;
    }
    if (kind == LF_INNER) {
        lf_common(v, false, vp7);
        return;
    }
    const int w = clip_s8(clip_s8(p1 - q1) + 3 * (q0 - p0));
    const int a0 = (27 * w + 63) >> 7, a1 = (18 * w + 63) >> 7, a2 = (9 * w + 63) >> 7;
    v[1] = clip_u8(p2 + a2);
    v[2] = clip_u8(p1 + a1);
    v[3] = clip_u8(p0 + a0);
    v[4] = clip_u8(q0 - a0);
    v[5] = clip_u8(q1 - a1);
    v[6] = clip_u8(q2 - a2);
}

// samples at s[k * step], k = -4..3 (simple: -2..1), filtered as one line; only what the kind may write is stored
__device__ __forceinline__ void lf_apply(uint8_t *s, int step, int kind, int E, int I, int H, bool vp7)
{
    const int r = kind == LF_SIMPLE ? 2 : 4, w = kind == LF_MBEDGE ? 3 : kind == LF_INNER ? 2 : 1;
    int v[8];
#pragma unroll
    for (int k = 0; k < 8; k++) v[k] = (k >= 4 - r && k < 4 + r) ? s[(k - 4) * step] : 0;
    lf_line(v, kind, E, I, H, vp7);
#pragma unroll
    for (int k = 0; k < 8; k++)
        if (k >= 4 - w && k < 4 + w) s[(k - 4) * step] = (uint8_t)v[k];
}

// hev_thresh_lut[keyframe][level] (vp8.c:2191-2202) in closed form: one step each at 15, (inter frames only) 20, and 40
__device__ __forceinline__ int hev_thresh(int level, bool keyframe) { return (level >= 15) + (!keyframe && level >= 20) + (level >= 40); }

__global__ void __launch_bounds__(32) vp8_lf_kernel(const __grid_constant__ LfArgs a)
{
    __shared__ uint8_t ty[kY * kY], tu[kC * kC], tv[kC * kC];   // [4 + row][4 + column] of the MB
    __shared__ int s_ticket;
    const int lane = threadIdx.x;
    if (lane == 0) s_ticket = atomicAdd(a.sync, 1);
    __syncwarp();
    const int r = s_ticket;
    if (r >= a.mbh) return;
    const int p = lane < 16 ? 0 : lane < 24 ? 1 : 2, i = lane < 16 ? lane : (lane - 16) & 7, n = p ? 8 : 16, pitch = p ? kC : kY;
    const bool vp7 = a.vp7 != 0, simple = a.simple != 0, active = !simple || p == 0;
    uint8_t *t = p == 0 ? ty : p == 1 ? tu : tv;
    uint8_t *row = t + (4 + i) * pitch + 4, *col = t + 4 * pitch + 4 + i;   // this lane's line (column pass) and column (row pass)
    const long long ls = a.ls[p];
    const int *prev = a.sync + r;
    int *mine = a.sync + 1 + r;
    for (int c = 0; c < a.mbw; c++) {
        uint8_t *g = a.plane[p] + (long long)r * n * ls + (long long)c * n;   // sample (0, 0) of the MB in this lane's plane
        // the previous MB's last 4 columns become the left halo; the MB itself: no other warp writes it before this one is done
        if (active) {
            if (c > 0)
#pragma unroll
                for (int k = 0; k < 4; k++) row[k - 4] = row[n - 4 + k];
            for (int x = 0; x < n; x++) row[x] = __ldcg(g + i * ls + x);
        }
        // byte loads: the 3-byte records sit at every alignment
        const uint8_t *rec = a.f + ((long long)r * a.fstride + c) * 3;
        const int level = rec[0], ilim = rec[1];
        const bool inner = rec[2] != 0, on = level > 0 && level < 64;
        if (r > 0 && lane == 0) {
            const int need = min(c + 2, a.mbw);
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
        __syncwarp();
        // the top halo: rows that (r - 1, c) and (r - 1, c + 1) have finished
        if (active && on && r > 0)
#pragma unroll
            for (int k = 1; k <= 4; k++) col[-k * pitch] = __ldcg(g - k * ls + i);
        __syncwarp();
        // limits (filter_mb, filter_mb_simple)
        int mbE, bE, I = ilim;
        if (simple || !vp7) {
            bE = 2 * level + ilim;
            mbE = bE + 4;
        } else {
            bE = p ? 2 * level : level;
            mbE = level + 2;
        }
        const int H = hev_thresh(level, a.keyframe != 0);
        const int kmb = simple ? LF_SIMPLE : LF_MBEDGE, kin = simple ? LF_SIMPLE : LF_INNER;
        const bool run = active && on;
        // column edges: the left MB edge, then (VP8, simple) the inner ones
        if (run) {
            if (c > 0) lf_apply(row, 1, kmb, mbE, I, H, vp7);
            if (inner && (simple || !vp7))
                for (int e = 4; e < n; e += 4) lf_apply(row + e, 1, kin, bE, I, H, vp7);
        }
        __syncwarp();
        // row edges: the top MB edge, then the inner ones
        if (run) {
            if (r > 0) lf_apply(col, pitch, kmb, mbE, I, H, vp7);
            if (inner)
                for (int e = 4; e < n; e += 4) lf_apply(col + e * pitch, pitch, kin, bE, I, H, vp7);
        }
        __syncwarp();
        // VP7: the inner column edges after the row edges
        if (run && inner && vp7 && !simple)
            for (int e = 4; e < n; e += 4) lf_apply(row + e, 1, kin, bE, I, H, vp7);
        __syncwarp();
        // the MB with the halo samples it may have changed (left: columns -3..-1 of its rows; top: rows -3..-1 of its columns)
        if (run) {
            for (int x = c > 0 ? -3 : 0; x < n; x++) g[i * ls + x] = row[x];
            if (r > 0)
#pragma unroll
                for (int k = 1; k <= 3; k++) g[-k * ls + i] = col[-k * pitch];
        }
        __threadfence();
        __syncwarp();
        if (lane == 0) st_release(mine, c + 1);
    }
}

// ---- drop-in members (host pointers): the footprint across each line (dst[-4..3], simple dst[-2..1]) of the 16 lines (16y) or of the
// 8 lines of U and of V (8uv) goes to a 16 x 8 device scratch laid out like the host's (dir 0, edge between columns: line l is scratch
// row l, pitch 8, q0 at column 4; dir 1, edge between rows: across-offset k is scratch row 4 + k, pitch 16, line l column l; V follows
// U at line 8); one thread per line runs lf_apply, and the samples the kind may write come back.
struct MemberArgs {
    uint8_t *scr;
    int dir, kind, vp7, E, I, H;
};

__global__ void __launch_bounds__(16) vp8_lf_member_kernel(const __grid_constant__ MemberArgs m)
{
    const int l = threadIdx.x;
    lf_apply(m.scr + (m.dir ? 4 * 16 + l : l * 8 + 4), m.dir ? 16 : 1, m.kind, m.E, m.I, m.H, m.vp7 != 0);
}

void member_host(int vp7, int dir, int kind, uint8_t *d0, uint8_t *d1, ptrdiff_t stride, int E, int I, int H)
{
    B200HostCall call("vp8 loop filter", nullptr, 128);
    uint8_t *scr = call.scratch;
    cudaStream_t st = call.stream;
    const int nl = d1 ? 8 : 16;                              // lines per plane
    // plane q's lines and across-offsets -n..n-1: host address, scratch address, bytes per copied row, rows
    auto copy = [&](int q, int n, bool up) {
        uint8_t *hs = (q ? d1 : d0) + (dir ? -(ptrdiff_t)n * stride : -(ptrdiff_t)n);
        uint8_t *ds = scr + (dir ? (size_t)(4 - n) * 16 + (size_t)(q * 8) : (size_t)(q * 8) * 8 + (size_t)(4 - n));
        const size_t dpitch = dir ? 16 : 8, w = dir ? (size_t)nl : 2 * (size_t)n, rows = dir ? 2 * (size_t)n : (size_t)nl;
        return up ? b200_h2d_rows(ds, dpitch, hs, stride, w, rows, st) : b200_d2h_rows(hs, stride, ds, dpitch, w, rows, st);
    };
    const int nr = kind == LF_SIMPLE ? 2 : 4, nw = kind == LF_MBEDGE ? 3 : kind == LF_INNER ? 2 : 1;
    for (int q = 0; q < (d1 ? 2 : 1); q++) call.check(copy(q, nr, true), "h2d edge");
    const MemberArgs m = { scr, dir, kind, vp7, E, I, H };
    vp8_lf_member_kernel<<<1, 16, 0, st>>>(m);
    B200_LAUNCHED();
    call.launched();
    for (int q = 0; q < (d1 ? 2 : 1); q++) call.check(copy(q, nw, false), "d2h edge");
    call.sync();
}

template <int V7, int DIR, int KIND>
void m_16y(uint8_t *dst, ptrdiff_t stride, int E, int I, int H) { member_host(V7, DIR, KIND, dst, nullptr, stride, E, I, H); }
template <int V7, int DIR, int KIND>
void m_8uv(uint8_t *u, uint8_t *v, ptrdiff_t stride, int E, int I, int H) { member_host(V7, DIR, KIND, u, v, stride, E, I, H); }
template <int V7, int DIR>
void m_simple(uint8_t *dst, ptrdiff_t stride, int flim) { member_host(V7, DIR, LF_SIMPLE, dst, nullptr, stride, flim, 0, 0); }

// vp8dsp.c:702-713 / :733-744; v filters the edge between two rows (dir 1), h the edge between two columns (dir 0)
template <int V7>
void fill(B200VP8DSPContext *c)
{
    c->vp8_v_loop_filter16y = m_16y<V7, 1, LF_MBEDGE>;
    c->vp8_h_loop_filter16y = m_16y<V7, 0, LF_MBEDGE>;
    c->vp8_v_loop_filter8uv = m_8uv<V7, 1, LF_MBEDGE>;
    c->vp8_h_loop_filter8uv = m_8uv<V7, 0, LF_MBEDGE>;
    c->vp8_v_loop_filter16y_inner = m_16y<V7, 1, LF_INNER>;
    c->vp8_h_loop_filter16y_inner = m_16y<V7, 0, LF_INNER>;
    c->vp8_v_loop_filter8uv_inner = m_8uv<V7, 1, LF_INNER>;
    c->vp8_h_loop_filter8uv_inner = m_8uv<V7, 0, LF_INNER>;
    c->vp8_v_loop_filter_simple = m_simple<V7, 1>;
    c->vp8_h_loop_filter_simple = m_simple<V7, 0>;
}

} // namespace

B200_API int b200_vp8_dsp_init_loopfilter(B200VP8DSPContext *c, int is_vp7)
{
    if (!c || (is_vp7 != 0 && is_vp7 != 1)) { b200_set_error("vp8 loop filter init: NULL context or is_vp7 not 0 / 1"); return B200_EINVAL; }
    if (!b200_default_device()) return B200_ENODEV;
    if (is_vp7) fill<1>(c);
    else fill<0>(c);
    return 0;
}

B200_API int b200_vp8_loopfilter_frame_device(B200Device *dev, int is_vp7, int simple, int keyframe, int mb_width, int mb_height,
                                              uint8_t *const planes[3], ptrdiff_t ls_y, ptrdiff_t ls_uv, const B200Vp8FilterStrength *f,
                                              int64_t f_stride)
{
    if (!planes || !planes[0] || !planes[1] || !planes[2] || !f) { b200_set_error("vp8 loop filter frame: NULL pointer"); return B200_EINVAL; }
    if ((is_vp7 != 0 && is_vp7 != 1) || (simple != 0 && simple != 1) || (keyframe != 0 && keyframe != 1)) {
        b200_set_error("vp8 loop filter frame: is_vp7, simple or keyframe not 0 / 1");
        return B200_EINVAL;
    }
    if (mb_width < 1 || mb_height < 1) { b200_set_error("vp8 loop filter frame: %dx%d macroblocks", mb_width, mb_height); return B200_EINVAL; }
    if (ls_y < 16 * (ptrdiff_t)mb_width || ls_uv < 8 * (ptrdiff_t)mb_width) {
        b200_set_error("vp8 loop filter frame: line size shorter than a plane row");
        return B200_EINVAL;
    }
    if (f_stride < mb_width) { b200_set_error("vp8 loop filter frame: f_stride %lld below %d", (long long)f_stride, mb_width); return B200_EINVAL; }
    if (int r = b200_use_device(dev)) return r;
    B200_LOCK_DEVICE(dev);
    int *timeouts = b200_wait_timeouts_word(dev->ordinal, B200_WAIT_VP8_LOOPFILTER, true);
    if (!timeouts) { b200_set_error("vp8 loop filter frame: no timeout counter for device %d", dev->ordinal); return B200_ENOMEM; }
    const size_t sync_bytes = sizeof(int) * (1 + (size_t)mb_height);
    int *sync = (int *)b200_scratch(dev, sync_bytes);
    if (!sync) return B200_ENOMEM;
    LfArgs a;
    memset(&a, 0, sizeof(a));
    for (int p = 0; p < 3; p++) a.plane[p] = planes[p];
    a.ls[0] = ls_y;
    a.ls[1] = a.ls[2] = ls_uv;
    a.f = reinterpret_cast<const uint8_t *>(f);
    a.fstride = f_stride;
    a.sync = sync;
    a.timeouts = timeouts;
    a.mbw = mb_width;
    a.mbh = mb_height;
    a.vp7 = is_vp7;
    a.simple = simple;
    a.keyframe = keyframe;
    B200_CUDA_OK(cudaMemsetAsync(sync, 0, sync_bytes, dev->stream));
    vp8_lf_kernel<<<(unsigned)mb_height, 32, 0, dev->stream>>>(a);
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

B200_API int b200_vp8_loopfilter_timeouts(B200Device *dev, int64_t *count)
{
    if (!count) { b200_set_error("vp8 loop filter timeouts: NULL pointer"); return B200_EINVAL; }
    if (int r = b200_use_device(dev)) return r;
    B200_CUDA_OK(cudaStreamSynchronize(dev->stream));
    int v = 0;
    int *w = b200_wait_timeouts_word(dev->ordinal, B200_WAIT_VP8_LOOPFILTER, false);
    if (w) B200_CUDA_OK(cudaMemcpy(&v, w, sizeof(int), cudaMemcpyDeviceToHost));
    *count = v;
    return 0;
}
