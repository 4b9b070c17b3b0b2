// vp9intra.cu — VP9 intra reconstruction on sm_90a: the intra_pred[4][15] members of VP9DSPContext (libavcodec/vp9dsp.h:40-122) as
// ff_vp9dsp_intrapred_init fills them for 8, 10 and 12 bit samples (vp9dsp_template.c:1120-1152), and a frame entry that runs
// intra_recon (vp9recon.c:219-287) over every intra transform block of a frame in one launch: prediction and residual add fused per block.
//
// Reference semantics reproduced bit for bit (checker: oracle/vp9intra_oracle.c):
//   predictors   vp9dsp_template.c:33-1106 restated per output sample in pred_px below: the directional modes as 3-tap / 2-tap averages
//                of one edge array (left bottom-to-top, the top-left sample, the top row), 4x4 DL's DST(3,3) = top[7], DL and VL at 8x8
//                and up replicating top[size - 1], TM clipped to the depth, DC_127 / 128 / 129 = (128 << (depth - 8)) - 1 / + 0 / + 1
//   edges        check_intra_mode (vp9recon.c:33-217) in closed form: mode_conv, the top row copied up to n_px_have = (cols * 8 >> ss_h)
//                - x samples and its last one replicated (127-like with no top), the top-left sample (129-like / 127-like without a
//                left / top), the 4x4 top-right only with have_right and 8 <= n_px_have (else top[3] replicated), the left column
//                likewise down to (rows * 8 >> ss_v) - y, bottom-to-top except for HU (129-like with no left)
//   residual     itxfm_add[4 * lossless + tx][txtp] (vp9itxfm_dev.cuh), txtp = ff_vp9_intra_txfm_type[mode] for luma, DCT_DCT for chroma
//
// The top row at a superblock row's top comes from the plane, not from a copy: the decoder's intra_pred_data holds the row before the
// loop filter (vp9.c:1387-1398), and the loop filter entry runs after this one, so the two are the same samples.
//
// Frame kernel: one warp per op, 4 warps per CTA, each with its own shared memory and no CTA-wide barrier.  A warp takes ops by an
// atomicAdd ticket in decode order, so every op it waits on has a smaller ticket and is held by a warp that is already running: the
// smallest unfinished op can always proceed, whatever else shares the GPU.  A marking launch first records, per 4x4 cell of each plane,
// the op that writes it (-1: not written by an intra op of this call).  Op t then waits, with acquire loads, only on the earlier ops that
// own a cell its mode reads (left column, top row, top-left, 4x4 top-right), reads the edges through L2, predicts, runs the inverse
// transform when eob is non-zero, adds and clips, stores the part of the block inside the plane, and publishes (fence, release store).
// Every wait is bounded by about one second of %globaltimer: a scheduling mistake gives wrong samples, never a hung GPU, and each wait
// that runs out is counted for b200_vp9_intra_timeouts().
#include "common.h"
#include "vp9itxfm_dev.cuh"
#include "wait_timeouts.h"
#include <cstring>

namespace {

// IntraPredMode (libavcodec/vp9.h:45-61)
enum { VERT = 0, HOR, DC, DIAG_DL, DIAG_DR, VERT_R, HOR_D, VERT_L, HOR_U, TM, LEFT_DC, TOP_DC, DC_128, DC_127, DC_129 };
enum { NEED_LEFT = 1, NEED_TOP = 2, NEED_TL = 4, NEED_TR = 8 };

constexpr int kWarps = 4;                                    // ops in flight per CTA
constexpr int kMaxCtas = 2048;                               // enough to fill the GPU; further warps would only find the tickets gone
constexpr unsigned long long kWaitNs = 1000000000ull;        // bound of one wait
constexpr int kTop = 9 + 32;                                 // top[-1 .. 31] (and top[4..7] of 4x4), as tb[k + 1]

struct IntraArgs {
    uint8_t *plane[3];
    long long ls[3];                                         // bytes
    const B200Vp9IntraOp *ops;
    const void *coef;
    int *sync;                                               // [0] ticket, [1 + k] op k published
    int *owner[3];                                           // per plane, cell (cy, cx) at [cy * cw + cx]: the op that writes it, or -1
    int *timeouts;                                           // waits that ran out (b200_vp9_intra_timeouts)
    int cw[3], W[3], H[3];                                   // cells per row; plane size in samples, the 8-aligned area
    int nops, depth;
};

// ---- inter-warp progress
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
// ---- end of inter-warp progress

// check_intra_mode's edges[] (vp9recon.c:67-93)
__host__ __device__ __forceinline__ int needs(int m)
{
    switch (m) {
    case VERT: case TOP_DC: return NEED_TOP;
    case HOR: case HOR_U: case LEFT_DC: return NEED_LEFT;
    case DC: return NEED_LEFT | NEED_TOP;
    case DIAG_DL: case VERT_L: return NEED_TOP | NEED_TR;
    case DIAG_DR: case VERT_R: case HOR_D: case TM: return NEED_LEFT | NEED_TOP | NEED_TL;
    default: return 0;
    }
}

// mode_conv[mode][have_left][have_top] (vp9recon.c:45-66)
__device__ __forceinline__ int conv_mode(int m, bool hl, bool ht)
{
    switch (m) {
    case VERT: case DIAG_DL: case VERT_L: return ht ? m : DC_127;
    case HOR: case HOR_U: return hl ? m : DC_129;
    case DC: return hl ? (ht ? DC : LEFT_DC) : (ht ? TOP_DC : DC_128);
    case TM: return hl ? (ht ? TM : HOR) : (ht ? VERT : DC_129);
    default: return m;
    }
}

__host__ __device__ __forceinline__ int avg2(int a, int b) { return (a + b + 1) >> 1; }
__host__ __device__ __forceinline__ int avg3(int a, int b, int c) { return (a + 2 * b + c + 2) >> 2; }

// sample (i, j) (column, row) of predictor m of size 1 << l2, from top[k] = tb[k + 1] (k >= -1) and the reference's left[] = lb
// (bottom-to-top, top-to-bottom for HU); dc = the block's value for the DC family (block_dc).  DR, VR and HD read the edge array
// E = left[0 .. n-1], top[-1], top[0 .. n-1].
__device__ __forceinline__ int pred_px(int m, int l2, int i, int j, const int *tb, const int *lb, int dc, int maxv)
{
    const int n = 1 << l2;
    auto T = [tb](int k) { return tb[k + 1]; };
    auto E = [tb, lb, n](int k) { return k < n ? lb[k] : tb[k - n]; };
    switch (m) {
    case VERT: return T(i);
    case HOR: return lb[n - 1 - j];
    case TM: return min(max(T(i) + lb[n - 1 - j] - T(-1), 0), maxv);
    case DIAG_DL: {
        const int s = i + j, e = n - 1;
        if (n == 4) return s == 6 ? T(7) : avg3(T(s), T(s + 1), T(s + 2));
        return avg3(T(min(s, e)), T(min(s + 1, e)), T(min(s + 2, e)));
    }
    case DIAG_DR: {
        const int k = n - 1 - j + i;
        return avg3(E(k), E(k + 1), E(k + 2));
    }
    case VERT_R: {                                           // rows 2h / 2h + 1 = ve / vo from n / 2 - 1 - h
        const int h = n / 2 - 1, k = h - (j >> 1) + i;
        if (k >= h) {
            const int q = n + k - h;
            return (j & 1) ? avg3(E(q - 1), E(q), E(q + 1)) : avg2(E(q), E(q + 1));
        }
        return (j & 1) ? avg3(E(2 * k + 1), E(2 * k + 2), E(2 * k + 3)) : avg3(E(2 * k + 2), E(2 * k + 3), E(2 * k + 4));
    }
    case HOR_D: {                                            // row j = v[2n - 2 - 2j ..]
        const int q = 2 * n - 2 - 2 * j + i;
        if (q >= 2 * n) return avg3(E(q - n), E(q - n + 1), E(q - n + 2));
        const int k = q >> 1;
        return (q & 1) ? avg3(E(k), E(k + 1), E(k + 2)) : avg2(E(k), E(k + 1));
    }
    case VERT_L: {                                           // rows 2h / 2h + 1 = ve / vo from h, top[e] past the end
        const int e = n == 4 ? 7 : n - 1, k = (j >> 1) + i;
        if (k >= e) return T(e);
        return (j & 1) ? avg3(T(k), T(min(k + 1, e)), T(min(k + 2, e))) : avg2(T(k), T(min(k + 1, e)));
    }
    case HOR_U: {                                            // row j = v[2j ..], left[n - 1] past the end
        const int q = 2 * j + i, e = n - 1, k = q >> 1;
        if (q >= 2 * n - 2) return lb[e];
        return (q & 1) ? avg3(lb[k], lb[min(k + 1, e)], lb[min(k + 2, e)]) : avg2(lb[k], lb[min(k + 1, e)]);
    }
    default: return dc;
    }
}

// the DC family's value (warp-wide: every lane calls it with the same arguments)
__device__ __forceinline__ int block_dc(int m, int l2, const int *tb, const int *lb, int depth, int lane)
{
    const int base = 128 << (depth - 8);
    if (m == DC_128 || m == DC_127 || m == DC_129) return base + (m == DC_127 ? -1 : m == DC_129 ? 1 : 0);
    if (m != DC && m != LEFT_DC && m != TOP_DC) return 0;
    int s = 0;
    if (lane < (1 << l2)) s = (m != TOP_DC ? lb[lane] : 0) + (m != LEFT_DC ? tb[lane + 1] : 0);
    for (int d = 16; d; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
    const int sh = m == DC ? l2 + 1 : l2;
    return (s + (1 << (sh - 1))) >> sh;
}

// itxfm_add's two passes over the warp's coefficient block A (n x n, row-major) into the residual A[j * n + i] of row j, column i
template <typename P, int N>
__device__ __forceinline__ void residual(int ta, int tb, int bits, typename Store<P>::C *A, typename Store<P>::Tmp *B, int lane)
{
    using C = typename Store<P>::C;
    using Tmp = typename Store<P>::Tmp;
    constexpr int pitch = N + Store<P>::kPad;
    if (lane < N) {
        C x[N];
        Tmp y[N];
#pragma unroll
        for (int k = 0; k < N; k++) x[k] = A[k * N + lane];
        tx1d<P, N>(ta, true, x, y);
#pragma unroll
        for (int k = 0; k < N; k++) B[k * pitch + lane] = y[k];
    }
    __syncwarp();
    if (lane < N) {
        Tmp x[N], y[N];
#pragma unroll
        for (int k = 0; k < N; k++) x[k] = B[lane * pitch + k];
        tx1d<P, N>(tb, false, x, y);
#pragma unroll
        for (int j = 0; j < N; j++)
            A[j * N + lane] = bits ? (C)((int)((unsigned)(int)y[j] + (1u << (bits - 1))) >> bits) : y[j];
    }
    __syncwarp();
}

__device__ __forceinline__ bool op_ok(const B200Vp9IntraOp &op)
{
    return op.plane <= 2 && op.tx <= 3 && op.mode <= 9 && op.x >= 0 && op.y >= 0 && !(op.x & 3) && !(op.y & 3) && op.coef_off >= 0 &&
           !(op.coef_off & 15) && (!(op.flags & B200_VP9_INTRA_LOSSLESS) || op.tx == 0);
}

// the marking launch: each op's cells inside its plane get its index
__global__ void vp9_intra_mark_kernel(const __grid_constant__ IntraArgs a)
{
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= a.nops) return;
    const B200Vp9IntraOp op = a.ops[k];
    if (!op_ok(op)) return;
    const int p = op.plane, n = 4 << op.tx;
    const int x1 = min(op.x + n, a.W[p]), y1 = min(op.y + n, a.H[p]);
    for (int cy = op.y >> 2; cy < (y1 + 3) >> 2; cy++)
        for (int cx = op.x >> 2; cx < (x1 + 3) >> 2; cx++) a.owner[p][(long long)cy * a.cw[p] + cx] = (int)k;
}

template <typename P>
__global__ void __launch_bounds__(32 * kWarps) vp9_intra_kernel(const __grid_constant__ IntraArgs a)
{
    using C = typename Store<P>::C;
    using Tmp = typename Store<P>::Tmp;
    using T = typename Store<P>::T;
    __shared__ C sA[kWarps][32 * 32];
    __shared__ Tmp sB[kWarps][32 * (32 + Store<P>::kPad)];
    __shared__ int sT[kWarps][kTop], sL[kWarps][32], sTicket[kWarps];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int *tb = sT[w], *lb = sL[w];
    const int base = 128 << (a.depth - 8), maxv = (1 << a.depth) - 1;
    for (;;) {
        if (lane == 0) sTicket[w] = atomicAdd(a.sync, 1);
        __syncwarp();
        const int t = sTicket[w];
        __syncwarp();
        if (t >= a.nops) break;
        const B200Vp9IntraOp op = a.ops[t];
        const int p = op.plane;
        if (op_ok(op) && op.x < a.W[p] && op.y < a.H[p]) {
            const int l2 = op.tx + 2, n = 1 << l2, x = op.x, y = op.y;
            const bool ht = y > 0, hl = op.flags & B200_VP9_INTRA_HAVE_LEFT, hr = op.flags & B200_VP9_INTRA_HAVE_RIGHT;
            const int m = conv_mode(op.mode, hl, ht), nm = needs(m);
            const int nh = a.W[p] - x, nv = a.H[p] - y;               // n_px_have of the top row and of the left column
            const bool tr = n == 4 && (nm & NEED_TR) && ht && hr && 8 <= nh;
            uint8_t *pl = a.plane[p];
            const long long ls = a.ls[p];
            auto at = [pl, ls](int yy, int xx) { return reinterpret_cast<P *>(pl + (long long)yy * ls) + xx; };
            // wait for the ops that own the cells this mode reads: the top row, the top-right, the top-left and the left column
            {
                const int ntop = (nm & NEED_TOP) && ht ? ((x + min(n, nh) - 1) >> 2) - (x >> 2) + 1 + (tr ? 1 : 0) : 0;
                const int ntl = (nm & NEED_TL) && ht && hl ? 1 : 0;
                const int nleft = (nm & NEED_LEFT) && hl ? ((y + min(n, nv) - 1) >> 2) - (y >> 2) + 1 : 0;
                int cy = -1, cx = 0;
                if (lane < ntop) cy = (y - 1) >> 2, cx = (x >> 2) + lane;
                else if (lane < ntop + ntl) cy = (y - 1) >> 2, cx = (x - 1) >> 2;
                else if (lane < ntop + ntl + nleft) cy = (y >> 2) + lane - ntop - ntl, cx = (x - 1) >> 2;
                if (cy >= 0) {
                    const int o = a.owner[p][(long long)cy * a.cw[p] + cx];
                    if (o >= 0 && o < t && !ld_acquire(a.sync + 1 + o)) {
                        const unsigned long long t0 = globaltimer();
                        unsigned ns = 32;
                        while (!ld_acquire(a.sync + 1 + o) && globaltimer() - t0 < kWaitNs) {
                            __nanosleep(ns);
                            ns = min(ns * 2, 1024u);
                        }
                        if (!ld_acquire(a.sync + 1 + o)) atomicAdd(a.timeouts, 1);
                    }
                }
            }
            __syncwarp();
            // the edges, through L2 (samples other warps of this launch have written)
            if (nm & NEED_TOP) {
                const int ne = n == 4 && (nm & NEED_TR) ? 8 : n;
                for (int k = lane - 1; k < ne; k += 32) {
                    int v;
                    if (k < 0) v = !(nm & NEED_TL) ? 0 : ht && hl ? (int)__ldcg(at(y - 1, x - 1)) : ht ? base + 1 : base - 1;
                    else if (!ht) v = base - 1;
                    else if (k < n) v = __ldcg(at(y - 1, x + min(k, nh - 1)));
                    else v = tr ? (int)__ldcg(at(y - 1, x + k)) : (int)__ldcg(at(y - 1, x + min(3, nh - 1)));
                    tb[k + 1] = v;
                }
            }
            if (nm & NEED_LEFT)
                for (int i = lane; i < n; i += 32) lb[m == HOR_U ? i : n - 1 - i] = hl ? (int)__ldcg(at(y + min(i, nv - 1), x - 1)) : base + 1;
            __syncwarp();
            const int dc = block_dc(m, l2, tb, lb, a.depth, lane);
            // the residual
            const bool lossless = op.flags & B200_VP9_INTRA_LOSSLESS;
            const int txtp = p ? 0 : (op.mode == VERT || op.mode == VERT_R || op.mode == VERT_L) ? 2       // ff_vp9_intra_txfm_type
                             : (op.mode == HOR || op.mode == HOR_D || op.mode == HOR_U) ? 1 : (op.mode == DIAG_DR || op.mode == TM) ? 3 : 0;
            const bool dconly = !lossless && op.eob == 1 && (op.tx == 3 || txtp == 0);
            const int bits = lossless ? 0 : op.tx < 2 ? 4 + op.tx : 6;
            C *A = sA[w];
            int rdc = 0;
            if (op.eob) {
                const C *src = reinterpret_cast<const C *>(a.coef) + op.coef_off;
                if (dconly) {
                    const T t1 = r14(mul((T)src[0], 11585));
                    const int v = (int)r14(mul(t1, 11585));
                    rdc = (int)((unsigned)v + (1u << (bits - 1))) >> bits;
                } else {
                    for (int e = lane; e < n * n; e += 32) A[e] = src[e];
                    __syncwarp();
                    const int ta = lossless ? T_WHT : op.tx == 3 ? T_DCT : (txtp & 1) ? T_ADST : T_DCT;
                    const int tb2 = lossless ? T_WHT : op.tx == 3 ? T_DCT : (txtp & 2) ? T_ADST : T_DCT;
                    switch (op.tx) {
                    case 0:  residual<P, 4>(ta, tb2, bits, A, sB[w], lane); break;
                    case 1:  residual<P, 8>(ta, tb2, bits, A, sB[w], lane); break;
                    case 2:  residual<P, 16>(ta, tb2, bits, A, sB[w], lane); break;
                    default: residual<P, 32>(ta, tb2, bits, A, sB[w], lane); break;
                    }
                }
            }
            // predict, add, clip, store the part inside the plane
            for (int e = lane; e < n * n; e += 32) {
                const int i = e & (n - 1), j = e >> l2;
                if (x + i >= a.W[p] || y + j >= a.H[p]) continue;
                int v = pred_px(m, l2, i, j, tb, lb, dc, maxv);
                if (op.eob) v = min(max((int)((unsigned)v + (unsigned)(dconly ? rdc : (int)A[e])), 0), maxv);
                *at(y + j, x + i) = (P)v;
            }
        }
        __threadfence();
        __syncwarp();
        if (lane == 0) st_release(a.sync + 1 + t, 1);
    }
}

bool depth_ok(int d) { return d == 8 || d == 10 || d == 12; }

// ---- drop-in members (host pointers): the samples the reference function reads go to a device scratch (top[-1 ..] at sample 0, left[]
// at sample kTop), one warp predicts the block with pred_px, and the block comes back.
struct MemberArgs {
    uint8_t *scr;
    int mode, l2, depth;
};

template <typename P>
__global__ void __launch_bounds__(32) vp9_intra_member_kernel(const __grid_constant__ MemberArgs m)
{
    __shared__ int tb[kTop], lb[32];
    const int lane = threadIdx.x, n = 1 << m.l2;
    const P *s = reinterpret_cast<const P *>(m.scr);
    for (int k = lane; k < kTop; k += 32) tb[k] = s[k];
    lb[lane] = s[kTop + lane];
    __syncwarp();
    const int dc = block_dc(m.mode, m.l2, tb, lb, m.depth, lane);
    P *blk = reinterpret_cast<P *>(m.scr) + kTop + 32;
    for (int e = lane; e < n * n; e += 32) blk[e] = (P)pred_px(m.mode, m.l2, e & (n - 1), e >> m.l2, tb, lb, dc, (1 << m.depth) - 1);
}

// the samples predictor `mode` of size n reads (vp9dsp_template.c:33-1106): top[t0 .. t1 - 1], left[l0 .. l1 - 1]
void footprint(int mode, int n, int &t0, int &t1, int &l0, int &l1)
{
    t0 = t1 = l0 = l1 = 0;
    switch (mode) {
    case VERT: case DC: case TOP_DC: t1 = n; break;
    case DIAG_DL: t1 = n == 4 ? 8 : n; break;
    case VERT_L: t1 = n == 4 ? 7 : n; break;
    case DIAG_DR: case VERT_R: case TM: t0 = -1, t1 = n; break;
    case HOR_D: t0 = -1, t1 = n - 1; break;
    default: break;
    }
    switch (mode) {
    case HOR: case DC: case LEFT_DC: case DIAG_DR: case HOR_D: case HOR_U: case TM: l1 = n; break;
    case VERT_R: l0 = 1, l1 = n; break;
    default: break;
    }
}

void member_host(int depth, int tx, int mode, uint8_t *dst, ptrdiff_t stride, const uint8_t *left, const uint8_t *top)
{
    const int n = 4 << tx, bps = depth > 8 ? 2 : 1;
    B200HostCall call("vp9 intra prediction", nullptr, (size_t)(kTop + 32 + 32 * 32) * bps);
    uint8_t *scr = call.scratch;
    cudaStream_t st = call.stream;
    int t0, t1, l0, l1;
    footprint(mode, n, t0, t1, l0, l1);
    call.check(cudaMemsetAsync(scr, 0, (size_t)(kTop + 32) * bps, st), "memset");
    if (t1 > t0)
        call.check(cudaMemcpyAsync(scr + (size_t)(t0 + 1) * bps, top + (ptrdiff_t)t0 * bps, (size_t)(t1 - t0) * bps, cudaMemcpyHostToDevice, st), "h2d top");
    if (l1 > l0)
        call.check(cudaMemcpyAsync(scr + (size_t)(kTop + l0) * bps, left + (ptrdiff_t)l0 * bps, (size_t)(l1 - l0) * bps, cudaMemcpyHostToDevice, st), "h2d left");
    const MemberArgs m = { scr, mode, tx + 2, depth };
    if (depth == 8) vp9_intra_member_kernel<uint8_t><<<1, 32, 0, st>>>(m);
    else vp9_intra_member_kernel<uint16_t><<<1, 32, 0, st>>>(m);
    B200_LAUNCHED();
    call.launched();
    call.check(b200_d2h_rows(dst, stride, scr + (size_t)(kTop + 32) * bps, (size_t)n * bps, (size_t)n * bps, (size_t)n, st), "d2h block");
    call.sync();
}

template <int D, int TX, int MODE>
void m_pred(uint8_t *dst, ptrdiff_t stride, const uint8_t *left, const uint8_t *top) { member_host(D, TX, MODE, dst, stride, left, top); }

// vp9dsp_template.c:1120-1152: at 12 bit only TM and the DC_127 / 128 / 129 functions are 12-bit ones, the rest are the 10-bit functions
template <int D, int TX>
void fill_size(B200VP9DSPContext *c)
{
    constexpr int S = D == 12 ? 10 : D;
    c->intra_pred[TX][VERT] = m_pred<S, TX, VERT>;
    c->intra_pred[TX][HOR] = m_pred<S, TX, HOR>;
    c->intra_pred[TX][DC] = m_pred<S, TX, DC>;
    c->intra_pred[TX][DIAG_DL] = m_pred<S, TX, DIAG_DL>;
    c->intra_pred[TX][DIAG_DR] = m_pred<S, TX, DIAG_DR>;
    c->intra_pred[TX][VERT_R] = m_pred<S, TX, VERT_R>;
    c->intra_pred[TX][HOR_D] = m_pred<S, TX, HOR_D>;
    c->intra_pred[TX][VERT_L] = m_pred<S, TX, VERT_L>;
    c->intra_pred[TX][HOR_U] = m_pred<S, TX, HOR_U>;
    c->intra_pred[TX][LEFT_DC] = m_pred<S, TX, LEFT_DC>;
    c->intra_pred[TX][TOP_DC] = m_pred<S, TX, TOP_DC>;
    c->intra_pred[TX][TM] = m_pred<D, TX, TM>;
    c->intra_pred[TX][DC_128] = m_pred<D, TX, DC_128>;
    c->intra_pred[TX][DC_127] = m_pred<D, TX, DC_127>;
    c->intra_pred[TX][DC_129] = m_pred<D, TX, DC_129>;
}
template <int D>
void fill(B200VP9DSPContext *c)
{
    fill_size<D, 0>(c); fill_size<D, 1>(c); fill_size<D, 2>(c); fill_size<D, 3>(c);
}

} // namespace

B200_API int b200_vp9_dsp_init_intrapred(B200VP9DSPContext *c, int bit_depth)
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

B200_API int b200_vp9_intra_recon_frame_device(B200Device *dev, int bit_depth, int ss_h, int ss_v, int width, int height,
                                               uint8_t *const planes[3], ptrdiff_t ls_y, ptrdiff_t ls_uv, int64_t nops,
                                               const B200Vp9IntraOp *ops, const void *coef)
{
    if (!planes || !planes[0] || !planes[1] || !planes[2]) { b200_set_error("vp9 intra frame: NULL plane"); return B200_EINVAL; }
    if (!depth_ok(bit_depth)) { b200_set_error("vp9 intra frame: bit depth %d is not 8, 10 or 12", bit_depth); return B200_EINVAL; }
    if ((ss_h != 0 && ss_h != 1) || (ss_v != 0 && ss_v != 1)) { b200_set_error("vp9 intra frame: ss_h / ss_v not 0 or 1"); return B200_EINVAL; }
    if (width < 1 || height < 1 || width > 65536 || height > 65536) { b200_set_error("vp9 intra frame: %dx%d picture", width, height); return B200_EINVAL; }
    if (nops < 0 || nops > (1LL << 30)) { b200_set_error("vp9 intra frame: nops %lld outside 0 .. 2^30", (long long)nops); return B200_EINVAL; }
    const int bps = bit_depth > 8 ? 2 : 1;
    const int cols = (width + 7) >> 3, rows = (height + 7) >> 3;
    const int W[3] = { cols * 8, (cols * 8) >> ss_h, (cols * 8) >> ss_h }, H[3] = { rows * 8, (rows * 8) >> ss_v, (rows * 8) >> ss_v };
    if (ls_y < (long long)W[0] * bps || ls_uv < (long long)W[1] * bps || ls_y % bps || ls_uv % bps) {
        b200_set_error("vp9 intra frame: stride shorter than a plane row or not a whole number of samples");
        return B200_EINVAL;
    }
    for (int p = 0; p < 3; p++)
        if ((uintptr_t)planes[p] % bps) { b200_set_error("vp9 intra frame: plane %d not aligned to a sample", p); return B200_EINVAL; }
    if (nops == 0) return 0;
    if (!ops || !coef || ((uintptr_t)ops & 7) || ((uintptr_t)coef & 15)) {
        b200_set_error("vp9 intra frame: ops / coef NULL or misaligned");
        return B200_EINVAL;
    }
    if (int r = b200_use_device(dev)) return r;
    B200_LOCK_DEVICE(dev);
    int *timeouts = b200_wait_timeouts_word(dev->ordinal, B200_WAIT_VP9_INTRA, true);
    if (!timeouts) { b200_set_error("vp9 intra frame: no timeout counter for device %d", dev->ordinal); return B200_ENOMEM; }
    // scratch: the ticket and one published flag per op, then the three cell maps
    size_t cells[3], bytes = sizeof(int) * (((size_t)nops + 1 + 3) & ~(size_t)3);
    const size_t sync_bytes = bytes;
    for (int p = 0; p < 3; p++) {
        cells[p] = (size_t)(W[p] >> 2) * (size_t)(H[p] >> 2);
        bytes += sizeof(int) * ((cells[p] + 3) & ~(size_t)3);
    }
    int *scr = (int *)b200_scratch(dev, bytes);
    if (!scr) return B200_ENOMEM;
    IntraArgs a;
    memset(&a, 0, sizeof(a));
    size_t off = sync_bytes / sizeof(int);
    for (int p = 0; p < 3; p++) {
        a.plane[p] = planes[p];
        a.ls[p] = p ? ls_uv : ls_y;
        a.owner[p] = scr + off;
        off += (cells[p] + 3) & ~(size_t)3;
        a.cw[p] = W[p] >> 2;
        a.W[p] = W[p];
        a.H[p] = H[p];
    }
    a.ops = ops;
    a.coef = coef;
    a.sync = scr;
    a.timeouts = timeouts;
    a.nops = (int)nops;
    a.depth = bit_depth;
    B200_CUDA_OK(cudaMemsetAsync(scr, 0, sync_bytes, dev->stream));
    B200_CUDA_OK(cudaMemsetAsync(a.owner[0], 0xFF, bytes - sync_bytes, dev->stream));
    vp9_intra_mark_kernel<<<(unsigned)((nops + 255) / 256), 256, 0, dev->stream>>>(a);
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    const long long ctas = (nops + kWarps - 1) / kWarps;
    const unsigned grid = (unsigned)(ctas < kMaxCtas ? ctas : kMaxCtas);
    if (bit_depth == 8) vp9_intra_kernel<uint8_t><<<grid, 32 * kWarps, 0, dev->stream>>>(a);
    else vp9_intra_kernel<uint16_t><<<grid, 32 * kWarps, 0, dev->stream>>>(a);
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

B200_API int b200_vp9_intra_timeouts(B200Device *dev, int64_t *count)
{
    if (!count) { b200_set_error("vp9 intra timeouts: NULL pointer"); return B200_EINVAL; }
    if (int r = b200_use_device(dev)) return r;
    B200_CUDA_OK(cudaStreamSynchronize(dev->stream));
    int v = 0;
    int *w = b200_wait_timeouts_word(dev->ordinal, B200_WAIT_VP9_INTRA, false);
    if (w) B200_CUDA_OK(cudaMemcpy(&v, w, sizeof(int), cudaMemcpyDeviceToHost));
    *count = v;
    return 0;
}
