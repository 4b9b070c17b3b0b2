// hevcpred.cu — HEVC intra prediction on sm_90a: the members of HEVCPredContext (libavcodec/hevc/pred.h) that ff_hevc_pred_init fills
// (pred_planar[4], pred_dc, pred_angular[4], ref_filter_3tap[3], ref_filter_strong; intra_pred[] takes decoder structs and stays NULL)
// for 8, 9, 10 and 12 bit samples, and a batched entry that runs intra_pred (hevc/pred_template.c) for a set of independent TUs.
//
// Per op, the kernel follows intra_pred's data flow, bit for bit (checked against the reference's own intra_pred, tests/test_hevc_pred.py):
//   1. neighbours: the left column left[-1..2 * size - 1] and the top row top[-1..2 * size - 1] in shared memory, taken from the plane
//      where the op's CAND_* flags allow (the bottom-left and top-right runs clipped to the picture and extended with their last sample);
//   2. constrained intra prediction (intra_map given): the PU checks that can clear a flag, the arrays preset to the byte 128, and the
//      substitution over the intra / inter map, lane-serial (CIP streams are rare), with the reference's quirks;
//   3. the substitution of unavailable runs, in closed form: in the scan order bottom-left, left, corner, top, top-right, an unavailable
//      run takes the last sample of the nearest available run before it, or the first sample of the first available run when none is
//      before it, and every sample is 1 << (depth - 1) when no run is available (the reference's if-chain, pred_template.c:296-332);
//   4. the filter decision and the 3-tap or strong filter;
//   5. planar / DC / angular, each lane computing runs of 4 samples and storing them as one word where aligned.
// A CTA of 4 warps takes 4 ops, one warp each.
#include "common.h"
#include <cstring>
#include <type_traits>

namespace {

constexpr int kOpsPerCta = 4;
constexpr int kPad = 4;                          // elements before index -1 (the CIP up-extension writes down to index -3)
constexpr int kArr = kPad + 1 + 128 + 8;         // one edge array: [-kPad - 1, 136)
constexpr int kRef = 3 * 32 + 8;                 // ref_tmp of pred_angular: [-size, size + 4)
constexpr int kWarpInts = 4 * kArr + kRef;       // left, top, filtered left, filtered top, ref_tmp

// ---- the filters, shared by the kernel and the host members (A = int for shared arrays, the sample type on the host)
// ref_filter_3tap's output at index i of an edge array of n = 2 * size samples (i in 0..n - 1); index -1 is filt3_corner
template <typename A>
__host__ __device__ __forceinline__ int filt3(const A *a, int i, int n)
{
    return i == n - 1 ? (int)a[n - 1] : ((int)a[i + 1] + 2 * (int)a[i] + (int)a[i - 1] + 2) >> 2;
}
template <typename A>
__host__ __device__ __forceinline__ int filt3_corner(const A *left, const A *top)
{
    return ((int)left[0] + 2 * (int)left[-1] + (int)top[0] + 2) >> 2;
}
// ref_filter_strong's output at index i (0..62) of an array whose ends are a[-1] and a[63]
template <typename A>
__host__ __device__ __forceinline__ int strong_at(const A *a, int i)
{
    return ((63 - i) * (int)a[-1] + (i + 1) * (int)a[63] + 32) >> 6;
}

__host__ __device__ __forceinline__ int clip_pix(int v, int maxv) { return v < 0 ? 0 : v > maxv ? maxv : v; }

__device__ const signed char kAngle[33] = { 32, 26, 21, 17, 13, 9, 5, 2, 0, -2, -5, -9, -13, -17, -21, -26, -32,
                                            -26, -21, -17, -13, -9, -5, -2, 0, 2, 5, 9, 13, 17, 21, 26, 32 };
__device__ const short kInvAngle[15] = { -4096, -1638, -910, -630, -482, -390, -315, -256, -315, -390, -482, -630, -910, -1638, -4096 };

template <typename P>
__device__ __forceinline__ void store4(P *p, int a, int b, int c, int d)
{
    if (((uintptr_t)p % (4 * sizeof(P))) == 0) {
        if (sizeof(P) == 1) *reinterpret_cast<uint32_t *>(p) = (uint32_t)a | (uint32_t)b << 8 | (uint32_t)c << 16 | (uint32_t)d << 24;
        else *reinterpret_cast<uint2 *>(p) = make_uint2((uint32_t)a | (uint32_t)b << 16, (uint32_t)c | (uint32_t)d << 16);
    } else {
        p[0] = (P)a; p[1] = (P)b; p[2] = (P)c; p[3] = (P)d;
    }
}

// Stage 5 for one warp: pred_planar / pred_dc / pred_angular of a size x size block from top / left (index -1 = corner) into dst
// (st samples per row).  R: the warp's ref_tmp scratch.  Every thread of the CTA calls it (it holds a barrier); act = this warp's op
// is live.
template <typename P>
__device__ __forceinline__ void predict(bool act, const int *top, const int *left, int *R, P *dst, long long st, int log2, int mode, bool luma,
                                        int depth, int lane)
{
    const int size = 1 << log2, maxv = (1 << depth) - 1;
    const int angle = act && mode >= 2 ? kAngle[mode - 2] : 0;
    const int last = (size * angle) >> 5;
    const bool tmp = act && mode >= 2 && angle < 0 && last < -1;
    int *ref_tmp = R + size;
    if (tmp) {
        const int *main = mode >= 18 ? top : left, *side = mode >= 18 ? left : top;
        for (int x = lane; x < size + 4; x += 32) ref_tmp[x] = main[x - 1];           // the word copy of x = 0..size step 4
        for (int x = last + lane; x <= -1; x += 32) ref_tmp[x] = side[-1 + ((x * kInvAngle[mode - 11] + 128) >> 8)];
    }
    __syncthreads();
    if (!act) return;
    const int *ref = tmp ? ref_tmp : (mode >= 18 ? top : left) - 1;
    int dc = 0;
    if (mode == 1) {
        dc = size;
        for (int i = 0; i < size; i++) dc += left[i] + top[i];
        dc >>= log2 + 1;
    }
    const int runs = size * size / 4, rpr = size / 4;
    for (int r = lane; r < runs; r += 32) {
        const int y = r / rpr, x0 = (r % rpr) * 4;
        int v[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int x = x0 + k;
            int s;
            if (mode == 0) {
                s = ((size - 1 - x) * left[y] + (x + 1) * top[size] + (size - 1 - y) * top[x] + (y + 1) * left[size] + size) >> (log2 + 1);
            } else if (mode == 1) {
                s = dc;
                if (luma && size < 32) {
                    if (x == 0 && y == 0) s = (left[0] + 2 * dc + top[0] + 2) >> 2;
                    else if (y == 0) s = (top[x] + 3 * dc + 2) >> 2;
                    else if (x == 0) s = (left[y] + 3 * dc + 2) >> 2;
                }
            } else {
                const int u = mode >= 18 ? x : y, w = mode >= 18 ? y : x;     // u along the reference array, w across
                const int idx = ((w + 1) * angle) >> 5, fact = ((w + 1) * angle) & 31;
                s = fact ? ((32 - fact) * ref[u + idx + 1] + fact * ref[u + idx + 2] + 16) >> 5 : ref[u + idx + 1];
                if (luma && size < 32) {
                    if (mode == 26 && x == 0) s = clip_pix(top[0] + ((left[y] - left[-1]) >> 1), maxv);
                    if (mode == 10 && y == 0) s = clip_pix(left[0] + ((top[x] - top[-1]) >> 1), maxv);
                }
            }
            v[k] = s;
        }
        store4(dst + (long long)y * st + x0, v[0], v[1], v[2], v[3]);
    }
}

struct IntraArgs {
    uint8_t *pix;
    long long stride;                            // bytes
    const B200HevcIntraOp *ops;
    long long nops;
    const uint8_t *map;
    long long mstride;
    int W, H, hs, vs, pw, ph, log2_pu, mpw, mph, depth;
};

// intra_pred's IS_INTRA(x, y) for the block at luma (x0, y0): the map entry of luma sample (x0 + x << hs, y0 + y << vs); outside the
// picture's map "not intra"
__device__ __forceinline__ bool is_intra(const IntraArgs &a, int x0, int y0, int x, int y)
{
    const int px = (x0 + x * (1 << a.hs)) >> a.log2_pu, py = (y0 + y * (1 << a.vs)) >> a.log2_pu;
    if (px < 0 || py < 0 || px >= a.mpw || py >= a.mph) return false;
    return __ldg(a.map + (long long)py * a.mstride + px) != 0;
}
__device__ __forceinline__ bool map_intra(const IntraArgs &a, int px, int py)
{
    if (px < 0 || py < 0 || px >= a.mpw || py >= a.mph) return false;
    return __ldg(a.map + (long long)py * a.mstride + px) != 0;
}

// EXTEND: the 4-sample fill of `len` samples (rounded up to 4, as the reference writes)
__device__ __forceinline__ void extend(int *p, int v, int len)
{
    for (int i = 0; i < len; i += 4) p[i] = p[i + 1] = p[i + 2] = p[i + 3] = v;
}

// Stage 2, after the PU checks and the raw fill: the constrained-intra substitution (pred_template.c:234-295), one lane
__device__ void cip_fill(const IntraArgs &a, int *left, int *top, int x0, int y0, int size, int bls, int bl, int l, int ul, int u, int ur)
{
    if (!(bl || l || ul || u || ur)) return;
    int smx = x0 + ((2 * size) << a.hs) < a.W ? 2 * size : (a.W - x0) >> a.hs;
    int smy = y0 + ((2 * size) << a.vs) < a.H ? 2 * size : (a.H - y0) >> a.vs;
    int j = size + (bl ? bls : 0) - 1, i, v;
    if (!ur) smx = x0 + (size << a.hs) < a.W ? size : (a.W - x0) >> a.hs;
    if (!bl) smy = y0 + (size << a.vs) < a.H ? size : (a.H - y0) >> a.vs;
    if (bl || l || ul) {
        while (j > -1 && !is_intra(a, x0, y0, -1, j)) j--;
        if (!is_intra(a, x0, y0, -1, j)) {
            j = 0;
            while (j < smx && !is_intra(a, x0, y0, j, -1)) j++;
            for (i = j; i > -1; i--)                                      // leftward copy over inter samples, down to top[-1]
                if (!is_intra(a, x0, y0, i - 1, -1)) top[i - 1] = top[i];
            left[-1] = top[-1];
        }
    } else {
        j = 0;
        while (j < smx && !is_intra(a, x0, y0, j, -1)) j++;
        if (j > 0) {
            for (i = j; i > 0; i--)
                if (!is_intra(a, x0, y0, i - 1, -1)) top[i - 1] = top[i];
            top[-1] = top[0];
        }
        left[-1] = top[-1];
    }
    left[-1] = top[-1];
    if (bl || l) {                                                       // downward, 4 samples at a time
        v = left[-1];
        for (i = 0; i < smy; i += 4) {
            if (!is_intra(a, x0, y0, -1, i)) left[i] = left[i + 1] = left[i + 2] = left[i + 3] = v;
            else v = left[i + 3];
        }
    }
    if (!l) extend(left, left[-1], size);
    if (!bl) extend(left + size, left[size - 1], size);
    if (x0 != 0) {                                                       // upward, 4 samples at a time
        v = left[smy - 1];
        for (i = smy - 1; i > -1; i -= 4) {
            if (!is_intra(a, x0, y0, -1, i - 3)) left[i - 3] = left[i - 2] = left[i - 1] = left[i] = v;
            else v = left[i - 3];
        }
        if (y0 != 0 && !is_intra(a, x0, y0, -1, -1)) left[-1] = left[0];
    } else {
        extend(left, 0, smy);                                            // x0 == 0: the column becomes the value 0
    }
    top[-1] = left[-1];
    if (y0 != 0) {                                                       // rightward, 4 samples at a time
        v = left[-1];
        for (i = 0; i < smx; i += 4) {
            if (!is_intra(a, x0, y0, i, -1)) top[i] = top[i + 1] = top[i + 2] = top[i + 3] = v;
            else v = top[i + 3];
        }
    }
}

template <typename P>
__global__ void __launch_bounds__(32 * kOpsPerCta) hevc_intra_kernel(IntraArgs a)
{
    extern __shared__ int ipred_smem[];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int *base = ipred_smem + w * kWarpInts;
    int *left = base + kPad + 1, *top = left + kArr, *fleft = top + kArr, *ftop = fleft + kArr, *R = ftop + kArr - kPad - 1;
    const long long o = (long long)blockIdx.x * kOpsPerCta + w;
    B200HevcIntraOp op;
    memset(&op, 0, sizeof(op));
    if (o < a.nops) {
        const uint4 raw = __ldg(reinterpret_cast<const uint4 *>(a.ops + o));
        memcpy(&op, &raw, sizeof(op));
    }
    const int log2 = op.log2_size, mode = op.mode, f = op.flags, size = 1 << (log2 & 7);
    int bl = f & B200_HEVC_INTRA_CAND_BL, l = f & B200_HEVC_INTRA_CAND_L, ul = f & B200_HEVC_INTRA_CAND_UL;
    int u = f & B200_HEVC_INTRA_CAND_U, ur = f & B200_HEVC_INTRA_CAND_UR;
    const bool luma = f & B200_HEVC_INTRA_LUMA;
    bool act = o < a.nops && log2 >= 2 && log2 <= 5 && mode <= 34 && op.x >= 0 && op.y >= 0 && op.x <= a.pw - size && op.y <= a.ph - size &&
               (op.x >= 1 || !(bl || l || ul)) && (op.y >= 1 || !(ul || u || ur));
    const int x = op.x, y = op.y, x0 = x << a.hs, y0 = y << a.vs;
    const int bls = act ? (min(y0 + 2 * (size << a.vs), a.H) - (y0 + (size << a.vs))) >> a.vs : 0;
    const int trs = act ? (min(x0 + 2 * (size << a.hs), a.W) - (x0 + (size << a.hs))) >> a.hs : 0;
    const long long st = a.stride / (long long)sizeof(P);
    P *src = act ? reinterpret_cast<P *>(a.pix + (long long)y * a.stride) + x : nullptr;
    const bool cip = a.map != nullptr;
    if (act && cip) {                                                    // the PU checks that can clear a flag (pred_template.c:165-208)
        int pv = (size << a.vs) >> a.log2_pu, ph = (size << a.hs) >> a.log2_pu;
        const bool ex = (x0 & ((1 << a.log2_pu) - 1)) == 0, ey = (y0 & ((1 << a.log2_pu) - 1)) == 0;
        if (!ph) ph++;
        if (bl && ex) {
            const int xp = (x0 - 1) >> a.log2_pu, yp = (y0 + (size << a.vs)) >> a.log2_pu, m = min(pv, a.mph - yp);
            bl = 0;
            for (int i = 0; i < m; i += 2) bl |= map_intra(a, xp, yp + i);
        }
        if (l && ex) {
            const int xp = (x0 - 1) >> a.log2_pu, yp = y0 >> a.log2_pu, m = min(pv, a.mph - yp);
            l = 0;
            for (int i = 0; i < m; i += 2) l |= map_intra(a, xp, yp + i);
        }
        if (ul) ul = map_intra(a, (x0 - 1) >> a.log2_pu, (y0 - 1) >> a.log2_pu);
        if (u && ey) {
            const int xp = x0 >> a.log2_pu, yp = (y0 - 1) >> a.log2_pu, m = min(ph, a.mpw - xp);
            u = 0;
            for (int i = 0; i < m; i += 2) u |= map_intra(a, xp + i, yp);
        }
        if (ur && ey) {
            const int yp = (y0 - 1) >> a.log2_pu, xp = (x0 + (size << a.hs)) >> a.log2_pu, m = min(ph, a.mpw - xp);
            ur = 0;
            for (int i = 0; i < m; i += 2) ur |= map_intra(a, xp + i, yp);
        }
    }
    // stage 1: the available runs (CIP: over the 128-byte preset)
    if (act) {
        const int preset = sizeof(P) == 1 ? 128 : 0x8080;
        for (int i = lane; i < 2 * size; i += 32) {
            int lv = preset, tv = preset;
            if (i < size ? l : bl) lv = src[(long long)(i < size ? i : size + min(i - size, bls - 1)) * st - 1];
            if (i < size ? u : ur) tv = src[(i < size ? i : size + min(i - size, trs - 1)) - st];
            if (cip || (i < size ? l : bl)) left[i] = lv;
            if (cip || (i < size ? u : ur)) top[i] = tv;
        }
        if (cip)
            for (int i = 2 * size + lane; i < 128; i += 32) left[i] = top[i] = preset;
        if (lane == 0) {
            if (cip) top[-1] = 128;
            if (ul) left[-1] = top[-1] = src[-1 - st];
        }
    }
    __syncthreads();
    if (act && cip && lane == 0) cip_fill(a, left, top, x0, y0, size, bls, bl, l, ul, u, ur);
    __syncthreads();
    // stage 3: the closed-form substitution; runs 0..4 = bottom-left, left, corner, top, top-right in scan order
    if (act) {
        const int av = (bl ? 1 : 0) | (l ? 2 : 0) | (ul ? 4 : 0) | (u ? 8 : 0) | (ur ? 16 : 0);
        const int mid = 1 << (a.depth - 1);
        for (int k = lane; k < 4 * size + 1; k += 32) {
            const int s = k < size ? 0 : k < 2 * size ? 1 : k == 2 * size ? 2 : k <= 3 * size ? 3 : 4;
            if (av >> s & 1) continue;
            int v = mid;
            if (av) {
                const int before = av & ((1 << s) - 1);
                int p = s + 1;                                               // nearest run before, else the first run after
                if (before) for (p = s - 1; !(before >> p & 1); p--) {}
                else while (!(av >> p & 1)) p++;
                const int *srcp = p == 0 ? left + (before ? size : 2 * size - 1) : p == 1 ? left + (before ? 0 : size - 1)
                                : p == 2 ? left - 1 : p == 3 ? top + (before ? size - 1 : 0) : top + (before ? 2 * size - 1 : size);
                v = *srcp;
            }
            int *dstp = k < 2 * size ? left + (2 * size - 1 - k) : k == 2 * size ? left - 1 : top + (k - 2 * size - 1);
            *dstp = v;
        }
    }
    __syncthreads();
    if (act && lane == 0) top[-1] = left[-1];
    __syncthreads();
    // stage 4: the filter decision (pred_template.c:334-359)
    int filt = 0;                                                        // 0 none, 1 3-tap, 2 strong
    if (act && (f & B200_HEVC_INTRA_SMOOTH) && mode != 1 && size != 4) {
        const int thr = log2 == 3 ? 7 : log2 == 4 ? 1 : 0;
        const int d26 = mode - 26 < 0 ? 26 - mode : mode - 26, d10 = mode - 10 < 0 ? 10 - mode : mode - 10;
        if ((d26 < d10 ? d26 : d10) > thr) {
            const int t = 1 << (a.depth - 5);
            const int et = top[-1] + top[63] - 2 * top[31], el = left[-1] + left[63] - 2 * left[31];
            filt = (f & B200_HEVC_INTRA_STRONG) && luma && log2 == 5 && (et < 0 ? -et : et) < t && (el < 0 ? -el : el) < t ? 2 : 1;
        }
    }
    __syncthreads();
    if (filt == 1) {
        const int n = 2 * size;
        for (int i = lane; i < n; i += 32) {
            fleft[i] = filt3(left, i, n);
            ftop[i] = filt3(top, i, n);
        }
        if (lane == 0) fleft[-1] = ftop[-1] = filt3_corner(left, top);
    } else if (filt == 2) {
        for (int i = lane; i < 63; i += 32) {
            ftop[i] = strong_at(top, i);
            left[i] = strong_at(left, i);                                // in place: reads only left[-1] and left[63]
        }
        if (lane == 0) { ftop[-1] = top[-1]; ftop[63] = top[63]; }
    }
    __syncthreads();
    predict<P>(act, filt ? ftop : top, filt == 1 ? fleft : left, R, src, st, log2, mode, luma, a.depth, lane);
}

// the prediction stage alone, for the members: one warp, top / left staged as int arrays of kArr elements (index -1 at kPad)
template <typename P>
__global__ void __launch_bounds__(32) hevc_pred_member_kernel(const int *staged, P *dst, long long st, int log2, int mode, int luma, int depth)
{
    extern __shared__ int ipred_smem[];
    int *left = ipred_smem + kPad + 1, *top = left + kArr, *R = top + kArr;
    for (int i = threadIdx.x; i < 2 * kArr; i += 32) ipred_smem[i] = staged[i];
    __syncthreads();
    predict<P>(true, top, left, R, dst, st, log2, mode, luma != 0, depth, threadIdx.x);
}

bool depth_ok(int d) { return d == 8 || d == 9 || d == 10 || d == 12; }

constexpr long long kChunkOps = 1LL << 24;
constexpr size_t kSmem = (size_t)kOpsPerCta * kWarpInts * sizeof(int);

cudaError_t launch_batch(IntraArgs a, cudaStream_t st)
{
    const long long nops = a.nops;
    const B200HevcIntraOp *ops = a.ops;
    for (long long b = 0; b < nops; b += kChunkOps) {
        a.ops = ops + b;
        a.nops = nops - b < kChunkOps ? nops - b : kChunkOps;
        const unsigned grid = (unsigned)((a.nops + kOpsPerCta - 1) / kOpsPerCta);
        if (a.depth == 8) hevc_intra_kernel<uint8_t><<<grid, 32 * kOpsPerCta, kSmem, st>>>(a);
        else hevc_intra_kernel<uint16_t><<<grid, 32 * kOpsPerCta, kSmem, st>>>(a);
        B200_LAUNCHED();
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

void die(const char *what)
{
    fprintf(stderr, "libb200dsp: hevc intra prediction failed: %s (%s)\n", what, b200_last_error());
    abort();
}

// ---- prediction members (host pointers): top[t0..t1) and left[t0..t1) staged (index -1 = the corner), the block predicted into a
// scratch block and copied back.  `stride` is in samples, as intra_pred passes it (linesize / sizeof(pixel)).
template <int D>
void member_run(uint8_t *dst, ptrdiff_t stride, const uint8_t *top_, const uint8_t *left_, int log2, int mode, int c_idx, int t0, int t1)
{
    typedef typename std::conditional<D == 8, uint8_t, uint16_t>::type P;
    const P *top = reinterpret_cast<const P *>(top_), *left = reinterpret_cast<const P *>(left_);
    const int size = 1 << log2;
    int staged[2 * kArr];
    memset(staged, 0, sizeof(staged));
    for (int i = t0; i < t1; i++) {
        staged[kPad + 1 + i] = left[i];
        staged[kArr + kPad + 1 + i] = top[i];
    }
    B200Device *dev = b200_default_device();
    if (!dev) die("no device");
    if (cudaSetDevice(dev->ordinal) != cudaSuccess) die("cudaSetDevice");
    B200_LOCK_DEVICE(dev);            // scratch + stream are per device: one host-pointer call at a time (released on return)
    const size_t blk = (size_t)size * size * sizeof(P);
    uint8_t *scr = (uint8_t *)b200_scratch(dev, sizeof(staged) + blk);
    if (!scr) die("scratch");
    cudaStream_t st = dev->stream;
    if (cudaMemcpyAsync(scr, staged, sizeof(staged), cudaMemcpyHostToDevice, st) != cudaSuccess) die("h2d edges");
    P *sdst = reinterpret_cast<P *>(scr + sizeof(staged));
    hevc_pred_member_kernel<P><<<1, 32, (2 * kArr + kRef) * sizeof(int), st>>>((const int *)scr, sdst, size, log2, mode, c_idx == 0, D);
    B200_LAUNCHED();
    if (cudaGetLastError() != cudaSuccess) die("launch");
    if (b200_d2h_rows(dst, stride * (ptrdiff_t)sizeof(P), sdst, (size_t)size * sizeof(P), (size_t)size * sizeof(P), (size_t)size, st) != cudaSuccess) die("d2h block");
    if (cudaStreamSynchronize(st) != cudaSuccess) die("sync");
}

template <int D, int L2>
void m_planar(uint8_t *src, const uint8_t *top, const uint8_t *left, ptrdiff_t stride)
{
    member_run<D>(src, stride, top, left, L2, 0, 0, 0, (1 << L2) + 1);
}

template <int D>
void m_dc(uint8_t *src, const uint8_t *top, const uint8_t *left, ptrdiff_t stride, int log2_size, int c_idx)
{
    if (log2_size < 2 || log2_size > 5) { b200_set_error("hevc pred_dc: log2_size %d is not 2..5", log2_size); return; }
    member_run<D>(src, stride, top, left, log2_size, 1, c_idx, 0, 1 << log2_size);
}

template <int D, int L2>
void m_angular(uint8_t *src, const uint8_t *top, const uint8_t *left, ptrdiff_t stride, int c_idx, int mode)
{
    if (mode < 2 || mode > 34) { b200_set_error("hevc pred_angular: mode %d is not 2..34", mode); return; }
    member_run<D>(src, stride, top, left, L2, mode, c_idx, -1, 2 << L2);
}

// ---- filter members: host only, the kernel's filter functions
template <int D>
void m_filter_3tap(uint8_t *filtered_left, uint8_t *filtered_top, const uint8_t *left_, const uint8_t *top_, int size)
{
    typedef typename std::conditional<D == 8, uint8_t, uint16_t>::type P;
    P *fl = reinterpret_cast<P *>(filtered_left), *ft = reinterpret_cast<P *>(filtered_top);
    const P *left = reinterpret_cast<const P *>(left_), *top = reinterpret_cast<const P *>(top_);
    const int n = 2 * size;
    fl[n - 1] = left[n - 1];
    ft[n - 1] = top[n - 1];
    for (int i = n - 2; i >= 0; i--) fl[i] = (P)filt3(left, i, n);
    ft[-1] = fl[-1] = (P)filt3_corner(left, top);
    for (int i = n - 2; i >= 0; i--) ft[i] = (P)filt3(top, i, n);
}

template <int D>
void m_filter_strong(uint8_t *filtered_top, uint8_t *left_, const uint8_t *top_)
{
    typedef typename std::conditional<D == 8, uint8_t, uint16_t>::type P;
    P *ft = reinterpret_cast<P *>(filtered_top), *left = reinterpret_cast<P *>(left_);
    const P *top = reinterpret_cast<const P *>(top_);
    ft[-1] = top[-1];
    ft[63] = top[63];
    for (int i = 0; i < 63; i++) ft[i] = (P)strong_at(top, i);
    for (int i = 0; i < 63; i++) left[i] = (P)strong_at(left, i);
}

template <int D>
void fill(B200HEVCPredContext *h)
{
    h->pred_planar[0] = m_planar<D, 2>;
    h->pred_planar[1] = m_planar<D, 3>;
    h->pred_planar[2] = m_planar<D, 4>;
    h->pred_planar[3] = m_planar<D, 5>;
    h->pred_dc = m_dc<D>;
    h->pred_angular[0] = m_angular<D, 2>;
    h->pred_angular[1] = m_angular<D, 3>;
    h->pred_angular[2] = m_angular<D, 4>;
    h->pred_angular[3] = m_angular<D, 5>;
    for (int k = 0; k < 3; k++) h->ref_filter_3tap[k] = m_filter_3tap<D>;
    h->ref_filter_strong = m_filter_strong<D>;
}

} // namespace

B200_API int b200_hevc_pred_init(B200HEVCPredContext *hpc, int bit_depth)
{
    if (!hpc) return B200_EINVAL;
    if (!depth_ok(bit_depth)) return B200_ENOSYS;
    if (!b200_default_device()) return B200_ENODEV;
    memset(hpc, 0, sizeof(*hpc));                                        // intra_pred[] stays NULL
    switch (bit_depth) {
    case 8:  fill<8>(hpc); break;
    case 9:  fill<9>(hpc); break;
    case 10: fill<10>(hpc); break;
    default: fill<12>(hpc); break;
    }
    return 0;
}

B200_API int b200_hevc_intra_pred_batch_device(B200Device *dev, int bit_depth, uint8_t *pix, ptrdiff_t stride, int width, int height, int hshift,
                                               int vshift, int64_t nops, const B200HevcIntraOp *ops, const uint8_t *intra_map,
                                               ptrdiff_t map_stride, int log2_min_pu_size)
{
    if (!depth_ok(bit_depth)) { b200_set_error("hevc intra batch: bit depth %d is not 8, 9, 10 or 12", bit_depth); return B200_EINVAL; }
    if (nops < 0) { b200_set_error("hevc intra batch: nops %lld < 0", (long long)nops); return B200_EINVAL; }
    if (width < 1 || height < 1) { b200_set_error("hevc intra batch: %dx%d is empty", width, height); return B200_EINVAL; }
    if ((hshift != 0 && hshift != 1) || (vshift != 0 && vshift != 1)) {
        b200_set_error("hevc intra batch: shifts %d, %d are not 0 or 1", hshift, vshift);
        return B200_EINVAL;
    }
    const int bps = bit_depth > 8 ? 2 : 1;
    if (stride < (ptrdiff_t)(width >> hshift) * bps || stride % bps) {
        b200_set_error("hevc intra batch: stride shorter than a plane row or not a whole number of samples");
        return B200_EINVAL;
    }
    if (intra_map && (log2_min_pu_size < 2 || log2_min_pu_size > 6 || map_stride < (width >> log2_min_pu_size))) {
        b200_set_error("hevc intra batch: log2_min_pu_size %d or map_stride %lld does not fit the picture", log2_min_pu_size, (long long)map_stride);
        return B200_EINVAL;
    }
    if (nops == 0) return 0;
    if (!pix || !ops || (uintptr_t)pix % bps || (uintptr_t)ops % 16) {
        b200_set_error("hevc intra batch: NULL pix / ops, pix not aligned to a sample or ops not aligned to 16 bytes");
        return B200_EINVAL;
    }
    if (!dev) dev = b200_default_device();
    if (!dev) return B200_ENODEV;
    B200_CUDA_OK(cudaSetDevice(dev->ordinal));
    IntraArgs a;
    a.pix = pix; a.stride = (long long)stride; a.ops = ops; a.nops = nops;
    a.map = intra_map; a.mstride = (long long)map_stride;
    a.W = width; a.H = height; a.hs = hshift; a.vs = vshift; a.pw = width >> hshift; a.ph = height >> vshift;
    a.log2_pu = intra_map ? log2_min_pu_size : 2;
    a.mpw = width >> a.log2_pu; a.mph = height >> a.log2_pu; a.depth = bit_depth;
    B200_CUDA_OK(launch_batch(a, dev->stream));
    return 0;
}
