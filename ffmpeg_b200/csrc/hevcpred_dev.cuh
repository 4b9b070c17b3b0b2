// hevcpred_dev.cuh — intra_pred (hevc/pred_template.c) for one op on one warp, shared by the batch kernel (hevcpred.cu, whose CTA
// synchronises with __syncthreads) and the picture kernel (hevcintra.cu, one warp per op, __syncwarp): the five stages listed at the
// top of hevcpred.cu, the filters (also used by the host members) and the constrained-intra substitution.  The barrier and the sample
// load are template parameters, so this header builds for the device and, with the stand-in runtime of tests/cuda_emu, for the host.
#pragma once
#include "common.h"

namespace {

constexpr int kPad = 4;                          // elements before index -1 (the CIP up-extension writes down to index -3)
constexpr int kArr = kPad + 1 + 128 + 8;         // one edge array: [-kPad - 1, 136)
constexpr int kRef = 3 * 32 + 8;                 // ref_tmp of pred_angular: [-size, size + 4)
constexpr int kWarpInts = 4 * kArr + kRef;       // left, top, filtered left, filtered top, ref_tmp

// ---- the filters, shared by the kernels and the host members (A = int for shared arrays, the sample type on the host)
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
// (st samples per row).  R: the warp's ref_tmp scratch.  Every thread of the barrier's group calls it (it holds one bar()); act = this
// warp's op is live.
template <typename P, typename Bar>
__device__ __forceinline__ void predict(bool act, const int *top, const int *left, int *R, P *dst, long long st, int log2, int mode, bool luma,
                                        int depth, int lane, Bar bar)
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
    bar();
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

// one component plane as intra_pred sees it: the luma picture size, the component's shifts and size, the intra map (NULL: no
// constrained intra prediction) with its min-PU geometry, the depth
struct PredPlane {
    const uint8_t *map;
    long long mstride;
    int W, H, hs, vs, pw, ph, log2_pu, mpw, mph, depth;
};

// intra_pred's IS_INTRA(x, y) for the block at luma (x0, y0): the map entry of luma sample (x0 + x << hs, y0 + y << vs); outside the
// picture's map "not intra"
__device__ __forceinline__ bool is_intra(const PredPlane &a, int x0, int y0, int x, int y)
{
    const int px = (x0 + x * (1 << a.hs)) >> a.log2_pu, py = (y0 + y * (1 << a.vs)) >> a.log2_pu;
    if (px < 0 || py < 0 || px >= a.mpw || py >= a.mph) return false;
    return __ldg(a.map + (long long)py * a.mstride + px) != 0;
}
__device__ __forceinline__ bool map_intra(const PredPlane &a, int px, int py)
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
__device__ void cip_fill(const PredPlane &a, int *left, int *top, int x0, int y0, int size, int bls, int bl, int l, int ul, int u, int ur)
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

// the checks that make an op of the batch entry write nothing: size, mode, the block inside the plane, the flagged neighbours too
__device__ __forceinline__ bool pred_op_ok(const PredPlane &a, int x, int y, int log2, int mode, int f)
{
    const int size = 1 << (log2 & 7);
    return log2 >= 2 && log2 <= 5 && mode <= 34 && x >= 0 && y >= 0 && x <= a.pw - size && y <= a.ph - size &&
           (x >= 1 || !(f & (B200_HEVC_INTRA_CAND_BL | B200_HEVC_INTRA_CAND_L | B200_HEVC_INTRA_CAND_UL))) &&
           (y >= 1 || !(f & (B200_HEVC_INTRA_CAND_UL | B200_HEVC_INTRA_CAND_U | B200_HEVC_INTRA_CAND_UR)));
}

// intra_pred of one op by one warp (lane 0..31), stages 1-5, into the plane at src (the block's top-left, st samples per row).
// base: the warp's kWarpInts ints of shared memory.  act: the op is live (pred_op_ok); every thread of the barrier's group calls
// this, live or not, as it holds bar() calls.  ld(p): how a neighbour sample of the plane is read.
template <typename P, typename Bar, typename Ld>
__device__ __forceinline__ void intra_pred_op(bool act, const PredPlane &a, int x, int y, int log2, int mode, int f, P *src, long long st,
                                              int *base, int lane, Bar bar, Ld ld)
{
    int *left = base + kPad + 1, *top = left + kArr, *fleft = top + kArr, *ftop = fleft + kArr, *R = ftop + kArr - kPad - 1;
    const int size = 1 << (log2 & 7);
    int bl = f & B200_HEVC_INTRA_CAND_BL, l = f & B200_HEVC_INTRA_CAND_L, ul = f & B200_HEVC_INTRA_CAND_UL;
    int u = f & B200_HEVC_INTRA_CAND_U, ur = f & B200_HEVC_INTRA_CAND_UR;
    const bool luma = f & B200_HEVC_INTRA_LUMA;
    const int x0 = x << a.hs, y0 = y << a.vs;
    const int bls = act ? (min(y0 + 2 * (size << a.vs), a.H) - (y0 + (size << a.vs))) >> a.vs : 0;
    const int trs = act ? (min(x0 + 2 * (size << a.hs), a.W) - (x0 + (size << a.hs))) >> a.hs : 0;
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
            if (i < size ? l : bl) lv = ld(src + (long long)(i < size ? i : size + min(i - size, bls - 1)) * st - 1);
            if (i < size ? u : ur) tv = ld(src + (i < size ? i : size + min(i - size, trs - 1)) - st);
            if (cip || (i < size ? l : bl)) left[i] = lv;
            if (cip || (i < size ? u : ur)) top[i] = tv;
        }
        if (cip)
            for (int i = 2 * size + lane; i < 128; i += 32) left[i] = top[i] = preset;
        if (lane == 0) {
            if (cip) top[-1] = 128;
            if (ul) left[-1] = top[-1] = ld(src - 1 - st);
        }
    }
    bar();
    if (act && cip && lane == 0) cip_fill(a, left, top, x0, y0, size, bls, bl, l, ul, u, ur);
    bar();
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
    bar();
    if (act && lane == 0) top[-1] = left[-1];
    bar();
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
    bar();
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
    bar();
    predict<P>(act, filt ? ftop : top, filt == 1 ? fleft : left, R, src, st, log2, mode, luma, a.depth, lane, bar);
}

} // namespace
