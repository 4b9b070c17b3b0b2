// h264pred.cu — libavcodec's H.264 intra prediction on sm_90a: H264PredContext (libavcodec/h264pred.h:94-114) as
// ff_h264_pred_init(h, AV_CODEC_ID_H264, bit_depth, chroma_format_idc) fills it for 8, 9, 10, 12 and 14 bit samples
// (libavcodec/h264pred.c:437-539), and two batched device entries.
//
// Reference semantics reproduced bit for bit (checker: oracle/h264pred_oracle.c), libavcodec/h264pred_template.c:
//   :34-301     pred4x4 (nine directional modes, LEFT_DC, TOP_DC, DC_128)
//   :303-461    pred16x16 (DC, V, H, PLANE, LEFT_DC, TOP_DC, DC_128)
//   :463-820    pred8x8 / pred8x16 (chroma) including the four mad_cow compositions (:694-743)
//   :822-1101   pred8x8l with the has_topleft / has_topright edge filter (PREDICT_8x8_LOAD_*, :822-851)
//   :1103-1330  the lossless add forms: no clipping (`pixel v; v += block[]` wraps modulo 2^8 / 2^16), coefficients cleared; the
//               8x8 / 8x16 / 16x16 forms are 4x4 forms applied in table order, so each sub-block predicts from its neighbour's
//               already added samples, and pred8x16_*_add take block_offset[i + 4] for i = 4..7.
//
// Prediction kernel: 16 lanes (one per output row) per op, 8 ops per 128-thread CTA.  The lanes of an op load the neighbours the
// reference function reads (and only those: a block on the picture edge may have no row above it) into shared memory, once per op;
// pred8x8l's edge filter is computed once per op by the same lanes, then every lane computes its row from the shared edge with the
// spec's closed forms (zVR / zHD / zHU, ITU-T H.264 8.3.1.2 / 8.3.2.2) and stores it as 4-sample words where the address allows.
// The plane gradients (a handful of shared loads) are recomputed by each lane rather than broadcast; they are not the cost.
// Add kernel: one lane owns a column (vertical) or a row (horizontal) and walks the op's 4x4 sub-blocks in scan order, which gives
// the reference's sequential result for the chained sub-blocks.  A vertical owner stores one sample per row, i.e. one 32-byte
// sector per row per lane group; the coefficients it reads it also clears.
#include "common.h"
#include <cmath>
#include <cstring>
#include <type_traits>

namespace {

enum { P4 = 0, P8L = 1, P8 = 2, P816 = 3, P16 = 4 };                   // b200_h264_pred_batch_device tables
enum { A4 = 0, A8L = 1, A8LF = 2, A8 = 3, A816 = 4, A16 = 5 };           // b200_h264_pred_add_batch_device tables
enum { NT = 1, NL = 2, NC = 4, NTR = 8 };                                // neighbours a mode reads: top row, left column, corner, top-right

// whether kind names a member ff_h264_pred_init fills for H.264 (h264pred.c:447-538)
__host__ __device__ __forceinline__ bool pred_kind_ok(int k)
{
    const int t = k >> 4, m = k & 15;
    return t <= P8L ? m <= 11 : t <= P816 ? m <= 10 : t == P16 ? m <= 6 : false;
}
__host__ __device__ __forceinline__ bool add_kind_ok(int k)
{
    const int t = k >> 4, m = k & 15;
    return t <= A8LF ? m <= 1 : t <= A16 ? (m == 1 || m == 2) : false;
}
__host__ __device__ __forceinline__ int pred_w(int t) { return t == P4 ? 4 : t == P16 ? 16 : 8; }
__host__ __device__ __forceinline__ int pred_h(int t) { return t == P4 ? 4 : t >= P816 ? 16 : 8; }
// the neighbours (NT / NL / NC / NTR) the reference function of (table, mode) reads; for pred8x8l the corner and the first top-right
// sample are also read by the edge filter when has_topleft / has_topright say so (that is decided by the caller)
__host__ __device__ __forceinline__ int pred_needs(int t, int m)
{
    if (t == P4 || t == P8L) {
        switch (m) {
        case 0: case 10: return NT;
        case 1: case 8: case 9: return NL;
        case 2: return NT | NL;
        case 3: case 7: return NT | NTR;
        case 4: case 5: case 6: return NT | NL | NC;
        default: return 0;
        }
    }
    // pred8x8 / pred8x16 / pred16x16: 0 DC, 1 HOR, 2 VERT, 3 PLANE, 4 LEFT_DC, 5 TOP_DC, 6 DC_128, 7-10 the mad_cow compositions
    switch (m) {
    case 0: case 7: case 8: return NT | NL;
    case 1: case 4: case 9: case 10: return NL;
    case 2: case 5: return NT;
    case 3: return NT | NL | NC;
    default: return 0;
    }
}
// index k of the 4x4 sub-block at [bx, by] (in 4x4 units) of the 8x8 / 8x16 / 16x16 add forms: h264_slice.c:554-563 puts block k at scan8[k]
__host__ __device__ __forceinline__ int sub_index(int t, int bx, int by)
{
    return t == A16 ? (by >> 1) * 8 + (bx >> 1) * 4 + (by & 1) * 2 + (bx & 1) : by * 2 + bx;
}

__device__ __forceinline__ int f3(int a, int b, int c) { return (a + 2 * b + c + 2) >> 2; }
__device__ __forceinline__ int f2(int a, int b) { return (a + b + 1) >> 1; }

// one sample of the directional modes 3..8 of pred4x4 (N = 4) and pred8x8l (N = 8): T[i] = top sample i (T[-1] the corner), L[i] = left
// sample i (L[-1] the corner); for pred8x8l both are the filtered edge
__device__ __forceinline__ int dir_sample(int m, int N, int x, int y, const int *T, const int *L)
{
    switch (m) {
    case 3:                                                              // DIAG_DOWN_LEFT
        return (x == N - 1 && y == N - 1) ? (T[2 * N - 2] + 3 * T[2 * N - 1] + 2) >> 2 : f3(T[x + y], T[x + y + 1], T[x + y + 2]);
    case 4:                                                              // DIAG_DOWN_RIGHT
        return x > y ? f3(T[x - y - 2], T[x - y - 1], T[x - y]) : x < y ? f3(L[y - x - 2], L[y - x - 1], L[y - x]) : f3(T[0], T[-1], L[0]);
    case 5: {                                                            // VERT_RIGHT, zVR = 2x - y
        const int z = 2 * x - y, i = x - (y >> 1);
        if (z >= 0) return (z & 1) ? f3(T[i - 2], T[i - 1], T[i]) : f2(T[i - 1], T[i]);
        if (z == -1) return f3(L[0], L[-1], T[0]);
        return f3(L[y - 2 * x - 1], L[y - 2 * x - 2], L[y - 2 * x - 3]);
    }
    case 6: {                                                            // HOR_DOWN, zHD = 2y - x
        const int z = 2 * y - x, i = y - (x >> 1);
        if (z >= 0) return (z & 1) ? f3(L[i - 2], L[i - 1], L[i]) : f2(L[i - 1], L[i]);
        if (z == -1) return f3(L[0], L[-1], T[0]);
        return f3(T[x - 2 * y - 1], T[x - 2 * y - 2], T[x - 2 * y - 3]);
    }
    case 7: {                                                            // VERT_LEFT
        const int i = x + (y >> 1);
        return (y & 1) ? f3(T[i], T[i + 1], T[i + 2]) : f2(T[i], T[i + 1]);
    }
    default: {                                                           // HOR_UP, zHU = x + 2y
        const int z = x + 2 * y, i = y + (x >> 1);
        if (z < 2 * N - 3) return (z & 1) ? f3(L[i], L[i + 1], L[i + 2]) : f2(L[i], L[i + 1]);
        if (z == 2 * N - 3) return (L[N - 2] + 3 * L[N - 1] + 2) >> 2;
        return L[N - 1];
    }
    }
}

template <typename P>
__device__ __forceinline__ void store4(P *p, int a, int b, int c, int d)
{
    if (sizeof(P) == 1 && !((uintptr_t)p & 3)) {
        *reinterpret_cast<uint32_t *>(p) = (uint32_t)a | (uint32_t)b << 8 | (uint32_t)c << 16 | (uint32_t)d << 24;
    } else if (sizeof(P) == 2 && !((uintptr_t)p & 7)) {
        uint2 w;
        w.x = (uint32_t)a | (uint32_t)b << 16;
        w.y = (uint32_t)c | (uint32_t)d << 16;
        *reinterpret_cast<uint2 *>(p) = w;
    } else {
        p[0] = (P)a; p[1] = (P)b; p[2] = (P)c; p[3] = (P)d;
    }
}

constexpr int kOpsPerCta = 8;
constexpr int kEdge = 18;                    // per op and edge array: index 0 = the corner, 1 + i = sample i (top: i < 17, left: i < 16)

// op o of this launch: kinds[o], flags[o], top-left sample at base + off[o] (bytes); stride in bytes.  16 lanes per op.
template <typename P>
__global__ void __launch_bounds__(128)
h264_pred_kernel(long long nops, const uint8_t *kinds, const uint8_t *flags, uint8_t *base, const long long *off, long long stride, int depth)
{
    extern __shared__ int pred_smem[];                                  // [kOpsPerCta][4][kEdge]: raw top, raw left, filtered top, filtered left
    const int g = threadIdx.x >> 4, lane = threadIdx.x & 15;
    const long long o = (long long)blockIdx.x * kOpsPerCta + g;
    int *RT = pred_smem + g * 4 * kEdge, *RL = RT + kEdge, *FT = RL + kEdge, *FL = FT + kEdge;
    const int kind = o < nops ? kinds[o] : 0xff;
    const bool act = pred_kind_ok(kind);
    const int t = kind >> 4, m = kind & 15;
    const int W = pred_w(t), H = pred_h(t);
    const int fl = act ? flags[o] : 0;
    const bool tl = fl & 1, tr = (fl & 2) != 0;
    const long long st = stride / (long long)sizeof(P);
    P *src = act ? reinterpret_cast<P *>(base + off[o]) : nullptr;
    const int need = act ? pred_needs(t, m) : 0;
    if (need) {
        // raw neighbours: exactly the samples the reference function reads
        const bool corner = (need & NC) || (t == P8L && tl && (need & (NT | NL)));
        int ntr = 0;                                                     // top-right samples after the W top ones
        if (t == P4 && (need & NTR)) ntr = 4;
        if (t == P8L && tr) ntr = (need & NTR) ? 8 : (need & NT) ? 1 : 0;
        if ((need & NT) && lane < W) RT[1 + lane] = src[lane - st];
        if (lane < ntr) RT[1 + W + lane] = (t == P4 && !tr) ? src[3 - st] : src[W + lane - st];
        if ((need & NL) && lane < H) RL[1 + lane] = src[lane * st - 1];
        if (lane == 0 && corner) RT[0] = RL[0] = src[-1 - st];
    }
    __syncthreads();
    if (t == P8L && need) {                                              // PREDICT_8x8_LOAD_{TOP,TOPRIGHT,LEFT,TOPLEFT}, h264pred_template.c:822-851
        const int *T = RT + 1, *L = RL + 1;
        if (need & NT) {
            int v;
            if (lane == 0) v = ((tl ? T[-1] : T[0]) + 2 * T[0] + T[1] + 2) >> 2;
            else if (lane < 7) v = f3(T[lane - 1], T[lane], T[lane + 1]);
            else if (lane == 7) v = ((tr ? T[8] : T[7]) + 2 * T[7] + T[6] + 2) >> 2;
            else if (!tr) v = T[7];
            else if (lane < 15) v = f3(T[lane - 1], T[lane], T[lane + 1]);
            else v = (T[14] + 3 * T[15] + 2) >> 2;
            if (lane < 8 || (need & NTR)) FT[1 + lane] = v;
        }
        if ((need & NL) && lane < 8) {
            int v;
            if (lane == 0) v = ((tl ? L[-1] : L[0]) + 2 * L[0] + L[1] + 2) >> 2;
            else if (lane < 7) v = f3(L[lane - 1], L[lane], L[lane + 1]);
            else v = (L[6] + 3 * L[7] + 2) >> 2;
            FL[1 + lane] = v;
        }
        if (lane == 0 && (need & NC)) FT[0] = FL[0] = (L[0] + 2 * L[-1] + T[0] + 2) >> 2;
    }
    __syncthreads();
    if (!act || lane >= H) return;
    const int *T = (t == P8L ? FT : RT) + 1, *L = (t == P8L ? FL : RL) + 1;
    const int y = lane, maxv = (1 << depth) - 1, mid = 1 << (depth - 1);
    P *row = src + y * st;
    if (t == P4 || t == P8L) {
        if (m >= 3 && m <= 8) {
            for (int x = 0; x < W; x += 4)
                store4(row + x, dir_sample(m, W, x, y, T, L), dir_sample(m, W, x + 1, y, T, L), dir_sample(m, W, x + 2, y, T, L),
                       dir_sample(m, W, x + 3, y, T, L));
            return;
        }
        int sT = 0, sL = 0;
        for (int i = 0; i < W; i++) {
            if (need & NT) sT += T[i];
            if (need & NL) sL += L[i];
        }
        const int sh = W == 4 ? 2 : 3;
        for (int x = 0; x < W; x += 4) {
            int v0, v1, v2, v3;
            if (m == 0) { v0 = T[x]; v1 = T[x + 1]; v2 = T[x + 2]; v3 = T[x + 3]; }
            else {
                const int v = m == 1 ? L[y] : m == 2 ? (sT + sL + W) >> (sh + 1) : m == 9 ? (sL + (W >> 1)) >> sh
                            : m == 10 ? (sT + (W >> 1)) >> sh : mid;
                v0 = v1 = v2 = v3 = v;
            }
            store4(row + x, v0, v1, v2, v3);
        }
        return;
    }
    if (m == 3) {                                                        // PLANE: H, V and a as the reference (template :410-456, :746-820)
        int Hs = 0, Vs = 0, a;
        if (t == P16) {
            for (int k = 1; k <= 8; k++) { Hs += k * (T[7 + k] - T[7 - k]); Vs += k * (L[7 + k] - L[7 - k]); }
            Hs = (5 * Hs + 32) >> 6; Vs = (5 * Vs + 32) >> 6;
            a = 16 * (L[15] + T[15] + 1) - 7 * (Vs + Hs);
        } else {
            for (int k = 1; k <= 4; k++) Hs += k * (T[3 + k] - T[3 - k]);
            Hs = (17 * Hs + 16) >> 5;
            if (t == P8) {
                for (int k = 1; k <= 4; k++) Vs += k * (L[3 + k] - L[3 - k]);
                Vs = (17 * Vs + 16) >> 5;
                a = 16 * (L[7] + T[7] + 1) - 3 * (Vs + Hs);
            } else {
                for (int k = 1; k <= 8; k++) Vs += k * (L[7 + k] - L[7 - k]);
                Vs = (5 * Vs + 32) >> 6;
                a = 16 * (L[15] + T[7] + 1) - 7 * Vs - 3 * Hs;
            }
        }
        const int b = a + y * Vs;
        for (int x = 0; x < W; x += 4)
            store4(row + x, min(max((b + x * Hs) >> 5, 0), maxv), min(max((b + (x + 1) * Hs) >> 5, 0), maxv),
                   min(max((b + (x + 2) * Hs) >> 5, 0), maxv), min(max((b + (x + 3) * Hs) >> 5, 0), maxv));
        return;
    }
    if (t == P16) {
        int sT = 0, sL = 0;
        for (int i = 0; i < 16; i++) {
            if (need & NT) sT += T[i];
            if (need & NL) sL += L[i];
        }
        const int v = m == 0 ? (sT + sL + 16) >> 5 : m == 1 ? L[y] : m == 4 ? (sL + 8) >> 4 : m == 5 ? (sT + 8) >> 4 : mid;
        for (int x = 0; x < 16; x += 4) {
            if (m == 2) store4(row + x, T[x], T[x + 1], T[x + 2], T[x + 3]);
            else store4(row + x, v, v, v, v);
        }
        return;
    }
    // pred8x8 / pred8x16: the DC family works on 4x4 quadrants (template :541-744); band = the 4-row band of this lane
    const int band = y >> 2;
    const int t03 = (need & NT) ? T[0] + T[1] + T[2] + T[3] : 0, t47 = (need & NT) ? T[4] + T[5] + T[6] + T[7] : 0;
    const int lb = (need & NL) ? L[4 * band] + L[4 * band + 1] + L[4 * band + 2] + L[4 * band + 3] : 0;
    const int l03 = (need & NL) ? L[0] + L[1] + L[2] + L[3] : 0;
    int left, right;                                                     // the values of x < 4 and x >= 4 on this row
    switch (m) {
    case 0: case 8:                                                      // DC; 0lt = DC, then pred4x4_top_dc on the top-left 4x4
        left = band == 0 ? (t03 + l03 + 4) >> 3 : (lb + 2) >> 2;
        right = band == 0 ? (t47 + 2) >> 2 : (t47 + lb + 4) >> 3;
        if (m == 8 && band == 0) left = (t03 + 2) >> 2;
        break;
    case 1: left = right = L[y]; break;
    case 4: case 9: case 10:                                             // LEFT_DC; l00 / 0l0 = LEFT_DC, then DC_128 on rows 4-7 / 0-3
        left = right = (lb + 2) >> 2;
        if ((m == 9 && band == 1) || (m == 10 && band == 0)) left = right = mid;
        break;
    case 5: case 7:                                                      // TOP_DC; l0t = TOP_DC, then pred4x4_dc on the top-left 4x4
        left = (t03 + 2) >> 2; right = (t47 + 2) >> 2;
        if (m == 7 && band == 0) left = (t03 + l03 + 4) >> 3;
        break;
    case 6: left = right = mid; break;
    default:                                                             // 2: VERT
        store4(row, T[0], T[1], T[2], T[3]);
        store4(row + 4, T[4], T[5], T[6], T[7]);
        return;
    }
    store4(row, left, left, left, left);
    store4(row + 4, right, right, right, right);
}

// add op o: kinds[o], flags[o], top-left sample at base + off[o] (bytes), coefficients at coef + coef_off[o] (elements).  16 lanes per op:
// lane = the column (vertical) or row (horizontal) it owns.
template <typename P, typename C>
__global__ void __launch_bounds__(128)
h264_pred_add_kernel(long long nops, const uint8_t *kinds, const uint8_t *flags, uint8_t *base, const long long *off, long long stride,
                     C *coef, const long long *coef_off)
{
    const long long o = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 4;
    const int lane = threadIdx.x & 15;
    if (o >= nops) return;
    const int kind = kinds[o];
    if (!add_kind_ok(kind)) return;
    const int t = kind >> 4, m = kind & 15;
    const int W = t == A4 ? 4 : t == A16 ? 16 : 8, H = t == A4 ? 4 : t >= A816 ? 16 : 8;
    const bool vert = t <= A8LF ? m == 0 : m == 2;
    if (lane >= (vert ? W : H)) return;
    const long long st = stride / (long long)sizeof(P);
    P *src = reinterpret_cast<P *>(base + off[o]);
    C *cf = coef + coef_off[o];
    if (t <= A8LF) {                                                     // one N x N block, coefficients row-major
        const int N = W;
        unsigned v;
        if (t == A8LF) {                                                 // start from the filtered edge (template :1103-1173)
            const int fl = flags[o];
            const bool tl = fl & 1, tr = (fl & 2) != 0;
            const int i = lane;
            if (vert) {
                const P *T = src - st;
                v = i == 0 ? ((tl ? T[-1] : T[0]) + 2 * T[0] + T[1] + 2) >> 2
                  : i == 7 ? ((tr ? T[8] : T[7]) + 2 * T[7] + T[6] + 2) >> 2 : (unsigned)f3(T[i - 1], T[i], T[i + 1]);
            } else {
                const P *L = src - 1;
                v = i == 0 ? ((tl ? L[-st] : L[0]) + 2 * L[0] + L[st] + 2) >> 2
                  : i == 7 ? (L[6 * st] + 3 * L[7 * st] + 2) >> 2 : (unsigned)f3(L[(i - 1) * st], L[i * st], L[(i + 1) * st]);
            }
        } else {
            v = vert ? src[lane - st] : src[lane * st - 1];
        }
        for (int k = 0; k < N; k++) {
            const int x = vert ? lane : k, y = vert ? k : lane;
            v = (P)(v + (unsigned)cf[y * N + x]);
            src[y * st + x] = (P)v;
            cf[y * N + x] = 0;
        }
        return;
    }
    // 4x4 sub-blocks in scan order: the owner of a column walks them top to bottom, the owner of a row left to right
    unsigned v = vert ? src[lane - st] : src[lane * st - 1];
    const int nb = (vert ? H : W) >> 2;
    for (int b = 0; b < nb; b++) {
        const int bx = vert ? lane >> 2 : b, by = vert ? b : lane >> 2;
        C *sb = cf + 16 * sub_index(t, bx, by);
        for (int k = 0; k < 4; k++) {
            const int x = vert ? lane : 4 * b + k, y = vert ? 4 * b + k : lane;
            const int ci = (y & 3) * 4 + (x & 3);
            v = (P)(v + (unsigned)sb[ci]);
            src[y * st + x] = (P)v;
            sb[ci] = 0;
        }
    }
}

// drop-in pred8x8_add / pred16x16_add: the reference's loop over an arbitrary block_offset table, one thread (a host-pointer call is
// latency-bound whatever it does).  offs[k] = byte offset of sub-block k in the window, coefficients of sub-block k at coef + 16 k.
template <typename P, typename C>
__global__ void h264_pred_add_table_kernel(uint8_t *base, const long long *offs, int nsub, int vert, long long stride, C *coef)
{
    if (threadIdx.x || blockIdx.x) return;
    const long long st = stride / (long long)sizeof(P);
    for (int k = 0; k < nsub; k++) {
        P *p = reinterpret_cast<P *>(base + offs[k]);
        C *b = coef + 16 * k;
        for (int i = 0; i < 4; i++) {
            unsigned v = vert ? p[i - st] : p[i * st - 1];
            for (int j = 0; j < 4; j++) {
                const int x = vert ? i : j, y = vert ? j : i;
                v = (P)(v + (unsigned)b[y * 4 + x]);
                p[y * st + x] = (P)v;
            }
        }
        for (int i = 0; i < 16; i++) b[i] = 0;
    }
}

constexpr long long kChunkOps = 1LL << 24;                               // ops per launch: 2^21 CTAs of 8 ops

bool depth_ok(int d) { return d == 8 || d == 9 || d == 10 || d == 12 || d == 14; }

cudaError_t launch_pred(int depth, long long nops, const uint8_t *kinds, const uint8_t *flags, uint8_t *pix, const long long *off, long long stride,
                        cudaStream_t st)
{
    const size_t smem = kOpsPerCta * 4 * kEdge * sizeof(int);
    for (long long b = 0; b < nops; b += kChunkOps) {
        const long long n = nops - b < kChunkOps ? nops - b : kChunkOps;
        const unsigned grid = (unsigned)((n + kOpsPerCta - 1) / kOpsPerCta);
        if (depth == 8) h264_pred_kernel<uint8_t><<<grid, 128, smem, st>>>(n, kinds + b, flags + b, pix, off + b, stride, depth);
        else h264_pred_kernel<uint16_t><<<grid, 128, smem, st>>>(n, kinds + b, flags + b, pix, off + b, stride, depth);
        B200_LAUNCHED();
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

cudaError_t launch_add(int depth, long long nops, const uint8_t *kinds, const uint8_t *flags, uint8_t *pix, const long long *off, long long stride,
                       void *coef, const long long *coef_off, cudaStream_t st)
{
    for (long long b = 0; b < nops; b += kChunkOps) {
        const long long n = nops - b < kChunkOps ? nops - b : kChunkOps;
        const unsigned grid = (unsigned)((n * 16 + 127) / 128);
        if (depth == 8)
            h264_pred_add_kernel<uint8_t, int16_t><<<grid, 128, 0, st>>>(n, kinds + b, flags + b, pix, off + b, stride, (int16_t *)coef, coef_off + b);
        else
            h264_pred_add_kernel<uint16_t, int32_t><<<grid, 128, 0, st>>>(n, kinds + b, flags + b, pix, off + b, stride, (int32_t *)coef, coef_off + b);
        B200_LAUNCHED();
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// ---- drop-in members (host pointers).  The window on the device: row 0 = the picture row above the block, rows 1.. the block; block
// column 0 at byte 16 of a row (the left neighbour just before it, the top-right samples after it).
constexpr size_t kPitch = 64, kX0 = 16, kRows = 17;
constexpr size_t kMeta = kPitch * kRows;                                 // kinds, flags, offsets, coefficients follow the window
constexpr const char *kFeature = "h264 intra prediction";

// copy the neighbours `need` names (NT: W top samples, + ntr top-right ones; NL: H left; NC: the corner) from the host picture
template <int BPS>
void h2d_neighbours(const B200HostCall &call, const uint8_t *src, ptrdiff_t stride, int need, int W, int H, int ntr, const uint8_t *topright)
{
    uint8_t *win = call.scratch + kPitch + kX0;                          // the block's top-left sample in the window
    cudaStream_t st = call.stream;
    if (need & NT) call.check(cudaMemcpyAsync(win - kPitch, src - stride, (size_t)W * BPS, cudaMemcpyHostToDevice, st), "h2d top");
    if (ntr)
        call.check(cudaMemcpyAsync(win - kPitch + W * BPS, topright ? topright : src - stride + W * BPS, (size_t)ntr * BPS, cudaMemcpyHostToDevice, st),
                   "h2d top-right");
    if (need & NL) call.check(b200_h2d_rows(win - BPS, kPitch, src - BPS, stride, BPS, (size_t)H, st), "h2d left");
    if (need & NC) call.check(cudaMemcpyAsync(win - kPitch - BPS, src - stride - BPS, BPS, cudaMemcpyHostToDevice, st), "h2d corner");
}

template <int DEPTH>
void pred_host(int t, int m, int fl, uint8_t *src, ptrdiff_t stride, const uint8_t *topright)
{
    constexpr int BPS = DEPTH > 8 ? 2 : 1;
    B200HostCall call(kFeature, nullptr, kMeta + 256);
    const int W = pred_w(t), H = pred_h(t), need = pred_needs(t, m);
    int ntr = 0, nd = need;
    if (t == P4 && (need & NTR)) ntr = 4;                                // from `topright`, wherever it points (h264_mb.c:676-691)
    if (t == P8L) {
        if ((fl & 2) && (need & NT)) ntr = (need & NTR) ? 8 : 1;
        if ((fl & 1) && (need & (NT | NL))) nd |= NC;
    }
    h2d_neighbours<BPS>(call, src, stride, nd, W, H, ntr, t == P4 ? topright : nullptr);
    uint8_t *meta = call.scratch + kMeta;
    struct { long long off; uint8_t kind, flags, pad[6]; } h;
    h.off = (long long)(kPitch + kX0);
    h.kind = (uint8_t)(t << 4 | m);
    h.flags = (uint8_t)(t == P4 ? (ntr ? 2 : 0) : fl);                   // pred4x4: the four samples are in the window's top row
    memset(h.pad, 0, sizeof(h.pad));
    call.check(cudaMemcpyAsync(meta, &h, sizeof(h), cudaMemcpyHostToDevice, call.stream), "h2d meta");
    call.check(launch_pred(DEPTH, 1, meta + 8, meta + 9, call.scratch, (const long long *)meta, (long long)kPitch, call.stream), "launch");
    call.check(b200_d2h_rows(src, stride, call.scratch + kPitch + kX0, kPitch, (size_t)W * BPS, (size_t)H, call.stream), "d2h");
    call.sync();
}

// pred4x4_add / pred8x8l_add / pred8x8l_filter_add through the device: the edge the function starts from, the coefficients, and back
template <int DEPTH>
void add_host(int t, int m, int fl, uint8_t *pix, int16_t *block, ptrdiff_t stride)
{
    constexpr int BPS = DEPTH > 8 ? 2 : 1;
    using C = typename std::conditional<(DEPTH > 8), int32_t, int16_t>::type;
    const int N = t == A4 ? 4 : 8;
    const size_t cbytes = (size_t)N * N * sizeof(C);
    B200HostCall call(kFeature, nullptr, kMeta + 256 + cbytes);
    const bool vert = m == 0;
    int need = vert ? NT : NL, ntr = 0;
    if (t == A8LF && (fl & 1)) need |= NC;                               // PREDICT_8x8_LOAD_TOP / _LEFT read the corner when has_topleft
    if (t == A8LF && (fl & 2) && vert) ntr = 1;                          // and SRC(8, -1) when has_topright
    h2d_neighbours<BPS>(call, pix, stride, need, N, N, ntr, nullptr);
    uint8_t *meta = call.scratch + kMeta, *dcoef = meta + 256;
    struct { long long off, coff; uint8_t kind, flags, pad[6]; } h;
    h.off = (long long)(kPitch + kX0);
    h.coff = 0;
    h.kind = (uint8_t)(t << 4 | m);
    h.flags = (uint8_t)fl;
    memset(h.pad, 0, sizeof(h.pad));
    cudaStream_t st = call.stream;
    call.check(cudaMemcpyAsync(meta, &h, sizeof(h), cudaMemcpyHostToDevice, st), "h2d meta");
    call.check(cudaMemcpyAsync(dcoef, block, cbytes, cudaMemcpyHostToDevice, st), "h2d coefficients");
    call.check(launch_add(DEPTH, 1, meta + 16, meta + 17, call.scratch, (const long long *)meta, (long long)kPitch, dcoef, (const long long *)(meta + 8), st),
               "launch");
    call.check(b200_d2h_rows(pix, stride, call.scratch + kPitch + kX0, kPitch, (size_t)N * BPS, (size_t)N, st), "d2h");
    call.check(cudaMemcpyAsync(block, dcoef, cbytes, cudaMemcpyDeviceToHost, st), "d2h coefficients");
    call.sync();
}

// pred8x8_add / pred16x16_add through the device with the caller's block_offset table, in table order (template :1275-1330; the 8x16
// forms take entries 0-3 and 8-11).  Each entry is split into a row (offset / stride, rounded) and a byte column; the rectangle of the
// sub-blocks plus the row above (vertical) or the column left of them (horizontal) is copied, the sub-blocks' rectangle copied back.
template <int DEPTH>
void add_table_host(int t, int m, uint8_t *pix, const int *block_offset, int16_t *block, ptrdiff_t stride)
{
    constexpr int BPS = DEPTH > 8 ? 2 : 1;
    using C = typename std::conditional<(DEPTH > 8), int32_t, int16_t>::type;
    if (stride == 0) B200HostCall::fail(kFeature, "zero stride");
    const int nsub = t == A16 ? 16 : t == A816 ? 8 : 4;
    const bool vert = m == 2;
    long long dx[16], dy[16], minx = 0, maxx = 0, miny = 0, maxy = 0;
    for (int k = 0; k < nsub; k++) {
        const long long o = block_offset[t == A816 && k >= 4 ? k + 4 : k];
        dy[k] = llround((double)o / (double)stride);
        dx[k] = o - dy[k] * (long long)stride;
        if (!k || dx[k] < minx) minx = dx[k];
        if (!k || dx[k] > maxx) maxx = dx[k];
        if (!k || dy[k] < miny) miny = dy[k];
        if (!k || dy[k] > maxy) maxy = dy[k];
    }
    const long long x0 = minx - (vert ? 0 : BPS), y0 = miny - (vert ? 1 : 0), x1 = maxx + 4 * BPS, y1 = maxy + 4;
    const size_t wbytes = (size_t)(x1 - x0), rows = (size_t)(y1 - y0), pitch = (wbytes + 15) & ~(size_t)15;
    const size_t cbytes = (size_t)nsub * 16 * sizeof(C), wsize = pitch * rows;
    B200HostCall call(kFeature, nullptr, wsize + 16 * sizeof(long long) + cbytes + 64);
    uint8_t *scr = call.scratch;
    cudaStream_t st = call.stream;
    uint8_t *doffs = scr + ((wsize + 15) & ~(size_t)15), *dcoef = doffs + 16 * sizeof(long long);
    long long offs[16];
    for (int k = 0; k < nsub; k++) offs[k] = (dy[k] - y0) * (long long)pitch + (dx[k] - x0);
    const uint8_t *org = pix + x0 + y0 * (long long)stride;
    call.check(b200_h2d_rows(scr, pitch, org, stride, wbytes, rows, st), "h2d window");
    call.check(cudaMemcpyAsync(doffs, offs, sizeof(offs), cudaMemcpyHostToDevice, st), "h2d offsets");
    call.check(cudaMemcpyAsync(dcoef, block, cbytes, cudaMemcpyHostToDevice, st), "h2d coefficients");
    using P = typename std::conditional<(DEPTH > 8), uint16_t, uint8_t>::type;
    h264_pred_add_table_kernel<P, C><<<1, 32, 0, st>>>(scr, (const long long *)doffs, nsub, vert, (long long)pitch, (C *)dcoef);
    B200_LAUNCHED();
    call.launched();
    // back: the sub-blocks' rectangle (without the row above / the column to the left)
    const long long bx0 = minx, by0 = miny;
    call.check(b200_d2h_rows(pix + bx0 + by0 * (long long)stride, stride, scr + (by0 - y0) * (long long)pitch + (bx0 - x0), pitch, (size_t)(x1 - bx0),
                             (size_t)(y1 - by0), st),
               "d2h");
    call.check(cudaMemcpyAsync(block, dcoef, cbytes, cudaMemcpyDeviceToHost, st), "d2h coefficients");
    call.sync();
}

template <int D, int M> void tab4(uint8_t *src, const uint8_t *topright, ptrdiff_t stride) { pred_host<D>(P4, M, 0, src, stride, topright); }
template <int D, int M> void tab8l(uint8_t *src, int topleft, int topright, ptrdiff_t stride)
{
    pred_host<D>(P8L, M, (topleft ? 1 : 0) | (topright ? 2 : 0), src, stride, nullptr);          // the decoder passes 0x8000 / 0x4000
}
template <int D, int T, int M> void tab8(uint8_t *src, ptrdiff_t stride) { pred_host<D>(T, M, 0, src, stride, nullptr); }
template <int D, int T, int M> void tab_add(uint8_t *pix, int16_t *block, ptrdiff_t stride) { add_host<D>(T, M, 0, pix, block, stride); }
template <int D, int M> void tab_filter_add(uint8_t *pix, int16_t *block, int topleft, int topright, ptrdiff_t stride)
{
    add_host<D>(A8LF, M, (topleft ? 1 : 0) | (topright ? 2 : 0), pix, block, stride);
}
template <int D, int T, int M> void tab_add_table(uint8_t *pix, const int *block_offset, int16_t *block, ptrdiff_t stride)
{
    add_table_host<D>(T, M, pix, block_offset, block, stride);
}

// h264pred.c:447-538 for codec_id H.264
template <int D>
void fill(B200H264PredContext *h, bool c422)
{
#define B200_P4(m) h->pred4x4[m] = tab4<D, m>; h->pred8x8l[m] = tab8l<D, m>;
    B200_P4(0) B200_P4(1) B200_P4(2) B200_P4(3) B200_P4(4) B200_P4(5) B200_P4(6) B200_P4(7) B200_P4(8) B200_P4(9) B200_P4(10) B200_P4(11)
#undef B200_P4
#define B200_P8(m) h->pred8x8[m] = c422 ? tab8<D, P816, m> : tab8<D, P8, m>;
    B200_P8(0) B200_P8(1) B200_P8(2) B200_P8(3) B200_P8(4) B200_P8(5) B200_P8(6) B200_P8(7) B200_P8(8) B200_P8(9) B200_P8(10)
#undef B200_P8
#define B200_P16(m) h->pred16x16[m] = tab8<D, P16, m>;
    B200_P16(0) B200_P16(1) B200_P16(2) B200_P16(3) B200_P16(4) B200_P16(5) B200_P16(6)
#undef B200_P16
    h->pred4x4_add[0] = tab_add<D, A4, 0>; h->pred4x4_add[1] = tab_add<D, A4, 1>;
    h->pred8x8l_add[0] = tab_add<D, A8L, 0>; h->pred8x8l_add[1] = tab_add<D, A8L, 1>;
    h->pred8x8l_filter_add[0] = tab_filter_add<D, 0>; h->pred8x8l_filter_add[1] = tab_filter_add<D, 1>;
    h->pred8x8_add[1] = c422 ? tab_add_table<D, A816, 1> : tab_add_table<D, A8, 1>;
    h->pred8x8_add[2] = c422 ? tab_add_table<D, A816, 2> : tab_add_table<D, A8, 2>;
    h->pred16x16_add[1] = tab_add_table<D, A16, 1>; h->pred16x16_add[2] = tab_add_table<D, A16, 2>;
}

int check_batch(int bit_depth, int64_t nops, ptrdiff_t stride)
{
    if (nops < 0 || stride < 0) { b200_set_error("h264 pred batch: negative nops or stride"); return B200_EINVAL; }
    if (!depth_ok(bit_depth)) { b200_set_error("h264 pred batch: bit depth %d is not 8, 9, 10, 12 or 14", bit_depth); return B200_EINVAL; }
    if (bit_depth > 8 && (stride & 1)) { b200_set_error("h264 pred batch: odd stride for 16-bit samples"); return B200_EINVAL; }
    return 0;
}

} // namespace

B200_API int b200_h264_pred_init(B200H264PredContext *h, int codec_id, int bit_depth, int chroma_format_idc)
{
    if (!h || chroma_format_idc < 0 || chroma_format_idc > 3) return B200_EINVAL;
    if (codec_id != B200_CODEC_ID_H264 || !depth_ok(bit_depth)) return B200_ENOSYS;      // SVQ3 / RV40 / VP7 / VP8: h264pred.c:556-587
    if (!b200_default_device()) return B200_ENODEV;
    memset(h, 0, sizeof(*h));                                            // the members the reference leaves NULL stay NULL
    const bool c422 = chroma_format_idc > 1;                             // h264pred.c:475, :487, :509, :530
    switch (bit_depth) {
    case 8:  fill<8>(h, c422); break;
    case 9:  fill<9>(h, c422); break;
    case 10: fill<10>(h, c422); break;
    case 12: fill<12>(h, c422); break;
    default: fill<14>(h, c422); break;
    }
    return 0;
}

B200_API int b200_h264_pred_batch_device(B200Device *dev, int bit_depth, int64_t nops, const uint8_t *kinds, const uint8_t *flags, uint8_t *pix,
                                         const int64_t *pix_off, ptrdiff_t stride)
{
    if (int r = check_batch(bit_depth, nops, stride)) return r;
    if (nops == 0) return 0;
    if (!kinds || !flags || !pix || !pix_off || (bit_depth > 8 && ((uintptr_t)pix & 1))) {
        b200_set_error("h264 pred batch: NULL or misaligned pointer");
        return B200_EINVAL;
    }
    if (int r = b200_use_device(dev)) return r;
    B200_CUDA_OK(launch_pred(bit_depth, nops, kinds, flags, pix, (const long long *)pix_off, (long long)stride, dev->stream));
    return 0;
}

B200_API int b200_h264_pred_add_batch_device(B200Device *dev, int bit_depth, int64_t nops, const uint8_t *kinds, const uint8_t *flags, uint8_t *pix,
                                             const int64_t *pix_off, ptrdiff_t stride, void *coef, const int64_t *coef_off)
{
    if (int r = check_batch(bit_depth, nops, stride)) return r;
    if (nops == 0) return 0;
    if (!kinds || !flags || !pix || !pix_off || !coef || !coef_off || (bit_depth > 8 && ((uintptr_t)pix & 1))) {
        b200_set_error("h264 pred add batch: NULL or misaligned pointer");
        return B200_EINVAL;
    }
    if (int r = b200_use_device(dev)) return r;
    B200_CUDA_OK(launch_add(bit_depth, nops, kinds, flags, pix, (const long long *)pix_off, (long long)stride, coef, (const long long *)coef_off, dev->stream));
    return 0;
}
