// vp9itxfm.cu — VP9 residual reconstruction on sm_90a: the itxfm_add[5][4] members of VP9DSPContext (libavcodec/vp9dsp.h:40-122) as
// vp9dsp_itxfm_init fills them for 8, 10 and 12 bit samples (vp9dsp_template.c:1755-1778), and a batched device entry that runs one
// member call per transform block, which is inter_recon's residual loop (vp9recon.c:608-652).
//
// Reference semantics reproduced bit for bit for any coefficient values (checker: oracle/vp9itxfm_oracle.c), vp9dsp_template.c:1155-1753:
//   [tx 0..2][type]  pass 1 = type a on every column of the dense sz x sz block, pass 2 = type b on every column of pass 1's result, with
//                    DCT_DCT idct / idct, DCT_ADST iadst / idct, ADST_DCT idct / iadst, ADST_ADST iadst / iadst; [3][*] idct / idct at
//                    32 points, [4][*] the Walsh-Hadamard transform (pass 1 takes its inputs >> 2, pass 2 as they are)
//   storage          8 bit: coefficients and both passes' results int16, arithmetic in 32 bits (wrapping: the multiplications are
//                    unsigned in the reference); 10 / 12 bit: int32 coefficients and results, arithmetic in int64 (no overflow for any
//                    int32 input).  The Walsh-Hadamard transform works in 32-bit ints at every depth.
//   add              output j of pass 2 for column i goes to dst row j, column i: clip(dst + ((int)(out + 2^(bits - 1)) >> bits)),
//                    bits 4 / 5 / 6 / 6 by size, no shift for the Walsh-Hadamard transform
//   DC only          idct / idct at 4..16 and every 32x32 slot with eob == 1: t = ((c0 * 11585 + 2^13) >> 14) * 11585 + 2^13) >> 14
//                    truncated to int, added to every sample; only c0 is read (and cleared by the members)
// The butterflies follow the VP9 bitstream specification's inverse DCT (an N-point DCT is the N/2-point DCT of the even inputs plus an
// odd part of rotations by cospi_k_64 = round(2^14 cos(k pi / 64))) and inverse ADST (rotations by cospi_k_64, rounded after the
// sums, and the 4-point ADST from sinpi_k_9), with every rounding (x + 2^13) >> 14 where the reference rounds.
//
// Kernel: hevcidct.cu's work distribution.  A CTA of 256 threads takes a run of 1-256 ops (chosen from the batch size) and walks it in
// rounds of at most kCap coefficients.  A round loads its ops' coefficients into shared memory as 16-byte vectors (only the first
// vector of a DC-only op), then runs three line passes over all its ops at once: pass 1 gives every thread one column of one op (the
// whole 1-D transform in registers, truncated to the storage type into a second shared array whose rows are padded to an odd number of
// words); pass 2 one column of that result (the second transform in registers, the rounding shift, the residual written back over the
// op's coefficients, which pass 1 has consumed); pass 3 one destination row (the add, the clip and a store of whole 4-sample words).
// Pass 2's thread owns a destination column (the reference adds output j of column i to row j), so the residual goes through shared
// memory once more to be stored row by row in whole words.  Nothing goes to global memory between the passes.
#include "common.h"
#include <cstring>

namespace {

constexpr int kThreads = 256;
constexpr int kMaxOps = 256;                                 // ops per CTA
constexpr int kHead = 2 * (kMaxOps + 1) + 2 * kMaxOps + 2;  // ints in front of the coefficients (a multiple of 4: 16-byte aligned)
enum { T_DCT = 0, T_ADST = 1, T_WHT = 2 };

// the two storage classes: coefficients C, the passes' results Tmp (the reference's dctcoef tmp[] and out[]: the same type as the
// coefficients), arithmetic T (uint32_t: 32-bit wrapping, as the reference's int with its unsigned multiplications), kCap coefficients
// per round (16 KB), the pass-1 array's row padding in elements (rows of odd words)
template <typename P> struct Store;
template <> struct Store<uint8_t> { using C = int16_t; using Tmp = int16_t; using T = uint32_t; static constexpr int kCap = 8192, kPad = 2; };
template <> struct Store<uint16_t> { using C = int32_t; using Tmp = int32_t; using T = long long; static constexpr int kCap = 4096, kPad = 1; };
template <typename P> constexpr int bcap() { return Store<P>::kCap + Store<P>::kCap / 4 * Store<P>::kPad; }   // N (N + pad) <= this share
template <typename P> constexpr size_t smem_bytes()
{
    return 4 * kHead + sizeof(typename Store<P>::C) * Store<P>::kCap + sizeof(typename Store<P>::Tmp) * bcap<P>();
}

struct ItxArgs {
    const B200Vp9TxOp *ops;
    long long nops;
    const void *coef;
    uint8_t *dst;
    long long dst_stride;
    int depth, ops_per_cta;
};

// (v + 2^13) >> 14 with the reference's arithmetic: the 32-bit sum read as int, or exact in int64
template <typename T>
__device__ __forceinline__ T r14(T v)
{
    if constexpr (sizeof(T) == 4) return (T)((int)(v + 8192u) >> 14);
    else return (v + 8192) >> 14;
}
template <typename T> __device__ __forceinline__ T mul(T v, int c) { return v * (T)c; }

// rotation by the pair (c, s): p = a c - b s, q = a s + b c, unrounded
template <typename T>
__device__ __forceinline__ void rot(T a, T b, int c, int s, T &p, T &q)
{
    p = mul(a, c) - mul(b, s);
    q = mul(a, s) + mul(b, c);
}
// the same, rounded
template <typename T>
__device__ __forceinline__ void rotr(T a, T b, int c, int s, T &p, T &q)
{
    rot(a, b, c, s, p, q);
    p = r14(p);
    q = r14(q);
}
// the ADST's input rotation: p = a c + b s, q = a s - b c, unrounded
template <typename T>
__device__ __forceinline__ void arot(T a, T b, int c, int s, T &p, T &q)
{
    p = mul(a, c) + mul(b, s);
    q = mul(a, s) - mul(b, c);
}

// inverse DCT of N points, inputs x[k S]
template <typename T, int N, int S>
__device__ __forceinline__ void idct(const T *x, T *y)
{
    if constexpr (N == 4) {
        const T e0 = r14(mul(x[0] + x[2 * S], 11585)), e1 = r14(mul(x[0] - x[2 * S], 11585));
        T o0, o1;
        rotr(x[S], x[3 * S], 6270, 15137, o0, o1);
        y[0] = e0 + o1;
        y[1] = e1 + o0;
        y[2] = e1 - o0;
        y[3] = e0 - o1;
    } else {
        T e[N / 2], o[N / 2];
        idct<T, N / 2, 2 * S>(x, e);
        if constexpr (N == 8) {
            T a4, a5, a6, a7;
            rotr(x[S], x[7 * S], 3196, 16069, a4, a7);
            rotr(x[5 * S], x[3 * S], 13623, 9102, a5, a6);
            const T b4 = a4 + a5, b5 = a4 - a5, b6 = a7 - a6, b7 = a7 + a6;
            o[0] = b7;
            o[1] = r14(mul(b6 + b5, 11585));
            o[2] = r14(mul(b6 - b5, 11585));
            o[3] = b4;
        } else if constexpr (N == 16) {
            T a8, a9, a10, a11, a12, a13, a14, a15;
            rotr(x[S], x[15 * S], 1606, 16305, a8, a15);
            rotr(x[9 * S], x[7 * S], 12665, 10394, a9, a14);
            rotr(x[5 * S], x[11 * S], 7723, 14449, a10, a13);
            rotr(x[13 * S], x[3 * S], 15679, 4756, a11, a12);
            const T b8 = a8 + a9, b9 = a8 - a9, b10 = a11 - a10, b11 = a11 + a10;
            const T b12 = a12 + a13, b13 = a12 - a13, b14 = a15 - a14, b15 = a15 + a14;
            T c9, c14, c10, c13;
            rotr(b14, b9, 6270, 15137, c9, c14);
            rot(b13, b10, 6270, 15137, c13, c10);
            c13 = r14(c13);
            c10 = r14((T)0 - c10);
            const T d8 = b8 + b11, d9 = c9 + c10, d10 = c9 - c10, d11 = b8 - b11;
            const T d12 = b15 - b12, d13 = c14 - c13, d14 = c14 + c13, d15 = b15 + b12;
            o[0] = d15;
            o[1] = d14;
            o[2] = r14(mul(d13 + d10, 11585));
            o[3] = r14(mul(d12 + d11, 11585));
            o[4] = r14(mul(d12 - d11, 11585));
            o[5] = r14(mul(d13 - d10, 11585));
            o[6] = d9;
            o[7] = d8;
        } else {
            static_assert(N == 32, "idct sizes 4..32");
            T a[32];                                             // a[16..31]: the odd part's stage values, indexed as in the spec
            rotr(x[S], x[31 * S], 804, 16364, a[16], a[31]);
            rotr(x[17 * S], x[15 * S], 12140, 11003, a[17], a[30]);
            rotr(x[9 * S], x[23 * S], 7005, 14811, a[18], a[29]);
            rotr(x[25 * S], x[7 * S], 15426, 5520, a[19], a[28]);
            rotr(x[5 * S], x[27 * S], 3981, 15893, a[20], a[27]);
            rotr(x[21 * S], x[11 * S], 14053, 8423, a[21], a[26]);
            rotr(x[13 * S], x[19 * S], 9760, 13160, a[22], a[25]);
            rotr(x[29 * S], x[3 * S], 16207, 2404, a[23], a[24]);
            T b[32];
#pragma unroll
            for (int k = 16; k < 32; k += 4) {                   // pairs (16,17) (19,18) (20,21) (23,22) ...: sum and difference
                b[k] = a[k] + a[k + 1];
                b[k + 1] = a[k] - a[k + 1];
                b[k + 2] = a[k + 3] - a[k + 2];
                b[k + 3] = a[k + 3] + a[k + 2];
            }
            T c17, c30, c18, c29, c21, c26, c22, c25;
            rotr(b[30], b[17], 3196, 16069, c17, c30);
            rot(b[29], b[18], 3196, 16069, c29, c18);
            c29 = r14(c29);
            c18 = r14((T)0 - c18);
            rotr(b[26], b[21], 13623, 9102, c21, c26);
            rot(b[25], b[22], 13623, 9102, c25, c22);
            c25 = r14(c25);
            c22 = r14((T)0 - c22);
            const T d16 = b[16] + b[19], d17 = c17 + c18, d18 = c17 - c18, d19 = b[16] - b[19];
            const T d20 = b[23] - b[20], d21 = c22 - c21, d22 = c22 + c21, d23 = b[23] + b[20];
            const T d24 = b[24] + b[27], d25 = c25 + c26, d26 = c25 - c26, d27 = b[24] - b[27];
            const T d28 = b[31] - b[28], d29 = c30 - c29, d30 = c30 + c29, d31 = b[31] + b[28];
            T e18, e29, e19, e28, e20, e27, e21, e26;
            rotr(d29, d18, 6270, 15137, e18, e29);
            rotr(d28, d19, 6270, 15137, e19, e28);
            rot(d27, d20, 6270, 15137, e27, e20);
            e27 = r14(e27);
            e20 = r14((T)0 - e20);
            rot(d26, d21, 6270, 15137, e26, e21);
            e26 = r14(e26);
            e21 = r14((T)0 - e21);
            const T f16 = d16 + d23, f17 = d17 + d22, f18 = e18 + e21, f19 = e19 + e20;
            const T f20 = e19 - e20, f21 = e18 - e21, f22 = d17 - d22, f23 = d16 - d23;
            const T f24 = d31 - d24, f25 = d30 - d25, f26 = e29 - e26, f27 = e28 - e27;
            const T f28 = e28 + e27, f29 = e29 + e26, f30 = d30 + d25, f31 = d31 + d24;
            o[0] = f31;
            o[1] = f30;
            o[2] = f29;
            o[3] = f28;
            o[4] = r14(mul(f27 + f20, 11585));
            o[5] = r14(mul(f26 + f21, 11585));
            o[6] = r14(mul(f25 + f22, 11585));
            o[7] = r14(mul(f24 + f23, 11585));
            o[8] = r14(mul(f24 - f23, 11585));
            o[9] = r14(mul(f25 - f22, 11585));
            o[10] = r14(mul(f26 - f21, 11585));
            o[11] = r14(mul(f27 - f20, 11585));
            o[12] = f19;
            o[13] = f18;
            o[14] = f17;
            o[15] = f16;
        }
#pragma unroll
        for (int i = 0; i < N / 2; i++) {
            y[i] = e[i] + o[i];
            y[N - 1 - i] = e[i] - o[i];
        }
    }
}

// inverse ADST of N = 4, 8, 16 points
template <typename T, int N>
__device__ __forceinline__ void iadst(const T *x, T *y)
{
    if constexpr (N == 4) {                                      // sinpi_k_9: 5283, 9929, 13377, 15212
        const T s0 = mul(x[0], 5283) + mul(x[2], 15212) + mul(x[3], 9929);
        const T s1 = mul(x[0], 9929) - mul(x[2], 5283) - mul(x[3], 15212);
        const T s2 = mul(x[0] - x[2] + x[3], 13377), s3 = mul(x[1], 13377);
        y[0] = r14(s0 + s3);
        y[1] = r14(s1 + s3);
        y[2] = r14(s2);
        y[3] = r14(s0 + s1 - s3);
    } else if constexpr (N == 8) {
        T p[8];
        arot(x[7], x[0], 16305, 1606, p[0], p[1]);
        arot(x[5], x[2], 14449, 7723, p[2], p[3]);
        arot(x[3], x[4], 10394, 12665, p[4], p[5]);
        arot(x[1], x[6], 4756, 15679, p[6], p[7]);
        T q[8];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            q[k] = r14(p[k] + p[k + 4]);
            q[k + 4] = r14(p[k] - p[k + 4]);
        }
        T u4, u5, u6, u7;
        arot(q[4], q[5], 15137, 6270, u4, u5);
        arot(q[7], q[6], 6270, 15137, u7, u6);
        const T v2 = q[0] - q[2], v3 = q[1] - q[3], v6 = r14(u4 - u6), v7 = r14(u5 - u7);
        y[0] = q[0] + q[2];
        y[7] = (T)0 - (q[1] + q[3]);
        y[1] = (T)0 - r14(u4 + u6);
        y[6] = r14(u5 + u7);
        y[3] = (T)0 - r14(mul(v2 + v3, 11585));
        y[4] = r14(mul(v2 - v3, 11585));
        y[2] = r14(mul(v6 + v7, 11585));
        y[5] = (T)0 - r14(mul(v6 - v7, 11585));
    } else {
        static_assert(N == 16, "iadst sizes 4..16");
        T p[16];
        arot(x[15], x[0], 16364, 804, p[0], p[1]);
        arot(x[13], x[2], 15893, 3981, p[2], p[3]);
        arot(x[11], x[4], 14811, 7005, p[4], p[5]);
        arot(x[9], x[6], 13160, 9760, p[6], p[7]);
        arot(x[7], x[8], 11003, 12140, p[8], p[9]);
        arot(x[5], x[10], 8423, 14053, p[10], p[11]);
        arot(x[3], x[12], 5520, 15426, p[12], p[13]);
        arot(x[1], x[14], 2404, 16207, p[14], p[15]);
        T q[16];
#pragma unroll
        for (int k = 0; k < 8; k++) {
            q[k] = r14(p[k] + p[k + 8]);
            q[k + 8] = r14(p[k] - p[k + 8]);
        }
        T u8, u9, u10, u11, u12, u13, u14, u15;
        arot(q[8], q[9], 16069, 3196, u8, u9);
        arot(q[10], q[11], 9102, 13623, u10, u11);
        arot(q[13], q[12], 3196, 16069, u13, u12);
        arot(q[15], q[14], 13623, 9102, u15, u14);
        T r[16];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            r[k] = q[k] + q[k + 4];
            r[k + 4] = q[k] - q[k + 4];
        }
        r[8] = r14(u8 + u12);
        r[9] = r14(u9 + u13);
        r[10] = r14(u10 + u14);
        r[11] = r14(u11 + u15);
        r[12] = r14(u8 - u12);
        r[13] = r14(u9 - u13);
        r[14] = r14(u10 - u14);
        r[15] = r14(u11 - u15);
        T w4, w5, w6, w7, w12, w13, w14, w15;
        arot(r[4], r[5], 15137, 6270, w4, w5);
        arot(r[7], r[6], 6270, 15137, w7, w6);
        arot(r[12], r[13], 15137, 6270, w12, w13);
        arot(r[15], r[14], 6270, 15137, w15, w14);
        const T s2 = r[0] - r[2], s3 = r[1] - r[3];
        const T s6 = r14(w4 - w6), s7 = r14(w5 - w7);
        const T s10 = r[8] - r[10], s11 = r[9] - r[11];
        const T s14 = r14(w12 - w14), s15 = r14(w13 - w15);
        y[0] = r[0] + r[2];
        y[15] = (T)0 - (r[1] + r[3]);
        y[3] = (T)0 - r14(w4 + w6);
        y[12] = r14(w5 + w7);
        y[1] = (T)0 - (r[8] + r[10]);
        y[14] = r[9] + r[11];
        y[2] = r14(w12 + w14);
        y[13] = (T)0 - r14(w13 + w15);
        y[7] = r14(mul((T)0 - (s2 + s3), 11585));
        y[8] = r14(mul(s2 - s3, 11585));
        y[4] = r14(mul(s7 + s6, 11585));
        y[11] = r14(mul(s7 - s6, 11585));
        y[6] = r14(mul(s11 + s10, 11585));
        y[9] = r14(mul(s11 - s10, 11585));
        y[5] = r14(mul((T)0 - (s14 + s15), 11585));
        y[10] = r14(mul(s14 - s15, 11585));
    }
}

// the Walsh-Hadamard transform in 32-bit ints at every depth; pass 1 takes its inputs >> 2
template <typename C>
__device__ __forceinline__ void iwht(const C *x, C *y, bool first)
{
    const int sh = first ? 2 : 0;
    const unsigned a = (unsigned)((int)x[0] >> sh), b = (unsigned)((int)x[3] >> sh);
    const unsigned c = (unsigned)((int)x[1] >> sh), d = (unsigned)((int)x[2] >> sh);
    const unsigned s = a + c, t = d - b;
    const unsigned h = (unsigned)((int)(s - t) >> 1);
    const unsigned y1 = h - b, y2 = h - c;
    y[0] = (C)(int)(s - y1);
    y[1] = (C)(int)y1;
    y[2] = (C)(int)y2;
    y[3] = (C)(int)(t + y2);
}

// one 1-D transform of N stored values x to N stored values y (truncated to the pass results' type)
template <typename P, int N, typename X>
__device__ __forceinline__ void tx1d(int type, bool first, const X *x, typename Store<P>::Tmp *y)
{
    using Tmp = typename Store<P>::Tmp;
    using T = typename Store<P>::T;
    if constexpr (N == 4) {
        if (type == T_WHT) {
            Tmp u[4];
#pragma unroll
            for (int k = 0; k < 4; k++) u[k] = (Tmp)x[k];
            iwht<Tmp>(u, y, first);
            return;
        }
    }
    T u[N], v[N];
#pragma unroll
    for (int k = 0; k < N; k++) u[k] = (T)x[k];
    if constexpr (N == 32) {
        idct<T, 32, 1>(u, v);
    } else {
        if (type == T_ADST) iadst<T, N>(u, v);
        else idct<T, N, 1>(u, v);
    }
#pragma unroll
    for (int k = 0; k < N; k++) y[k] = (Tmp)v[k];
}

// meta of an op: log2 size | type a << 8 | type b << 10 | DC only << 12 | bits << 13; -1 for an op the guard refuses
__host__ __device__ __forceinline__ bool dc_only(int tx, int type, int eob) { return eob == 1 && (tx == 3 || (tx < 3 && type == 0)); }

template <typename P>
__device__ __forceinline__ int op_meta(const B200Vp9TxOp &op)
{
    if (op.tx > 4 || op.type > 3 || (op.coef_off & 15) || (op.dst_off & (4 * sizeof(P) - 1))) return -1;
    const int tx = op.tx;
    if (tx == 4) return 2 | T_WHT << 8 | T_WHT << 10;
    const int ta = tx == 3 ? T_DCT : (op.type & 1) ? T_ADST : T_DCT;
    const int tb = tx == 3 ? T_DCT : (op.type & 2) ? T_ADST : T_DCT;
    return (tx + 2) | ta << 8 | tb << 10 | (dc_only(tx, op.type, op.eob) ? 1 << 12 : 0) | (tx < 2 ? 4 + tx : 6) << 13;
}

template <typename P, int N>
__device__ __forceinline__ void pass1(int m, int c, const typename Store<P>::C *A, typename Store<P>::Tmp *B)
{
    using C = typename Store<P>::C;
    constexpr int pitch = N + Store<P>::kPad;
    C x[N];
    typename Store<P>::Tmp y[N];
#pragma unroll
    for (int k = 0; k < N; k++) x[k] = A[k * N + c];
    tx1d<P, N>((m >> 8) & 3, true, x, y);
#pragma unroll
    for (int k = 0; k < N; k++) B[k * pitch + c] = y[k];          // row k of B = output k of every column
}

template <typename P, int N>
__device__ __forceinline__ void pass2(int m, int i, typename Store<P>::C *A, const typename Store<P>::Tmp *B)
{
    using C = typename Store<P>::C;
    constexpr int pitch = N + Store<P>::kPad;
    typename Store<P>::Tmp x[N], y[N];
#pragma unroll
    for (int k = 0; k < N; k++) x[k] = B[i * pitch + k];          // output i of column k of pass 1
    tx1d<P, N>((m >> 10) & 3, false, x, y);
    const int bits = m >> 13;
#pragma unroll
    for (int j = 0; j < N; j++)
        A[j * N + i] = bits ? (C)((int)((unsigned)(int)y[j] + (1u << (bits - 1))) >> bits) : y[j];
}

// one destination word of 4 samples: load, add (32-bit wrapping, as the reference's int sum), clip, store
template <typename P>
__device__ __forceinline__ void add4(P *d, const int *r, int maxv)
{
    auto px = [maxv](int s, int v) { return (unsigned)min(max((int)((unsigned)s + (unsigned)v), 0), maxv); };
    if constexpr (sizeof(P) == 1) {
        const unsigned w = *reinterpret_cast<const unsigned *>(d);
        unsigned o = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) o |= px((w >> (8 * k)) & 0xFF, r[k]) << (8 * k);
        *reinterpret_cast<unsigned *>(d) = o;
    } else {
        const uint2 w = *reinterpret_cast<const uint2 *>(d);
        uint2 o;
        o.x = px(w.x & 0xFFFF, r[0]) | px(w.x >> 16, r[1]) << 16;
        o.y = px(w.y & 0xFFFF, r[2]) | px(w.y >> 16, r[3]) << 16;
        *reinterpret_cast<uint2 *>(d) = o;
    }
}

template <typename P, int N>
__device__ __forceinline__ void pass3(int m, int j, long long dst_off, const typename Store<P>::C *A, const ItxArgs &a)
{
    using T = typename Store<P>::T;
    int r[N];
    if (m & (1 << 12)) {
        const T t1 = r14(mul((T)A[0], 11585));
        const int t = (int)r14(mul(t1, 11585));                   // the reference's `const int t`
        const int bits = m >> 13;
        const int v = (int)((unsigned)t + (1u << (bits - 1))) >> bits;
#pragma unroll
        for (int k = 0; k < N; k++) r[k] = v;
    } else {
#pragma unroll
        for (int k = 0; k < N; k++) r[k] = A[j * N + k];
    }
    P *d = reinterpret_cast<P *>(a.dst + dst_off + (long long)j * a.dst_stride);
    const int maxv = (1 << a.depth) - 1;
#pragma unroll
    for (int k = 0; k < N; k += 4) add4<P>(d + k, r + k, maxv);
}

// largest i in [lo, hi) with v[i] <= x (v non-decreasing, v[lo] <= x)
__device__ __forceinline__ int find(const int *v, int lo, int hi, int x)
{
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (v[mid] <= x) lo = mid;
        else hi = mid;
    }
    return lo;
}

template <typename P>
__global__ void __launch_bounds__(kThreads) vp9_itx_kernel(ItxArgs a)
{
    using C = typename Store<P>::C;
    constexpr int kCap = Store<P>::kCap, kPad = Store<P>::kPad, kVec = 16 / sizeof(C);
    extern __shared__ int4 vp9_itx_smem[];
    int *S = reinterpret_cast<int *>(vp9_itx_smem);          // [i] = first coefficient of op i in the CTA's run, [n] = total
    int *L = S + kMaxOps + 1;                                // [i] = first line of op i
    int *meta = L + kMaxOps + 1;                             // op_meta
    int *boff = meta + kMaxOps;                              // first element of op i in Bs, relative to its round
    using Tmp = typename Store<P>::Tmp;
    C *As = reinterpret_cast<C *>(S + kHead);
    Tmp *Bs = reinterpret_cast<Tmp *>(As + kCap);
    const C *coef = reinterpret_cast<const C *>(a.coef);
    const int tid = threadIdx.x;
    const long long o0 = (long long)blockIdx.x * a.ops_per_cta;
    const int n = (int)(a.nops - o0 < a.ops_per_cta ? a.nops - o0 : a.ops_per_cta);
    const B200Vp9TxOp *ops = a.ops + o0;
    if (tid < n) {
        const int m = op_meta<P>(ops[tid]);
        const int l2 = m < 0 ? 0 : m & 0xFF;
        meta[tid] = m;
        S[tid + 1] = m < 0 ? 0 : 1 << (2 * l2);
        L[tid + 1] = m < 0 ? 0 : 1 << l2;
    }
    if (tid == 0) S[0] = L[0] = 0;
    __syncthreads();
    for (int d = 1; d < n; d <<= 1) {                        // inclusive scan of S[1..n], L[1..n]
        int s = 0, l = 0;
        if (tid < n && tid >= d) s = S[tid + 1 - d], l = L[tid + 1 - d];
        __syncthreads();
        if (tid < n && tid >= d) S[tid + 1] += s, L[tid + 1] += l;
        __syncthreads();
    }
    for (int r0 = 0; r0 < n;) {
        const int r1 = find(S, r0, n + 1, S[r0] + kCap);    // ops r0 .. r1 - 1 fit in a round (r1 > r0: an op is at most 1024)
        const int sa = S[r0], la = L[r0];
        for (int i = r0 + tid; i < r1; i += kThreads) boff[i] = S[i] - sa + kPad * (L[i] - la);
        const int nv = (S[r1] - sa) / kVec;
        for (int v = tid; v < nv; v += kThreads) {
            const int s = sa + kVec * v, i = find(S, r0, r1, s);
            if ((meta[i] & (1 << 12)) && s != S[i]) continue;   // a DC-only op reads its first coefficient
            const int4 q = *reinterpret_cast<const int4 *>(coef + ops[i].coef_off + (s - S[i]));
            *reinterpret_cast<int4 *>(As + (s - sa)) = q;
        }
        __syncthreads();
        const int nl = L[r1] - la;
        for (int t = tid; t < nl; t += kThreads) {
            const int i = find(L, r0, r1, la + t), m = meta[i], c = la + t - L[i];
            if (m & (1 << 12)) continue;
            const C *A = As + (S[i] - sa);
            Tmp *B = Bs + boff[i];
            switch (m & 0xFF) {
            case 2:  pass1<P, 4>(m, c, A, B); break;
            case 3:  pass1<P, 8>(m, c, A, B); break;
            case 4:  pass1<P, 16>(m, c, A, B); break;
            default: pass1<P, 32>(m, c, A, B); break;
            }
        }
        __syncthreads();
        for (int t = tid; t < nl; t += kThreads) {
            const int i = find(L, r0, r1, la + t), m = meta[i], c = la + t - L[i];
            if (m & (1 << 12)) continue;
            C *A = As + (S[i] - sa);
            const Tmp *B = Bs + boff[i];
            switch (m & 0xFF) {
            case 2:  pass2<P, 4>(m, c, A, B); break;
            case 3:  pass2<P, 8>(m, c, A, B); break;
            case 4:  pass2<P, 16>(m, c, A, B); break;
            default: pass2<P, 32>(m, c, A, B); break;
            }
        }
        __syncthreads();
        for (int t = tid; t < nl; t += kThreads) {
            const int i = find(L, r0, r1, la + t), m = meta[i], j = la + t - L[i];
            const C *A = As + (S[i] - sa);
            const long long off = ops[i].dst_off;
            switch (m & 0xFF) {
            case 2:  pass3<P, 4>(m, j, off, A, a); break;
            case 3:  pass3<P, 8>(m, j, off, A, a); break;
            case 4:  pass3<P, 16>(m, j, off, A, a); break;
            default: pass3<P, 32>(m, j, off, A, a); break;
            }
        }
        __syncthreads();
        r0 = r1;
    }
}

constexpr long long kChunkOps = 1LL << 20;                   // ops per launch

bool depth_ok(int d) { return d == 8 || d == 10 || d == 12; }

cudaError_t launch(ItxArgs a, cudaStream_t st)
{
    const long long nops = a.nops;
    const long long per = (nops + 1055) / 1056;             // about 8 CTAs per SM for a frame; 1 op per CTA for a few ops
    a.ops_per_cta = (int)(per < 1 ? 1 : per > kMaxOps ? kMaxOps : per);
    const B200Vp9TxOp *ops = a.ops;
    for (long long b = 0; b < nops; b += kChunkOps) {
        a.ops = ops + b;
        a.nops = nops - b < kChunkOps ? nops - b : kChunkOps;
        const unsigned grid = (unsigned)((a.nops + a.ops_per_cta - 1) / a.ops_per_cta);
        if (a.depth == 8) vp9_itx_kernel<uint8_t><<<grid, kThreads, smem_bytes<uint8_t>(), st>>>(a);
        else vp9_itx_kernel<uint16_t><<<grid, kThreads, smem_bytes<uint16_t>(), st>>>(a);
        B200_LAUNCHED();
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

void die(const char *what)
{
    fprintf(stderr, "libb200dsp: vp9 inverse transform failed: %s (%s)\n", what, b200_last_error());
    abort();
}

// ---- drop-in members (host pointers): the block's coefficients and the sz x sz block of dst through the device scratch, one op, the
// block back; the coefficients are then left as the reference leaves them (only block[0] cleared on the DC-only path, all else zeroed)
void member_host(int depth, int tx, int type, uint8_t *dst, ptrdiff_t stride, int16_t *block, int eob)
{
    const int N = tx == 4 ? 4 : 4 << tx, bps = depth > 8 ? 2 : 1, cs = depth > 8 ? 4 : 2;
    const size_t cbytes = (size_t)N * N * cs, dpitch = (size_t)N * bps;
    B200Device *dev = b200_default_device();
    if (!dev) die("no device");
    if (cudaSetDevice(dev->ordinal) != cudaSuccess) die("cudaSetDevice");
    B200_LOCK_DEVICE(dev);            // scratch + stream are per device: one host-pointer call at a time (released on return)
    uint8_t *scr = (uint8_t *)b200_scratch(dev, 256 + 4096 + 2048);
    if (!scr) die("scratch");
    cudaStream_t st = dev->stream;
    uint8_t *dop = scr, *dcoef = scr + 256, *ddst = dcoef + 4096;
    B200Vp9TxOp op;
    memset(&op, 0, sizeof(op));
    op.tx = (uint8_t)tx;
    op.type = (uint8_t)type;
    op.eob = (uint16_t)(eob == 1);   // only eob == 1 means anything to the members; any other int runs the full transform
    if (cudaMemcpyAsync(dop, &op, sizeof(op), cudaMemcpyHostToDevice, st) != cudaSuccess) die("h2d op");
    if (cudaMemcpyAsync(dcoef, block, cbytes, cudaMemcpyHostToDevice, st) != cudaSuccess) die("h2d coefficients");
    if (b200_h2d_rows(ddst, dpitch, dst, stride, dpitch, (size_t)N, st) != cudaSuccess) die("h2d block");
    ItxArgs a = { (const B200Vp9TxOp *)dop, 1, dcoef, ddst, (long long)dpitch, depth, 1 };
    if (launch(a, st) != cudaSuccess) die("launch");
    if (b200_d2h_rows(dst, stride, ddst, dpitch, dpitch, (size_t)N, st) != cudaSuccess) die("d2h block");
    if (cudaStreamSynchronize(st) != cudaSuccess) die("sync");
    memset(block, 0, dc_only(tx, type, eob) ? (size_t)cs : cbytes);
}

template <int D, int TX, int TYPE>
void m_itxfm(uint8_t *dst, ptrdiff_t stride, int16_t *block, int eob) { member_host(D, TX, TYPE, dst, stride, block, eob); }

// vp9dsp_template.c:1755-1778: four functions per size at 4..16, one for every 32x32 slot, one for every lossless slot
template <int D, int TX>
void fill_size(B200VP9DSPContext *c)
{
    if constexpr (TX < 3) {
        c->itxfm_add[TX][0] = m_itxfm<D, TX, 0>;
        c->itxfm_add[TX][1] = m_itxfm<D, TX, 1>;
        c->itxfm_add[TX][2] = m_itxfm<D, TX, 2>;
        c->itxfm_add[TX][3] = m_itxfm<D, TX, 3>;
    } else {
        c->itxfm_add[TX][0] = c->itxfm_add[TX][1] = c->itxfm_add[TX][2] = c->itxfm_add[TX][3] = m_itxfm<D, TX, 0>;
    }
}
template <int D>
void fill(B200VP9DSPContext *c)
{
    fill_size<D, 0>(c); fill_size<D, 1>(c); fill_size<D, 2>(c); fill_size<D, 3>(c); fill_size<D, 4>(c);
}

} // namespace

B200_API int b200_vp9_dsp_init_itxfm(B200VP9DSPContext *c, int bit_depth)
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

B200_API int b200_vp9_itxfm_add_batch_device(B200Device *dev, int bit_depth, int64_t nops, const B200Vp9TxOp *ops, const void *coef,
                                             uint8_t *dst, ptrdiff_t dst_stride)
{
    if (nops < 0) { b200_set_error("vp9 itxfm batch: negative nops"); return B200_EINVAL; }
    if (!depth_ok(bit_depth)) { b200_set_error("vp9 itxfm batch: bit depth %d is not 8, 10 or 12", bit_depth); return B200_EINVAL; }
    const int bps = bit_depth > 8 ? 2 : 1;
    if (dst_stride % (4 * bps)) { b200_set_error("vp9 itxfm batch: dst_stride not a multiple of 4 samples"); return B200_EINVAL; }
    if (nops == 0) return 0;
    if (!ops || !coef || !dst || ((uintptr_t)ops & 7) || ((uintptr_t)coef & 15) || ((uintptr_t)dst % (4 * bps))) {
        b200_set_error("vp9 itxfm batch: NULL or misaligned pointer");
        return B200_EINVAL;
    }
    if (!dev) dev = b200_default_device();
    if (!dev) return B200_ENODEV;
    B200_CUDA_OK(cudaSetDevice(dev->ordinal));
    ItxArgs a = { ops, (long long)nops, coef, dst, (long long)dst_stride, bit_depth, 1 };
    B200_CUDA_OK(launch(a, dev->stream));
    return 0;
}
