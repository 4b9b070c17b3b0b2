// vp9itxfm_dev.cuh — the VP9 1-D inverse transforms of vp9dsp_template.c:1155-1753 in device code, shared by vp9itxfm.cu (the
// itxfm_add members and the residual batch) and vp9intra.cu (the intra frame entry, which adds the same residual after its prediction).
// Storage classes, roundings and wrapping are described at the top of vp9itxfm.cu.
#pragma once

namespace {

enum { T_DCT = 0, T_ADST = 1, T_WHT = 2 };

// the two storage classes: coefficients C, the passes' results Tmp (the reference's dctcoef tmp[] and out[]: the same type as the
// coefficients), arithmetic T (uint32_t: 32-bit wrapping, as the reference's int with its unsigned multiplications), kCap coefficients
// per round (16 KB), the pass-1 array's row padding in elements (rows of odd words)
template <typename P> struct Store;
template <> struct Store<uint8_t> { using C = int16_t; using Tmp = int16_t; using T = uint32_t; static constexpr int kCap = 8192, kPad = 2; };
template <> struct Store<uint16_t> { using C = int32_t; using Tmp = int32_t; using T = long long; static constexpr int kCap = 4096, kPad = 1; };
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

} // namespace
