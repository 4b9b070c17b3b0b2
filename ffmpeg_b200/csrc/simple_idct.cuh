// simple_idct.cuh — the arithmetic of libavcodec's "simple" IDCT (simple_idct_template.c) for every depth and route: the
// constants, the 8-point butterfly, the row pass (idctRowCondDC, :114-206) and the column sums (IDCT_COLS, :209-257).  All sums
// are taken mod 2^32 like the reference's unsigned arithmetic.  Used by the 8-bit kernels (idct.cu) and by the 10 / 12 bit and
// ProRes kernels (idct_hbd.cu), inside their anonymous namespaces.  Host compilers get plain C++ for the two inline-PTX helpers,
// so that tests/cuda_emu can run the high-bit-depth kernels on the CPU.
#pragma once

// simple_idct_template.c:63-104.  DC: the shift of the row pass's DC-only shortcut, (row[0] << DC) & 0xffff, or (row[0] + 1) >> 1
// for DC = -1.  110 is the EXTRA_SHIFT instantiation proresdsp.c makes of the 10-bit constants (simple_idct_template.c:73-76:
// ROW_SHIFT 13, COL_SHIFT 18, DC_SHIFT 1) with the two extra bits its row pass is called with (proresdsp.c:61-62) folded in.
template <int V> struct SimpleIdct;
template <> struct SimpleIdct<8>   { static constexpr unsigned W1 = 22725, W2 = 21407, W3 = 19266, W4 = 16383, W5 = 12873, W6 = 8867, W7 = 4520;
                                     static constexpr int ROW = 11, COL = 20, DC = 3; };
template <> struct SimpleIdct<10>  { static constexpr unsigned W1 = 22725, W2 = 21407, W3 = 19265, W4 = 16384, W5 = 12873, W6 = 8867, W7 = 4520;
                                     static constexpr int ROW = 12, COL = 19, DC = 2; };
template <> struct SimpleIdct<12>  { static constexpr unsigned W1 = 45451, W2 = 42813, W3 = 38531, W4 = 32767, W5 = 25746, W6 = 17734, W7 = 9041;
                                     static constexpr int ROW = 16, COL = 17, DC = -1; };
template <> struct SimpleIdct<110> { static constexpr unsigned W1 = 22725, W2 = 21407, W3 = 19265, W4 = 16384, W5 = 12873, W6 = 8867, W7 = 4520;
                                     static constexpr int ROW = 15, COL = 18, DC = -1; };

// sign-extend the low half in one PRMT: selector nibble 9 = "replicate the sign of byte 1".  __byte_perm() masks the
// selector to 3 bits per nibble, so the sign-replicate mode needs the PTX instruction itself.
__device__ __forceinline__ int sx_lo(unsigned v)
{
#ifdef __CUDA_ARCH__
    int d;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(v), "r"(0u), "r"(0x9910u));
    return d;
#else
    return (int)(int16_t)(v & 0xffffu);
#endif
}
__device__ __forceinline__ int sx_hi(unsigned v) { return (int)v >> 16; }

// The 8-point butterfly shared by both passes (simple_idct_template.c:157-199 rows, :209-257 columns), all sums mod 2^32
// like the reference's unsigned arithmetic.  Every output sum is ONE multiply-add chain that starts from the even part
// (a_i + b_i accumulated in place) and its mirror output is 2*a_i - (a_i + b_i): 22 multiply-adds + 8 adds per
// transform instead of 22 + 14, and the adds that remain are the only work left for the ALU pipe.
//   e[0..7] = a0+b0, a1+b1, a2+b2, a3+b3, a3-b3, a2-b2, a1-b1, a0-b0   (before the final shift)
// mad.lo through inline PTX so that the compiler cannot re-associate the chains back into separate sums
__device__ __forceinline__ unsigned mad(unsigned k, unsigned x, unsigned acc)
{
#ifdef __CUDA_ARCH__
    unsigned d;
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(x), "r"(k), "r"(acc));
    return d;
#else
    return k * x + acc;
#endif
}
template <unsigned K1, unsigned K2, unsigned K3, unsigned K4, unsigned K5, unsigned K6, unsigned K7>
__device__ __forceinline__ void odd_even_sums(int c0, int c1, int c2, int c3, int c4, int c5, int c6, int c7, unsigned rnd, unsigned *e)
{
    const unsigned u1 = (unsigned)c1, u2 = (unsigned)c2, u3 = (unsigned)c3, u5 = (unsigned)c5, u6 = (unsigned)c6, u7 = (unsigned)c7;
    const unsigned p = mad(K4, (unsigned)(c0 + c4), rnd), q = mad(K4, (unsigned)(c0 - c4), rnd);
    const unsigned a0 = mad(K2, u2, mad(K6, u6, p)), a3 = 2u * p - a0;
    const unsigned a1 = mad(K6, u2, mad(0u - K2, u6, q)), a2 = 2u * q - a1;
    e[0] = mad(K1, u1, mad(K3, u3, mad(K5, u5, mad(K7, u7, a0))));
    e[1] = mad(K3, u1, mad(0u - K7, u3, mad(0u - K1, u5, mad(0u - K5, u7, a1))));
    e[2] = mad(K5, u1, mad(0u - K1, u3, mad(K7, u5, mad(K3, u7, a2))));
    e[3] = mad(K7, u1, mad(0u - K5, u3, mad(K3, u5, mad(0u - K1, u7, a3))));
    e[7] = 2u * a0 - e[0]; e[6] = 2u * a1 - e[1]; e[5] = 2u * a2 - e[2]; e[4] = 2u * a3 - e[3];
}

// Row pass (simple_idct_template.c:114-206) on one row packed as four (int16, int16) words.  Every constant and the rounding
// term are pre-multiplied by 2^(16 - ROW): only bits ROW..ROW+15 of the reference's 32-bit row sums survive its ">> ROW, store
// as int16" step, and those are bits 16..31 of the scaled sum mod 2^32 — so the high half of each scaled sum IS the int16 the
// reference stores.  A row without AC terms takes the DC-only shortcut instead: (row[0] << DC) & 0xffff, or (row[0] + 1) >> 1.
template <int V>
__device__ __forceinline__ void row_sums(int r0, int r1, int r2, int r3, int r4, int r5, int r6, int r7, unsigned *e)
{
    using C = SimpleIdct<V>;
    constexpr unsigned S = 1u << (16 - C::ROW);
    odd_even_sums<S * C::W1, S * C::W2, S * C::W3, S * C::W4, S * C::W5, S * C::W6, S * C::W7>(r0, r1, r2, r3, r4, r5, r6, r7, 1u << 15, e);
}
__device__ __forceinline__ bool row_dc_only(const uint4 &in) { return ((in.x >> 16) | in.y | in.z | in.w) == 0; }
template <int V> __device__ __forceinline__ unsigned row_dc(unsigned x0)        // x0: row[0] in the low 16 bits
{
    using C = SimpleIdct<V>;
    return (C::DC >= 0 ? x0 << (C::DC >= 0 ? C::DC : 0) : (unsigned)((sx_lo(x0) + 1) >> 1)) & 0xffffu;
}

// The row pass's two result forms.  The int form unpacks the row before the DC-only test and the packed form after it: the
// results are the same, and each order is the one the kernels that use the form were tuned with.
// 8 sign-extended int16 results
template <int V>
__device__ __forceinline__ void row_pass(const uint4 &in, int *o)
{
    const int r0 = sx_lo(in.x), r1 = sx_hi(in.x), r2 = sx_lo(in.y), r3 = sx_hi(in.y);
    const int r4 = sx_lo(in.z), r5 = sx_hi(in.z), r6 = sx_lo(in.w), r7 = sx_hi(in.w);
    if (row_dc_only(in)) {
        const int dc = (int)(int16_t)row_dc<V>((unsigned)r0);
#pragma unroll
        for (int i = 0; i < 8; i++) o[i] = dc;
        return;
    }
    unsigned e[8];
    row_sums<V>(r0, r1, r2, r3, r4, r5, r6, r7, e);
#pragma unroll
    for (int i = 0; i < 8; i++) o[i] = (int)e[i] >> 16;
}
// four packed (int16, int16) words: the high halves of the scaled sums are picked by PRMT
template <int V>
__device__ __forceinline__ void row_pass(const uint4 &in, unsigned *o)
{
    if (row_dc_only(in)) {
        const unsigned dc = row_dc<V>(in.x & 0xffffu);
        o[0] = o[1] = o[2] = o[3] = dc | (dc << 16);
        return;
    }
    unsigned e[8];
    row_sums<V>(sx_lo(in.x), sx_hi(in.x), sx_lo(in.y), sx_hi(in.y), sx_lo(in.z), sx_hi(in.z), sx_lo(in.w), sx_hi(in.w), e);
    o[0] = __byte_perm(e[0], e[1], 0x7632); o[1] = __byte_perm(e[2], e[3], 0x7632);
    o[2] = __byte_perm(e[4], e[5], 0x7632); o[3] = __byte_perm(e[6], e[7], 0x7632);
}

// IDCT_COLS (simple_idct_template.c:209-257; the zero tests there only skip additions of zero): the eight sums of one column,
// top to bottom, before the final >> COL.  The rounding term is folded into c0 as W4 * (c0 + (1 << (COL - 1)) / W4).
template <int V>
__device__ __forceinline__ void col_sums(int c0, int c1, int c2, int c3, int c4, int c5, int c6, int c7, unsigned *e)
{
    using C = SimpleIdct<V>;
    odd_even_sums<C::W1, C::W2, C::W3, C::W4, C::W5, C::W6, C::W7>(c0, c1, c2, c3, c4, c5, c6, c7, C::W4 * ((1u << (C::COL - 1)) / C::W4), e);
}

// the same, shifted: the eight results of one column
template <int V>
__device__ __forceinline__ void col_pass(int c0, int c1, int c2, int c3, int c4, int c5, int c6, int c7, int *o)
{
    unsigned e[8];
    col_sums<V>(c0, c1, c2, c3, c4, c5, c6, c7, e);
#pragma unroll
    for (int i = 0; i < 8; i++) o[i] = (int)e[i] >> SimpleIdct<V>::COL;
}
