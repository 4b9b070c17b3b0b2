// mpv_unquant.cuh — the arithmetic of libavcodec's MPEG-1 / MPEG-2 / H.263-MPEG-4 inverse quantisers
// (libavcodec/mpegvideo_unquantize.c:50-276) and the host set-up of its tables, shared by the quantiser kernel (unquant.cu) and
// the quantiser fused in front of the tiled IDCT (idct.cu), inside their anonymous namespaces.  How a kernel walks a block and
// how it applies the MPEG-2 mismatch toggle to block[63] stay with the kernel.
#pragma once

struct UnquantDev {                       // passed by value as (part of) a __grid_constant__ parameter: the per-lane table look-ups
                                          // index the constant bank directly (a plain by-value parameter is copied to local memory
                                          // per thread when indexed at run time)
    uint16_t intra[64], inter[64];
    uint8_t scanpos[64];                  // scan index of each raster coefficient (inverse of ScanTable.permutated)
    uint8_t raster_end[64];
    int y_dc, c_dc, q_type, aic, ac_pred;
};

// B200MpvUnquant -> kernel parameters; false when permutated[] is not a permutation of 0..63
inline bool mpv_unquant_params(const B200MpvUnquant *p, UnquantDev *P)
{
    memcpy(P->intra, p->intra_matrix, sizeof(P->intra));
    memcpy(P->inter, p->inter_matrix, sizeof(P->inter));
    memcpy(P->raster_end, p->raster_end, sizeof(P->raster_end));
    bool seen[64] = { false };
    for (int i = 0; i < 64; i++) {
        const int j = p->permutated[i];
        if (j > 63 || seen[j]) return false;
        seen[j] = true;
        P->scanpos[j] = (uint8_t)i;
    }
    P->y_dc = p->y_dc_scale; P->c_dc = p->c_dc_scale; P->q_type = p->q_scale_type; P->aic = p->h263_aic; P->ac_pred = p->ac_pred;
    return true;
}

__constant__ uint8_t c_nonlinear_qscale[32] = {                    // ff_mpeg2_non_linear_qscale (ISO/IEC 13818-2 table 7-6)
    0, 1, 2, 3, 4, 5, 6, 7, 8, 10, 12, 14, 16, 18, 20, 22, 24, 28, 32, 36, 40, 44, 48, 52, 56, 64, 72, 80, 88, 96, 104, 112,
};

template <int V> struct MpvVariant {
    static constexpr bool H263 = V == B200_UNQUANT_H263_INTRA || V == B200_UNQUANT_H263_INTER;
    static constexpr bool INTRA = V == B200_UNQUANT_MPEG1_INTRA || V == B200_UNQUANT_MPEG2_INTRA ||
                                  V == B200_UNQUANT_MPEG2_INTRA_BITEXACT || V == B200_UNQUANT_H263_INTRA;
    static constexpr bool MISMATCH = V == B200_UNQUANT_MPEG2_INTRA_BITEXACT || V == B200_UNQUANT_MPEG2_INTER;
};

template <int V> __device__ __forceinline__ int dequant(int level, int q, int m)
{
    const unsigned a = (unsigned)(level < 0 ? -level : level);
    int v;
    if (V == B200_UNQUANT_MPEG1_INTRA)      { v = (int)(a * q * m) >> 3; v = (v - 1) | 1; }
    else if (V == B200_UNQUANT_MPEG1_INTER) { v = (int)(((a << 1) + 1) * q * m) >> 4; v = (v - 1) | 1; }
    else if (V == B200_UNQUANT_MPEG2_INTER) { v = (int)(((a << 1) + 1) * q * m) >> 5; }
    else                                    { v = (int)(a * q * m) >> 4; }
    return level < 0 ? -v : v;
}

// raster coefficient j: its matrix entry and the scan position "inside the coded part of the block" is tested on
template <int V> __device__ __forceinline__ int mpv_matrix(const UnquantDev &P, int j)
{
    return (int)(MpvVariant<V>::INTRA ? P.intra[j] : P.inter[j]);
}
template <int V> __device__ __forceinline__ int mpv_scanpos(const UnquantDev &P, int j)
{
    return MpvVariant<V>::H263 ? j : (int)P.scanpos[j];
}

// per block: the quantiser step q, the H.263 rounding term qadd and the last coded scan position ncoef
struct MpvBlock { int q, qadd, ncoef; };
template <int V> __device__ __forceinline__ MpvBlock mpv_block(const UnquantDev &P, int qs, int last)
{
    using T = MpvVariant<V>;
    MpvBlock b = { qs, 0, last };
    if (T::H263) {
        b.q = qs << 1;
        b.qadd = (T::INTRA && P.aic) ? 0 : ((qs - 1) | 1);
        b.ncoef = (T::INTRA && P.ac_pred) ? 63 : (last >= 0 ? (int)P.raster_end[last] : -1);
    } else if (V >= B200_UNQUANT_MPEG2_INTRA) {
        b.q = P.q_type ? (int)c_nonlinear_qscale[qs & 31] : qs << 1;
    }
    return b;
}

// per coefficient: raster index j of block n (0..5 in its macroblock), matrix entry m, scan position pos.  level is dequantised in
// place; the MPEG-2 mismatch parity of what is stored is xored into parity.
template <int V>
__device__ __forceinline__ void mpv_coef(const UnquantDev &P, const MpvBlock &b, int n, int j, int m, int pos, int &level, int &parity)
{
    using T = MpvVariant<V>;
    if (T::INTRA && j == 0 && !(T::H263 && P.aic)) {
        level = (int)(int16_t)(level * (n < 4 ? P.y_dc : P.c_dc));
        if (T::MISMATCH) parity ^= level & 1;
    }
    if (pos >= (T::INTRA ? 1 : 0) && pos <= b.ncoef && level != 0) {
        int v;
        if (T::H263) v = level < 0 ? level * b.q - b.qadd : level * b.q + b.qadd;
        else         v = dequant<V>(level, b.q, m);
        if (T::MISMATCH) parity ^= v & 1;
        level = (int)(int16_t)v;
    }
}
