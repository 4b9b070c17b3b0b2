// unquant.cu — libavcodec's MPEG-1 / MPEG-2 / H.263-MPEG-4 inverse quantisers on sm_90a (C ABI: "mpegvideo unquantize").
//
// Reference semantics reproduced bit-for-bit (checker: oracle/mpv_oracle.c), libavcodec/mpegvideo_unquantize.c:
//   dct_unquantize_mpeg1_intra_c :50-79     dct_unquantize_mpeg1_inter_c :81-109    dct_unquantize_mpeg2_intra_c :111-140
//   dct_unquantize_mpeg2_intra_bitexact :142-176   dct_unquantize_mpeg2_inter_c :178-211
//   dct_unquantize_h263_intra_c :213-247    dct_unquantize_h263_inter_c :249-276
// i.e. the members of MPVUnquantDSPContext (mpegvideo_unquantize.h:31-44) as ff_mpv_unquantize_init() fills them; they run
// right in front of the IDCT in mpv_reconstruct_mb (put_dct / add_dequant_dct, mpegvideo_dec.c).  Results are stored back
// into int16 with wrap-around like the reference's assignments; the MPEG-2 mismatch control toggles block[63].
//
// Kernel: one warp per 8x8 block, a lane owns two neighbouring coefficients (one 32-bit word, so a warp moves the 128-byte
// block in one transaction each way); "is this coefficient inside the coded part of the scan" is a table look-up of the
// coefficient's scan position; the mismatch parity is one warp xor-reduction.  HBM-bound: 128 B in + 128 B out per block.
#include "common.h"
#include <cstring>

namespace {

constexpr int WARPS = 4;

// [device-code unquant] (tests/cuda_emu runs this block on the CPU against the checker; comment markers only)
// named from include/, a search path of every build of this block: tests/cuda_emu compiles a copy of it from another directory
#include "../ffmpeg_b200/csrc/mpv_unquant.cuh"

template <int V>
__global__ void __launch_bounds__(32 * WARPS)
mpv_unquant_kernel(const __grid_constant__ UnquantDev P, int16_t *blocks, long long nblocks, const uint8_t *blk_n, const uint8_t *qscale,
                   const int8_t *last_index)
{
    const int lane = threadIdx.x & 31;
    // a lane always owns coefficients 2 * lane and 2 * lane + 1: its matrix entries and scan positions are fetched once (32 different
    // constant-bank addresses per warp instruction are served one after the other), then the warp walks over blocks
    int mat[2], spos[2];
#pragma unroll
    for (int k = 0; k < 2; k++) {
        mat[k] = mpv_matrix<V>(P, 2 * lane + k);
        spos[k] = mpv_scanpos<V>(P, 2 * lane + k);
    }
    const long long nwarps = (long long)gridDim.x * WARPS;
    for (long long b = (long long)blockIdx.x * WARPS + (threadIdx.x >> 5); b < nblocks; b += nwarps) {      // whole warps leave together
        const int n = blk_n ? (int)__ldg(blk_n + b) : (int)(b % 6);
        const int qs = __ldg(qscale + b), last = __ldg(last_index + b);
        unsigned *wp = reinterpret_cast<unsigned *>(blocks + 64 * b) + lane;
        const unsigned word = *wp;
        int lv[2] = { (int)(int16_t)(word & 0xffffu), (int)(int16_t)(word >> 16) };
        int parity = 0;
        const MpvBlock blk = mpv_block<V>(P, qs, last);
#pragma unroll
        for (int k = 0; k < 2; k++) mpv_coef<V>(P, blk, n, 2 * lane + k, mat[k], spos[k], lv[k], parity);
        if (MpvVariant<V>::MISMATCH) {
            const unsigned par = __reduce_xor_sync(0xffffffffu, (unsigned)parity);
            if (lane == 31) lv[1] ^= (int)(1u ^ (par & 1u));                    // sum starts at -1: block[63] ^= sum & 1
        }
        *wp = ((unsigned)lv[0] & 0xffffu) | ((unsigned)lv[1] << 16);
    }
}

// [/device-code unquant]
} // namespace

B200_API int b200_mpv_unquantize_batch_device(B200Device *dev, int variant, const B200MpvUnquant *p, int16_t *blocks, int64_t nblocks,
                                              const uint8_t *blk_n, const uint8_t *qscale, const int8_t *last_index)
{
    if (int r = b200_use_device(dev)) return r;
    if (!p || nblocks < 0 || variant < 0 || variant > B200_UNQUANT_H263_INTER) return B200_EINVAL;
    if (nblocks == 0) return 0;
    if (!blocks || !qscale || !last_index || (reinterpret_cast<uintptr_t>(blocks) & 3)) return B200_EINVAL;
    UnquantDev P;
    if (!mpv_unquant_params(p, &P)) { b200_set_error("b200_mpv_unquantize: permutated[] is not a permutation of 0..63"); return B200_EINVAL; }
    long long grid = (nblocks + WARPS - 1) / WARPS;
    const long long cap = (long long)(dev->sm_count > 0 ? dev->sm_count : 132) * 16 * 8;      // persistent warps: each walks nblocks / (grid * WARPS) blocks
    if (grid > cap) grid = cap;
    dim3 g((unsigned)grid), t(32 * WARPS);
    cudaStream_t st = dev->stream;
    switch (variant) {
#define CASE(V) case V: mpv_unquant_kernel<V><<<g, t, 0, st>>>(P, blocks, (long long)nblocks, blk_n, qscale, last_index); break;
    CASE(B200_UNQUANT_MPEG1_INTRA) CASE(B200_UNQUANT_MPEG1_INTER) CASE(B200_UNQUANT_MPEG2_INTRA)
    CASE(B200_UNQUANT_MPEG2_INTRA_BITEXACT) CASE(B200_UNQUANT_MPEG2_INTER) CASE(B200_UNQUANT_H263_INTRA) CASE(B200_UNQUANT_H263_INTER)
#undef CASE
    }
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}
