// h264idct.cu — libavcodec H.264 residual transforms on sm_90a for 8, 9, 10, 12 and 14 bit samples: idct_add / idct8_add / idct_dc_add /
// idct8_dc_add of H264DSPContext as ff_h264dsp_init(c, depth, ...) installs them (libavcodec/h264dsp.c:66-158) (C ABI: "h264 residual").
//
// Reference semantics reproduced bit-for-bit (checker: oracle/idct_oracle.c):
//   ff_h264_idct_add_<depth>_c      libavcodec/h264idct_template.c:33-70     4x4, result added to dst, coefficients cleared
//   ff_h264_idct8_add_<depth>_c     libavcodec/h264idct_template.c:72-145    8x8
//   ff_h264_idct_dc_add_<depth>_c / ff_h264_idct8_dc_add_<depth>_c   :147-181   DC-only blocks
// dctcoef is int16_t with uint8 samples at 8 bits, int32_t with uint16 samples above.  The first pass and the + 32 on the DC coefficient
// write back into dctcoef (an int16 store wraps), sums are mod 2^32 (SUINT): both are kept.  The sum >> 6 is clipped to the sample depth.
//
// Batched kernel: one thread per block.  Every consumed coefficient block is zeroed like the reference's memset (the decoder relies on
// it for the next macroblock).  8 bit: 32 / 128 bytes of coefficients in 16-byte accesses, destination rows as 4- / 8-byte words (the
// reference requires dst 4-aligned, h264dsp.h:81).  16 bit: coefficients one by one (the 16-bit entry takes 4-byte-aligned blocks), a
// destination row in one 8- / 16-byte access where dst and stride allow it, else sample by sample.
#include "common.h"
#include <cstring>
#include <type_traits>

namespace {

template <typename P> using dctcoef = std::conditional_t<sizeof(P) == 1, int16_t, int32_t>;

// a store into dctcoef, read back
template <typename P> __device__ __forceinline__ int coef(unsigned v) { return (int)(dctcoef<P>)v; }

// a destination row of N samples: 4-byte words, accessed as one unsigned / uint2 / uint4
template <int WORDS> struct RowVec;
template <> struct RowVec<1> { using T = unsigned; };
template <> struct RowVec<2> { using T = uint2; };
template <> struct RowVec<4> { using T = uint4; };

// clipped samples of the word d plus the residuals v[] (four uint8 or two uint16 samples)
__device__ __forceinline__ unsigned add_word(unsigned d, const int *v, int, uint8_t)
{
    const unsigned p0 = (unsigned)__vimin_s32_relu((int)__byte_perm(d, 0, 0x4440) + v[0], 255);
    const unsigned p1 = (unsigned)__vimin_s32_relu((int)__byte_perm(d, 0, 0x4441) + v[1], 255);
    const unsigned p2 = (unsigned)__vimin_s32_relu((int)__byte_perm(d, 0, 0x4442) + v[2], 255);
    const unsigned p3 = (unsigned)__vimin_s32_relu((int)(d >> 24) + v[3], 255);
    return __byte_perm(__byte_perm(p0, p1, 0x1140), __byte_perm(p2, p3, 0x1140), 0x5410);
}
__device__ __forceinline__ unsigned add_word(unsigned d, const int *v, int maxv, uint16_t)
{
    return (unsigned)__vimin_s32_relu((int)(d & 0xffff) + v[0], maxv) | (unsigned)__vimin_s32_relu((int)(d >> 16) + v[1], maxv) << 16;
}

__device__ __forceinline__ void idct8_1d(const int *in, unsigned *out)
{
    const unsigned a0 = in[0] + (unsigned)in[4], a2 = in[0] - (unsigned)in[4];
    const unsigned a4 = (in[2] >> 1) - (unsigned)in[6], a6 = (in[6] >> 1) + (unsigned)in[2];
    const unsigned b0 = a0 + a6, b2 = a2 + a4, b4 = a2 - a4, b6 = a0 - a6;
    const int a1 = (int)(-(unsigned)in[3] + (unsigned)in[5] - (unsigned)in[7] - (unsigned)(in[7] >> 1));
    const int a3 = (int)((unsigned)in[1] + (unsigned)in[7] - (unsigned)in[3] - (unsigned)(in[3] >> 1));
    const int a5 = (int)(-(unsigned)in[1] + (unsigned)in[7] + (unsigned)in[5] + (unsigned)(in[5] >> 1));
    const int a7 = (int)((unsigned)in[3] + (unsigned)in[5] + (unsigned)in[1] + (unsigned)(in[1] >> 1));
    const unsigned b1 = (unsigned)(a7 >> 2) + (unsigned)a1, b3 = (unsigned)a3 + (unsigned)(a5 >> 2);
    const unsigned b5 = (unsigned)(a3 >> 2) - (unsigned)a5, b7 = (unsigned)a7 - (unsigned)(a1 >> 2);
    out[0] = b0 + b7; out[7] = b0 - b7; out[1] = b2 + b5; out[6] = b2 - b5;
    out[2] = b4 + b3; out[5] = b4 - b3; out[3] = b6 + b1; out[4] = b6 - b1;
}

// kind 0: 4x4, 1: 8x8, 2: 4x4 DC only, 3: 8x8 DC only.  P = uint8_t (depth 8) or uint16_t (9 / 10 / 12 / 14).  blk_off in coefficients
// (multiples of 8 at 8 bits: blocks are 16-byte aligned), dst_off and stride in bytes.
template <typename P, int KIND>
__global__ void __launch_bounds__(128)
h264_idct_kernel(long long n, dctcoef<P> *blocks, const int64_t *blk_off, uint8_t *dst, const int64_t *dst_off, long long stride, int depth)
{
    constexpr int N = (KIND & 1) ? 8 : 4, NC = N * N, SPW = 4 / sizeof(P), WORDS = N / SPW;     // samples per word, words per row
    using Row = typename RowVec<WORDS>::T;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    dctcoef<P> *b = blocks + __ldg(blk_off + i);
    uint8_t *d = dst + __ldg(dst_off + i);
    const int maxv = sizeof(P) == 1 ? 255 : (1 << depth) - 1;
    // a row in one access; the 8-bit entry guarantees the alignment, at 16 bits a misaligned row goes sample by sample
    const bool vec = sizeof(P) == 1 || ((reinterpret_cast<uintptr_t>(d) | (uintptr_t)stride) % sizeof(Row)) == 0;
    // every destination row is requested before the first store: written row by row (load, add, store) each row's load would sit
    // behind the previous row's store in program order and the thread would make one trip to memory per row (ncu: 138 warps stalled
    // on the long scoreboard per issue with the memory system at 15 %)
    unsigned dv[N][WORDS];
    auto load_rows = [&] {
#pragma unroll
        for (int r = 0; r < N; r++) {
            if (vec) {
                const Row v = *reinterpret_cast<const Row *>(d + r * stride);
                memcpy(dv[r], &v, sizeof(Row));
            } else {
                const P *p = reinterpret_cast<const P *>(d + r * stride);
#pragma unroll
                for (int k = 0; k < WORDS; k++) dv[r][k] = p[2 * k] | (unsigned)p[2 * k + 1] << 16;
            }
        }
    };
    auto store_rows = [&](const int (*res)[N]) {
#pragma unroll
        for (int r = 0; r < N; r++) {
#pragma unroll
            for (int k = 0; k < WORDS; k++) dv[r][k] = add_word(dv[r][k], res[r] + SPW * k, maxv, P());
            if (vec) {
                Row v;
                memcpy(&v, dv[r], sizeof(Row));
                *reinterpret_cast<Row *>(d + r * stride) = v;
            } else {
                P *p = reinterpret_cast<P *>(d + r * stride);
#pragma unroll
                for (int k = 0; k < WORDS; k++) { p[2 * k] = (P)dv[r][k]; p[2 * k + 1] = (P)(dv[r][k] >> 16); }
            }
        }
    };
    int res[N][N];                                              // res[row][column]: what is added to the sample
    if (KIND >= 2) {
        const int dc = (int)((unsigned)b[0] + 32u) >> 6;
        load_rows();
        b[0] = 0;
#pragma unroll
        for (int r = 0; r < N; r++)
#pragma unroll
            for (int x = 0; x < N; x++) res[r][x] = dc;
        store_rows(res);
        return;
    }
    int c[NC];
    if (sizeof(P) == 1) {
        uint4 q[NC / 8];
        uint4 *bp = reinterpret_cast<uint4 *>(b);
#pragma unroll
        for (int k = 0; k < NC / 8; k++) q[k] = bp[k];
        load_rows();
#pragma unroll
        for (int k = 0; k < NC / 8; k++) {
            bp[k] = make_uint4(0, 0, 0, 0);
            const unsigned w[4] = { q[k].x, q[k].y, q[k].z, q[k].w };
#pragma unroll
            for (int j = 0; j < 4; j++) { c[8 * k + 2 * j] = coef<P>(w[j]); c[8 * k + 2 * j + 1] = (int)w[j] >> 16; }
        }
    } else {
#pragma unroll
        for (int k = 0; k < NC; k++) c[k] = b[k];
        load_rows();
#pragma unroll
        for (int k = 0; k < NC; k++) b[k] = 0;
    }
    c[0] = coef<P>((unsigned)(c[0] + 32));                      // block[0] += 1 << 5
    if (KIND == 0) {
#pragma unroll
        for (int x = 0; x < 4; x++) {
            const unsigned z0 = c[x] + (unsigned)c[x + 8], z1 = c[x] - (unsigned)c[x + 8];
            const unsigned z2 = (c[x + 4] >> 1) - (unsigned)c[x + 12], z3 = c[x + 4] + (unsigned)(c[x + 12] >> 1);
            c[x] = coef<P>(z0 + z3); c[x + 4] = coef<P>(z1 + z2); c[x + 8] = coef<P>(z1 - z2); c[x + 12] = coef<P>(z0 - z3);
        }
#pragma unroll
        for (int x = 0; x < 4; x++) {
            const unsigned z0 = c[4 * x] + (unsigned)c[2 + 4 * x], z1 = c[4 * x] - (unsigned)c[2 + 4 * x];
            const unsigned z2 = (c[1 + 4 * x] >> 1) - (unsigned)c[3 + 4 * x], z3 = c[1 + 4 * x] + (unsigned)(c[3 + 4 * x] >> 1);
            res[0][x] = (int)(z0 + z3) >> 6; res[1][x] = (int)(z1 + z2) >> 6; res[2][x] = (int)(z1 - z2) >> 6; res[3][x] = (int)(z0 - z3) >> 6;
        }
    } else {
#pragma unroll
        for (int x = 0; x < 8; x++) {
            int in[8]; unsigned out[8];
#pragma unroll
            for (int k = 0; k < 8; k++) in[k] = c[x + 8 * k];
            idct8_1d(in, out);
#pragma unroll
            for (int k = 0; k < 8; k++) c[x + 8 * k] = coef<P>(out[k]);
        }
#pragma unroll
        for (int x = 0; x < 8; x++) {
            int in[8]; unsigned out[8];
#pragma unroll
            for (int k = 0; k < 8; k++) in[k] = c[k + 8 * x];
            idct8_1d(in, out);
#pragma unroll
            for (int k = 0; k < 8; k++) res[k][x] = (int)out[k] >> 6;
        }
    }
    store_rows(res);
}

template <typename P>
int launch(cudaStream_t st, int kind, int depth, long long n, dctcoef<P> *blocks, const int64_t *blk_off, uint8_t *dst, const int64_t *dst_off,
           long long stride)
{
    const long long ctas = (n + 127) / 128;
    if (ctas > 0x7fffffffLL) return B200_EINVAL;
    const unsigned g = (unsigned)ctas;
    switch (kind) {
    case 0: h264_idct_kernel<P, 0><<<g, 128, 0, st>>>(n, blocks, blk_off, dst, dst_off, stride, depth); break;
    case 1: h264_idct_kernel<P, 1><<<g, 128, 0, st>>>(n, blocks, blk_off, dst, dst_off, stride, depth); break;
    case 2: h264_idct_kernel<P, 2><<<g, 128, 0, st>>>(n, blocks, blk_off, dst, dst_off, stride, depth); break;
    default: h264_idct_kernel<P, 3><<<g, 128, 0, st>>>(n, blocks, blk_off, dst, dst_off, stride, depth); break;
    }
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

// drop-in: one block through the device (host pointers; above 8 bits `block` holds int32 coefficients behind the reference's int16_t * type)
template <int DEPTH, int KIND>
void host_fn(uint8_t *dst, int16_t *block16, ptrdiff_t stride)
{
    using P = std::conditional_t<DEPTH == 8, uint8_t, uint16_t>;
    constexpr int N = (KIND & 1) ? 8 : 4, NC = N * N;
    dctcoef<P> *block = reinterpret_cast<dctcoef<P> *>(block16);
    constexpr size_t CB = 64 * sizeof(dctcoef<P>);                // coefficients of an 8x8 block
    B200HostCall call("h264 idct", nullptr, CB + 256);
    uint8_t *scr = call.scratch;
    dctcoef<P> *dblk = (dctcoef<P> *)scr;
    uint8_t *dpix = scr + CB;                                      // N rows, pitch 16 bytes
    int64_t *meta = (int64_t *)(scr + CB + 128);
    cudaStream_t st = call.stream;
    const int64_t m[2] = { 0, 0 };
    call.check(cudaMemcpyAsync(dblk, block, (KIND >= 2 ? 1 : NC) * sizeof(dctcoef<P>), cudaMemcpyHostToDevice, st), "h2d block");
    call.check(b200_h2d_rows(dpix, 16, dst, stride, N * sizeof(P), N, st), "h2d dst");
    call.check(cudaMemcpyAsync(meta, m, sizeof(m), cudaMemcpyHostToDevice, st), "h2d meta");
    call.launched(launch<P>(st, KIND, DEPTH, 1, dblk, meta, dpix, meta + 1, 16));
    call.check(b200_d2h_rows(dst, stride, dpix, 16, N * sizeof(P), N, st), "d2h");
    call.sync();
    if (KIND >= 2) block[0] = 0; else memset(block, 0, NC * sizeof(dctcoef<P>));     // what the reference leaves behind
}

template <int DEPTH>
void fill(B200H264IDCTContext *c)
{
    c->idct_add = host_fn<DEPTH, 0>; c->idct8_add = host_fn<DEPTH, 1>; c->idct_dc_add = host_fn<DEPTH, 2>; c->idct8_dc_add = host_fn<DEPTH, 3>;
}

} // namespace

B200_API int b200_h264_idct_init(B200H264IDCTContext *c, int bit_depth, int chroma_format_idc)
{
    (void)chroma_format_idc;
    if (!c) return B200_EINVAL;
    if (!b200_default_device()) return B200_ENODEV;
    switch (bit_depth) {                                           // h264dsp.c:139-158
    case 8:  fill<8>(c);  return 0;
    case 9:  fill<9>(c);  return 0;
    case 10: fill<10>(c); return 0;
    case 12: fill<12>(c); return 0;
    case 14: fill<14>(c); return 0;
    }
    return B200_ENOSYS;
}

B200_API int b200_h264_idct_batch_device(B200Device *dev, int kind, int64_t n, int16_t *blocks, const int64_t *blk_off,
                                         uint8_t *dst, const int64_t *dst_off, ptrdiff_t stride)
{
    if (!dev || n < 0 || !blocks || !blk_off || !dst || !dst_off || kind < 0 || kind > 3) return B200_EINVAL;
    if (((uintptr_t)blocks & 15) || ((uintptr_t)dst & ((kind & 1) ? 7 : 3)) || (stride & ((kind & 1) ? 7 : 3))) return B200_EINVAL;
    if (n == 0) return 0;
    if (int r = b200_use_device(dev)) return r;
    return launch<uint8_t>(dev->stream, kind, 8, n, blocks, blk_off, dst, dst_off, (long long)stride);
}

B200_API int b200_h264_idct_hbd_batch_device(B200Device *dev, int bit_depth, int kind, int64_t n, int32_t *blocks, const int64_t *blk_off,
                                             uint8_t *dst, const int64_t *dst_off, ptrdiff_t stride)
{
    if (!dev || n < 0 || !blocks || !blk_off || !dst || !dst_off || kind < 0 || kind > 3) return B200_EINVAL;
    if (bit_depth != 9 && bit_depth != 10 && bit_depth != 12 && bit_depth != 14) return B200_ENOSYS;
    if (((uintptr_t)blocks & 3) || ((uintptr_t)dst & 1) || (stride & 1)) return B200_EINVAL;
    if (n == 0) return 0;
    if (int r = b200_use_device(dev)) return r;
    return launch<uint16_t>(dev->stream, kind, bit_depth, n, blocks, blk_off, dst, dst_off, (long long)stride);
}
