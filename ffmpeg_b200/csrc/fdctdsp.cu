// fdctdsp.cu — FDCTDSPContext (libavcodec/fdctdsp.h:28-31) as ff_fdctdsp_init fills it (libavcodec/fdctdsp.c:27-45):
//   fdct / fdct248 = ff_jpeg_fdct_islow_8 / ff_fdct248_islow_8     jfdctint_template.c:173-412 with BIT_DEPTH 8 (default)
//                    ff_jpeg_fdct_islow_10 / ff_fdct248_islow_10   the same template with BIT_DEPTH 10 (bits_per_raw_sample 9 or 10)
//                    ff_fdct_ifast / ff_fdct_ifast248              jfdctfst.c:140-343 (dct_algo FF_DCT_FASTINT)
// FF_DCT_FAAN (floating point) is not built: b200_fdctdsp_init refuses it and the caller keeps the C functions.
//
// Work split: eight lanes per 8x8 block (four blocks per warp), a lane holds one row in registers (one 16-byte load), row pass, 8x8 transpose
// with xor-shuffles (fdct_dev.cuh), column pass, transpose back, one 16-byte store.  16 + 16 bytes of HBM traffic per row, nothing staged.
#include "common.h"
#include "fdct_dev.cuh"

namespace {

// kind: 0 islow 8-bit, 1 ifast, 2 islow 10-bit; +4: the 2-4-8 column pass
__global__ void __launch_bounds__(256)
fdct_kernel(int kind, int16_t *blocks, long long n)
{
    const long long b = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
    const int row = threadIdx.x & 7;
    const bool on = b < n;                                         // idle lane groups transform zeros: every lane takes part in the shuffles
    int v[8];
    uint4 *p = reinterpret_cast<uint4 *>(blocks + (on ? b : 0) * 64 + row * 8);
    {
        const uint4 q = on ? *p : make_uint4(0, 0, 0, 0);
        const unsigned w[4] = { q.x, q.y, q.z, q.w };
#pragma unroll
        for (int k = 0; k < 4; k++) { v[2 * k] = (int)(short)(w[k] & 0xffff); v[2 * k + 1] = (int)w[k] >> 16; }
    }
    const int algo = kind & 3;
    if (algo == 1) fdct_fast8(v); else if (algo == 2) fdct_slow8<false, 1, 2>(v); else fdct_slow8<false, 4, 4>(v);
    transpose8(v, row);
    if (kind & 4) { if (algo == 1) fdct248_fast8(v); else if (algo == 2) fdct248_slow8<2>(v); else fdct248_slow8<4>(v); }
    else          { if (algo == 1) fdct_fast8(v); else if (algo == 2) fdct_slow8<true, 1, 2>(v); else fdct_slow8<true, 4, 4>(v); }
    transpose8(v, row);
    if (on) {
        uint4 q;
        q.x = (unsigned)(v[0] & 0xffff) | ((unsigned)v[1] << 16); q.y = (unsigned)(v[2] & 0xffff) | ((unsigned)v[3] << 16);
        q.z = (unsigned)(v[4] & 0xffff) | ((unsigned)v[5] << 16); q.w = (unsigned)(v[6] & 0xffff) | ((unsigned)v[7] << 16);
        *p = q;
    }
}

int kind_of(int dct_algo, int bits_per_raw_sample)
{
    if (bits_per_raw_sample == 10 || bits_per_raw_sample == 9) return 2;      // fdctdsp.c:29-31: the depth is looked at first
    if (dct_algo == 1) return 1;                                               // FF_DCT_FASTINT
    if (dct_algo == 6) return -1;                                              // FF_DCT_FAAN
    return 0;
}

template <int KIND>
void host_fdct(int16_t *block)
{
    B200HostCall call("fdct", nullptr, 128);
    int16_t *scr = (int16_t *)call.scratch;
    call.check(cudaMemcpyAsync(scr, block, 128, cudaMemcpyHostToDevice, call.stream), "h2d");
    fdct_kernel<<<1, 32, 0, call.stream>>>(KIND, scr, 1);
    B200_LAUNCHED();
    call.launched();
    call.check(cudaMemcpyAsync(block, scr, 128, cudaMemcpyDeviceToHost, call.stream), "d2h");
    call.sync();
}

} // namespace

B200_API int b200_fdctdsp_init(B200FDCTDSPContext *c, int dct_algo, int bits_per_raw_sample)
{
    if (!c) return B200_EINVAL;
    if (!b200_default_device()) return B200_ENODEV;
    const int kind = kind_of(dct_algo, bits_per_raw_sample);
    if (kind < 0) { b200_set_error("fdctdsp: FF_DCT_FAAN is not implemented"); return B200_ENOSYS; }
    if (kind == 0) { c->fdct = host_fdct<0>; c->fdct248 = host_fdct<4>; }
    else if (kind == 1) { c->fdct = host_fdct<1>; c->fdct248 = host_fdct<5>; }
    else { c->fdct = host_fdct<2>; c->fdct248 = host_fdct<6>; }
    return 0;
}

B200_API int b200_fdct_batch_device(B200Device *dev, int dct_algo, int bits_per_raw_sample, int is248, int16_t *blocks, int64_t n)
{
    if (int r = b200_use_device(dev)) return r;
    if (!blocks || n < 0 || ((uintptr_t)blocks & 15)) return B200_EINVAL;
    const int kind = kind_of(dct_algo, bits_per_raw_sample);
    if (kind < 0) { b200_set_error("fdctdsp: FF_DCT_FAAN is not implemented"); return B200_ENOSYS; }
    if (n == 0) return 0;
    const long long ctas = (n + 31) / 32;                          // 256 threads = 32 blocks of 8 lanes
    if (ctas > 0x7fffffffLL) return B200_EINVAL;
    fdct_kernel<<<(unsigned)ctas, 256, 0, dev->stream>>>(kind | (is248 ? 4 : 0), blocks, n);
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}
