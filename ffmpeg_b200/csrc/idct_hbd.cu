// idct_hbd.cu — libavcodec's "simple" IDCT at 10 and 12 bit (int16 coefficients, uint16 pixels) on sm_90a.
//
// Reference semantics reproduced bit-for-bit (checker: the 10 / 12 bit part of oracle/idct_oracle.c), libavcodec/simple_idct_template.c:
//   :63-104   constants (10 bit: W3 = 19265, W4 = 16384, ROW_SHIFT 12, COL_SHIFT 19, DC_SHIFT 2; 12 bit: W1..W7 = 45451 ... 9041,
//             ROW_SHIFT 16, COL_SHIFT 17, DC_SHIFT -1)
//   :114-206  idctRowCondDC: rows without AC terms become (row[0] << 2) resp. (row[0] + 1) >> 1, & 0xffff; results back in int16
//   :209-327  IDCT_COLS, idctSparseCol{,Put,Add}; :329-368 ff_simple_idct_{put,add,}_int16_{10,12}bit
// which ff_idctdsp_init installs for bits_per_raw_sample 9, 10 (the 10-bit set) and 12 (idctdsp.c:248-266).  Sums mod 2^32.
//
// The constants of each depth, the row pass and the column sums come from simple_idct.cuh, which the 8-bit kernels (idct.cu) use
// too; this file holds the kernels (how a block is loaded, stored and clipped) and the entry points.
//
// First version, correctness before speed: one thread per 8x8 block, the block held in registers (eight 16-byte loads), row
// pass and column pass fully unrolled.  HBM-bound by bytes (128 B in + 128 B out per block); the 8-bit kernel's staging through
// shared memory (idct.cu) is the model for the tuned version.
#include "common.h"
#include <cstring>

namespace {

// [device-code idct_hbd] (tests/cuda_emu runs this block on the CPU against the checker; comment markers only)
// named from include/, a search path of every build of this block: tests/cuda_emu compiles a copy of it from another directory
#include "../ffmpeg_b200/csrc/simple_idct.cuh"

// KIND 0: in place on the coefficients, 1: put, 2: add.  dest = uint16 pixels; offsets and line sizes in BYTES (even).
template <int DEPTH, int KIND>
__global__ void __launch_bounds__(128)
idct_hbd_kernel(int16_t *blocks, long long n, uint8_t *dest, const int64_t *dest_off, const int32_t *line_size, int uniform_ls)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint4 rows[8];                                        // every row requested before the first row pass branches
    const uint4 *src = reinterpret_cast<const uint4 *>(blocks + 64 * i);
#pragma unroll
    for (int r = 0; r < 8; r++) rows[r] = src[r];
    int v[64];
#pragma unroll
    for (int r = 0; r < 8; r++) row_pass<DEPTH>(rows[r], v + 8 * r);
    constexpr int MAXV = (1 << DEPTH) - 1;
    uint16_t *d = nullptr;
    long long ls = 0;
    if (KIND != 0) {
        d = reinterpret_cast<uint16_t *>(dest + __ldg(dest_off + i));
        ls = (line_size ? __ldg(line_size + i) : uniform_ls) / 2;
    }
#pragma unroll
    for (int c = 0; c < 8; c++) {
        int o[8];
        col_pass<DEPTH>(v[c], v[8 + c], v[16 + c], v[24 + c], v[32 + c], v[40 + c], v[48 + c], v[56 + c], o);
#pragma unroll
        for (int j = 0; j < 8; j++) v[8 * j + c] = o[j];
    }
    if (KIND != 0) {
        // put / add: whole rows (8 samples = 16 bytes) when the rows are 16-byte aligned; for `add` every destination row is loaded
        // before the first store (a load - add - store per sample would make one trip to memory per sample)
        const bool vec = ((reinterpret_cast<uintptr_t>(d) | (uintptr_t)(ls * 2)) & 15) == 0;
        if (vec) {
            uint4 dv[8];
#pragma unroll
            for (int j = 0; j < 8; j++) dv[j] = KIND == 2 ? *reinterpret_cast<const uint4 *>(d + j * ls) : make_uint4(0, 0, 0, 0);
#pragma unroll
            for (int j = 0; j < 8; j++) {
                const unsigned w[4] = { dv[j].x, dv[j].y, dv[j].z, dv[j].w };
                unsigned o2[4];
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const int x0 = v[8 * j + 2 * k] + (int)(w[k] & 0xffffu), x1 = v[8 * j + 2 * k + 1] + (int)(w[k] >> 16);
                    o2[k] = (unsigned)min(max(x0, 0), MAXV) | ((unsigned)min(max(x1, 0), MAXV) << 16);
                }
                *reinterpret_cast<uint4 *>(d + j * ls) = make_uint4(o2[0], o2[1], o2[2], o2[3]);
            }
        } else {
#pragma unroll
            for (int j = 0; j < 8; j++) {                          // unaligned rows: a row at a time
                int dd[8];
#pragma unroll
                for (int k = 0; k < 8; k++) dd[k] = KIND == 2 ? (int)d[j * ls + k] : 0;
#pragma unroll
                for (int k = 0; k < 8; k++) d[j * ls + k] = (uint16_t)min(max(dd[k] + v[8 * j + k], 0), MAXV);
            }
        }
    }
    if (KIND == 0) {
        uint4 *out = reinterpret_cast<uint4 *>(blocks + 64 * i);
#pragma unroll
        for (int r = 0; r < 8; r++) {
            uint4 q;
            q.x = ((unsigned)v[8 * r + 0] & 0xffffu) | ((unsigned)v[8 * r + 1] << 16);
            q.y = ((unsigned)v[8 * r + 2] & 0xffffu) | ((unsigned)v[8 * r + 3] << 16);
            q.z = ((unsigned)v[8 * r + 4] & 0xffffu) | ((unsigned)v[8 * r + 5] << 16);
            q.w = ((unsigned)v[8 * r + 6] & 0xffffu) | ((unsigned)v[8 * r + 7] << 16);
            out[r] = q;
        }
    }
}

// ProresDSPContext.idct_put (libavcodec/proresdsp.c:56-82,102-167): coefficients * qmat (int16 wrap), row pass, 8192 added to the first
// row, in-place column pass (int16), pixels clipped to [4, 2^bits - 5].  VARIANT 110: 10 bit, 12: 12 bit.  One thread per block;
// the coefficient blocks are left untouched (the reference overwrites them).
template <int VARIANT>
__global__ void __launch_bounds__(128)
prores_idct_put_kernel(const int16_t *blocks, long long n, const int16_t *qmat, uint8_t *dest, const int64_t *dest_off, const int32_t *line_size,
                       int uniform_ls)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    unsigned w[32];                                       // the dequantised block as (int16, int16) pairs, all loaded before the row passes
#pragma unroll
    for (int k = 0; k < 32; k++)
        w[k] = ((unsigned)(blocks[64 * i + 2 * k] * qmat[2 * k]) & 0xffffu) | ((unsigned)(blocks[64 * i + 2 * k + 1] * qmat[2 * k + 1]) << 16);
    int v[64];
#pragma unroll
    for (int r = 0; r < 8; r++) row_pass<VARIANT>(make_uint4(w[4 * r], w[4 * r + 1], w[4 * r + 2], w[4 * r + 3]), v + 8 * r);
    constexpr int BITS = VARIANT == 110 ? 10 : 12, LO = 4, HI = (1 << BITS) - 4 - 1;
    uint16_t *d = reinterpret_cast<uint16_t *>(dest + dest_off[i]);
    const long long ls = (line_size ? line_size[i] : uniform_ls) >> 1;
#pragma unroll
    for (int c = 0; c < 8; c++) {
        int o[8];
        v[c] = (int)(int16_t)(v[c] + 8192);
        col_pass<VARIANT>(v[c], v[8 + c], v[16 + c], v[24 + c], v[32 + c], v[40 + c], v[48 + c], v[56 + c], o);
#pragma unroll
        for (int j = 0; j < 8; j++) d[j * ls + c] = (uint16_t)min(max((int)(int16_t)o[j], LO), HI);
    }
}
// [/device-code idct_hbd]

template <int DEPTH>
int launch(cudaStream_t st, int kind, int16_t *blocks, long long n, uint8_t *dest, const int64_t *off, const int32_t *ls, int uls)
{
    const long long grid = (n + 127) / 128;
    if (grid > 0x7fffffffLL) return B200_EINVAL;
    dim3 g((unsigned)grid), t(128);
    if (kind == B200_IDCT)          idct_hbd_kernel<DEPTH, 0><<<g, t, 0, st>>>(blocks, n, dest, off, ls, uls);
    else if (kind == B200_IDCT_PUT) idct_hbd_kernel<DEPTH, 1><<<g, t, 0, st>>>(blocks, n, dest, off, ls, uls);
    else                            idct_hbd_kernel<DEPTH, 2><<<g, t, 0, st>>>(blocks, n, dest, off, ls, uls);
    B200_LAUNCHED();
    return 0;
}

void die(const char *what)
{
    fprintf(stderr, "libb200dsp: high-bit-depth idct failed: %s (%s)\n", what, b200_last_error());
    abort();
}

// drop-in: one block through the device (host pointers); put / add leave the caller's coefficient block as it was (the
// reference uses it as scratch; no caller reads it afterwards)
template <int DEPTH>
void host_op(int kind, uint8_t *dest, ptrdiff_t line_size, int16_t *block)
{
    B200Device *dev = b200_default_device();
    if (!dev) die("no device");
    if (kind != B200_IDCT && ((line_size > -16 && line_size < 16) || (line_size & 1))) die("|line_size| must be even and >= 16 bytes");
    if (cudaSetDevice(dev->ordinal) != cudaSuccess) die("cudaSetDevice");
    B200_LOCK_DEVICE(dev);      // scratch + stream are per device: one host-pointer call at a time (released on return)
    uint8_t *scr = (uint8_t *)b200_scratch(dev, 128 + 8 * 16 + 16);
    if (!scr) die("scratch");
    int16_t *dblk = (int16_t *)scr;
    uint8_t *ddst = scr + 128;
    int64_t *doff = (int64_t *)(scr + 128 + 128);
    cudaStream_t st = dev->stream;
    const int64_t zero = 0;
    if (cudaMemcpyAsync(dblk, block, 128, cudaMemcpyHostToDevice, st) != cudaSuccess) die("h2d block");
    if (kind != B200_IDCT) {
        if (kind == B200_IDCT_ADD && b200_h2d_rows(ddst, 16, dest, line_size, 16, 8, st) != cudaSuccess) die("h2d dest");
        if (cudaMemcpyAsync(doff, &zero, 8, cudaMemcpyHostToDevice, st) != cudaSuccess) die("h2d off");
    }
    if (launch<DEPTH>(st, kind, dblk, 1, ddst, doff, nullptr, 16) < 0 || cudaGetLastError() != cudaSuccess) die("launch");
    if (kind == B200_IDCT) { if (cudaMemcpyAsync(block, dblk, 128, cudaMemcpyDeviceToHost, st) != cudaSuccess) die("d2h block"); }
    else if (b200_d2h_rows(dest, line_size, ddst, 16, 16, 8, st) != cudaSuccess) die("d2h dest");
    if (cudaStreamSynchronize(st) != cudaSuccess) die("sync");
}

template <int DEPTH> void tab_idct(int16_t *b) { host_op<DEPTH>(B200_IDCT, nullptr, 0, b); }
template <int DEPTH> void tab_put(uint8_t *d, ptrdiff_t ls, int16_t *b) { host_op<DEPTH>(B200_IDCT_PUT, d, ls, b); }
template <int DEPTH> void tab_add(uint8_t *d, ptrdiff_t ls, int16_t *b) { host_op<DEPTH>(B200_IDCT_ADD, d, ls, b); }

} // namespace

B200_API int b200_idctdsp_init_hbd(B200IDCTDSPContext *c, int idct_algo, int bits_per_raw_sample, int lowres)
{
    if (!c) return B200_EINVAL;
    // ff_idctdsp_init, libavcodec/idctdsp.c:248-266: 9 and 10 bit -> the int16 10-bit functions, 12 bit -> the 12-bit ones
    const int depth = bits_per_raw_sample == 9 ? 10 : bits_per_raw_sample;
    if (lowres != 0 || (depth != 10 && depth != 12) || (idct_algo != 0 && idct_algo != 2)) return B200_ENOSYS;
    int ret = b200_idctdsp_init(c, idct_algo, 8, 0);          // the three clamp helpers stay the 8-bit ones, as in the reference
    if (ret < 0) return ret;
    if (depth == 10) { c->idct = tab_idct<10>; c->idct_put = tab_put<10>; c->idct_add = tab_add<10>; }
    else             { c->idct = tab_idct<12>; c->idct_put = tab_put<12>; c->idct_add = tab_add<12>; }
    return 0;
}

B200_API int b200_idct_hbd_batch_device(B200Device *dev, int depth, int kind, int16_t *blocks, int64_t nblocks, uint8_t *dest,
                                        const int64_t *dest_off, const int32_t *line_size, int uniform_line_size)
{
    if (!dev) dev = b200_default_device();
    if (!dev) return B200_ENODEV;
    if (depth == 9) depth = 10;
    if ((depth != 10 && depth != 12) || kind < B200_IDCT || kind > B200_IDCT_ADD || nblocks < 0) return B200_EINVAL;
    if (nblocks == 0) return 0;
    if (!blocks || (reinterpret_cast<uintptr_t>(blocks) & 15)) return B200_EINVAL;
    if (kind != B200_IDCT && (!dest || !dest_off || (reinterpret_cast<uintptr_t>(dest) & 1) || (!line_size && (uniform_line_size & 1))))
        return B200_EINVAL;
    B200_CUDA_OK(cudaSetDevice(dev->ordinal));
    const int ret = depth == 10 ? launch<10>(dev->stream, kind, blocks, nblocks, dest, dest_off, line_size, uniform_line_size)
                                : launch<12>(dev->stream, kind, blocks, nblocks, dest, dest_off, line_size, uniform_line_size);
    if (ret < 0) return ret;
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

// ---- ProresDSPContext (libavcodec/proresdsp.h:28-35, ff_proresdsp_init proresdsp.c:169-194)
namespace {

int launch_prores(cudaStream_t st, int bits, const int16_t *blocks, long long n, const int16_t *qmat, uint8_t *dest, const int64_t *off,
                  const int32_t *ls, int uls)
{
    const long long grid = (n + 127) / 128;
    if (grid > 0x7fffffffLL) return B200_EINVAL;
    if (bits == 10) prores_idct_put_kernel<110><<<(unsigned)grid, 128, 0, st>>>(blocks, n, qmat, dest, off, ls, uls);
    else            prores_idct_put_kernel<12><<<(unsigned)grid, 128, 0, st>>>(blocks, n, qmat, dest, off, ls, uls);
    B200_LAUNCHED();
    return 0;
}

template <int BITS>
void prores_tab_put(uint16_t *out, ptrdiff_t linesize, int16_t *block, const int16_t *qmat)
{
    B200Device *dev = b200_default_device();
    if (!dev) die("no device");
    if ((linesize > -16 && linesize < 16) || (linesize & 1)) die("|line size| must be even and >= 16 bytes");
    if (cudaSetDevice(dev->ordinal) != cudaSuccess) die("cudaSetDevice");
    B200_LOCK_DEVICE(dev);      // scratch + stream are per device: one host-pointer call at a time (released on return)
    uint8_t *scr = (uint8_t *)b200_scratch(dev, 128 + 128 + 128 + 16);
    if (!scr) die("scratch");
    int16_t *dblk = (int16_t *)scr, *dq = (int16_t *)(scr + 128);
    uint8_t *ddst = scr + 256;
    int64_t *doff = (int64_t *)(scr + 384);
    cudaStream_t st = dev->stream;
    const int64_t zero = 0;
    if (cudaMemcpyAsync(dblk, block, 128, cudaMemcpyHostToDevice, st) != cudaSuccess) die("h2d block");
    if (cudaMemcpyAsync(dq, qmat, 128, cudaMemcpyHostToDevice, st) != cudaSuccess) die("h2d qmat");
    if (cudaMemcpyAsync(doff, &zero, 8, cudaMemcpyHostToDevice, st) != cudaSuccess) die("h2d off");
    if (launch_prores(st, BITS, dblk, 1, dq, ddst, doff, nullptr, 16) < 0 || cudaGetLastError() != cudaSuccess) die("launch");
    if (b200_d2h_rows(out, linesize, ddst, 16, 16, 8, st) != cudaSuccess) die("d2h");
    if (cudaStreamSynchronize(st) != cudaSuccess) die("sync");
}

} // namespace

B200_API int b200_proresdsp_init(B200ProresDSPContext *c, int bits_per_raw_sample)
{
    if (!c) return B200_EINVAL;
    if (bits_per_raw_sample != 10 && bits_per_raw_sample != 12) return B200_ENOSYS;
    if (!b200_default_device()) return B200_ENODEV;
    memset(c, 0, sizeof(*c));
    c->idct_permutation_type = 0;                                    // FF_IDCT_PERM_NONE
    for (int i = 0; i < 64; i++) c->idct_permutation[i] = (uint8_t)i;
    c->idct_put = bits_per_raw_sample == 10 ? prores_tab_put<10> : prores_tab_put<12>;
    c->idct_put_bayer = nullptr;                                     // ProRes RAW (32-bit coefficients + linearisation curve): not built
    return 0;
}

B200_API int b200_prores_idct_put_batch_device(B200Device *dev, int bits, const int16_t *blocks, int64_t nblocks, const int16_t *qmat,
                                               uint8_t *dest, const int64_t *dest_off, const int32_t *line_size, int uniform_line_size)
{
    if (!dev) dev = b200_default_device();
    if (!dev) return B200_ENODEV;
    if ((bits != 10 && bits != 12) || nblocks < 0) return B200_EINVAL;
    if (nblocks == 0) return 0;
    if (!blocks || !qmat || !dest || !dest_off || (reinterpret_cast<uintptr_t>(dest) & 1) || (!line_size && (uniform_line_size & 1))) return B200_EINVAL;
    B200_CUDA_OK(cudaSetDevice(dev->ordinal));
    const int ret = launch_prores(dev->stream, bits, blocks, nblocks, qmat, dest, dest_off, line_size, uniform_line_size);
    if (ret < 0) return ret;
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}
