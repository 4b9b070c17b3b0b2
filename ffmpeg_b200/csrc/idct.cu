// idct.cu — libavcodec idctdsp (8-bit "simple" IDCT) on sm_90a: kernels + the C ABI (include/b200dsp.h, "idctdsp").
//
// Reference semantics reproduced bit-for-bit (checker: oracle/idct_oracle.c):
//   idctRowCondDC            libavcodec/simple_idct_template.c:114-206
//   idctSparseCol{,Put,Add}  libavcodec/simple_idct_template.c:209-327
//   ff_simple_idct_{put,add,}_int16_8bit  :329-368
//   put/put_signed/add_pixels_clamped     libavcodec/idctdsp.c:73-165
//
// Mapping: 8 lanes cooperate on one 8x8 block, lane r owns row r.  A warp therefore reads 4 consecutive blocks =
// 512 contiguous bytes with one 128-bit load per lane (fully coalesced), runs the row pass in registers, transposes
// the 8x8 int16 tile with warp shuffles (3 butterfly stages: lane^4, lane^2, lane^1), runs the column pass, transposes
// back and writes one 8-byte destination row per lane.  No shared memory, no re-reads: HBM traffic is the algorithmic
// 128 B in + 64 B out (+64 B dest read for add) per block.
#include "common.h"
#include <cstring>

namespace {

#include "simple_idct.cuh"
#include "mpv_unquant.cuh"

// 8x8 transpose of 16-bit elements held as 4 packed words per lane by groups of 8 lanes.
__device__ __forceinline__ void transpose8x8(unsigned q[4], int lane)
{
    const unsigned full = 0xffffffffu;
    {   // 4x4 blocks between lane and lane^4
        const bool up = lane & 4;
        unsigned s0 = up ? q[0] : q[2], s1 = up ? q[1] : q[3];
        s0 = __shfl_xor_sync(full, s0, 4); s1 = __shfl_xor_sync(full, s1, 4);
        if (up) { q[0] = s0; q[1] = s1; } else { q[2] = s0; q[3] = s1; }
    }
    {   // 2x2 blocks between lane and lane^2
        const bool up = lane & 2;
        unsigned s0 = up ? q[0] : q[1], s1 = up ? q[2] : q[3];
        s0 = __shfl_xor_sync(full, s0, 2); s1 = __shfl_xor_sync(full, s1, 2);
        if (up) { q[0] = s0; q[2] = s1; } else { q[1] = s0; q[3] = s1; }
    }
    {   // single elements between lane and lane^1
        const bool odd = lane & 1;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const unsigned o = __shfl_xor_sync(full, q[k], 1);
            q[k] = odd ? __byte_perm(o, q[k], 0x7632) : __byte_perm(q[k], o, 0x5410);
        }
    }
}

__device__ __forceinline__ unsigned clip4(int a, int b, int c, int d)
{
    return (unsigned)min(max(a, 0), 255) | ((unsigned)min(max(b, 0), 255) << 8) |
           ((unsigned)min(max(c, 0), 255) << 16) | ((unsigned)min(max(d, 0), 255) << 24);
}

struct Mb420Geom {                 // implied destinations of a 4:2:0 macroblock stream
    int mb_w, mb_h;
    uint8_t *plane[3]; int linesize[3]; long long frame_stride[3];
};

// KIND: B200_IDCT / _PUT / _ADD.  MB420: destinations implied by the block index, else dest_off/line_size arrays.
template <int KIND, bool MB420>
__global__ void __launch_bounds__(256)
idct8x8_kernel(const int16_t *blocks, int16_t *blocks_out, long long nblocks,
               uint8_t *dest, const int64_t *__restrict__ dest_off, const int32_t *__restrict__ line_size,
               int uniform_ls, Mb420Geom g)
{
    const int lane = threadIdx.x & 31;
    const int row = lane & 7;
    const long long warp = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const long long blk = warp * 4 + (lane >> 3);
    const bool live = blk < nblocks;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (live) {
        const uint4 *src = reinterpret_cast<const uint4 *>(blocks) + blk * 8 + row;
        v = KIND == B200_IDCT ? *src : __ldg(src);   // in-place variant must not use the read-only path
    }
    unsigned q[4];
    row_pass<8>(v, q);
    transpose8x8(q, lane);        // lane now owns column `row`
    {
        int o[8];
        col_pass<8>(sx_lo(q[0]), sx_hi(q[0]), sx_lo(q[1]), sx_hi(q[1]), sx_lo(q[2]), sx_hi(q[2]), sx_lo(q[3]), sx_hi(q[3]), o);
        // results fit in 12 bits signed, so packing them as int16 loses nothing
#pragma unroll
        for (int k = 0; k < 4; k++) q[k] = __byte_perm((unsigned)o[2 * k], (unsigned)o[2 * k + 1], 0x5410);
    }
    transpose8x8(q, lane);        // lane owns output row `row` again
    if (!live) return;
    if (KIND == B200_IDCT) {
        reinterpret_cast<uint4 *>(blocks_out)[blk * 8 + row] = make_uint4(q[0], q[1], q[2], q[3]);
        return;
    }
    uint8_t *d; long long ls;
    if (MB420) {
        const long long per_frame = (long long)g.mb_w * g.mb_h * 6;
        const long long f = blk / per_frame;
        const int r = (int)(blk - f * per_frame);
        const int mb = r / 6, k = r - mb * 6;
        const int mby = mb / g.mb_w, mbx = mb - mby * g.mb_w;
        if (k < 4) {
            ls = g.linesize[0];
            d = g.plane[0] + f * g.frame_stride[0] + (long long)(mby * 16 + (k >> 1) * 8) * ls + mbx * 16 + (k & 1) * 8;
        } else {
            ls = k == 4 ? g.linesize[1] : g.linesize[2];
            d = (k == 4 ? g.plane[1] + f * g.frame_stride[1] : g.plane[2] + f * g.frame_stride[2]) + (long long)(mby * 8) * ls + mbx * 8;
        }
    } else {
        ls = line_size ? __ldg(line_size + blk) : uniform_ls;
        d = dest + __ldg(dest_off + blk);
    }
    d += row * ls;
    int v0 = sx_lo(q[0]), v1 = sx_hi(q[0]), v2 = sx_lo(q[1]), v3 = sx_hi(q[1]);
    int v4 = sx_lo(q[2]), v5 = sx_hi(q[2]), v6 = sx_lo(q[3]), v7 = sx_hi(q[3]);
    const bool al8 = ((reinterpret_cast<uintptr_t>(d)) & 7) == 0;
    if (KIND == B200_IDCT_ADD) {
        uint2 p;
        if (al8) p = *reinterpret_cast<const uint2 *>(d);
        else {
            p.x = d[0] | (d[1] << 8) | (d[2] << 16) | ((unsigned)d[3] << 24);
            p.y = d[4] | (d[5] << 8) | (d[6] << 16) | ((unsigned)d[7] << 24);
        }
        v0 += p.x & 0xff; v1 += (p.x >> 8) & 0xff; v2 += (p.x >> 16) & 0xff; v3 += p.x >> 24;
        v4 += p.y & 0xff; v5 += (p.y >> 8) & 0xff; v6 += (p.y >> 16) & 0xff; v7 += p.y >> 24;
    }
    uint2 o;
    o.x = clip4(v0, v1, v2, v3);
    o.y = clip4(v4, v5, v6, v7);
    if (al8) *reinterpret_cast<uint2 *>(d) = o;
    else {
#pragma unroll
        for (int i = 0; i < 4; i++) { d[i] = (uint8_t)(o.x >> (8 * i)); d[4 + i] = (uint8_t)(o.y >> (8 * i)); }
    }
}

// ================================================================================================ thread-per-block kernels
// One thread owns one 8x8 block: no shuffles, no transposes — the row pass leaves 64 ints in registers and the column
// pass reads them by column.  Coalescing is recovered through shared memory:
//   in : the CTA's coefficient blocks are one contiguous byte range; it is copied with 16-byte cp.async (LDGSTS) into
//        shared memory with the 16-byte row slots of block b XOR-swizzled by (b & 7), so that lane t reading row j of
//        its own block (slot j ^ (t & 7)) is bank-conflict free;
//   out: (macroblock stream) each 8-macroblock segment of a macroblock row owns a 16 x 128 luma tile and two 8 x 64
//        chroma tiles in shared memory; threads drop their 8-byte rows there and the tile goes out as full 16-byte
//        chunks of whole rows (128-byte lines).  For `add` the tile is first filled from the destination the same way.
// HBM traffic stays the algorithmic 128 B in + 64 B out (+ 64 B) per block.

// 16-byte LDGSTS to a 32-bit shared-window address (convert the base pointer ONCE with smem_addr(): doing the
// generic->shared conversion per copy costs three extra instructions each)
__device__ __forceinline__ unsigned smem_addr(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cp_async16(unsigned smem_dst, const void *gsrc)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_dst), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// Full 8x8 inverse transform of the block whose swizzled rows start at `rows` (8 x uint4), lane swizzle key `key`.
// Result: for KIND == B200_IDCT the int16 block (packed, 8 x uint4 via outp); else 8 rows of clipped bytes (two words
// each) with `dest_rows` (8 x uint2 of existing pixels) added first when KIND == B200_IDCT_ADD.
template <int KIND>
__device__ __forceinline__ void idct_block(const uint4 *rows, int key, const uint2 *dest_rows, uint2 *out_rows, uint4 *out_coef)
{
    int R[8][8];
#pragma unroll
    for (int j = 0; j < 8; j++) row_pass<8>(rows[j ^ key], R[j]);
    unsigned P[8][4];                                  // per output row: four s16x2 pairs (clamped for put/add)
#pragma unroll
    for (int c = 0; c < 8; c += 2) {
        int oa[8], ob[8];
        col_pass<8>(R[0][c], R[1][c], R[2][c], R[3][c], R[4][c], R[5][c], R[6][c], R[7][c], oa);
        col_pass<8>(R[0][c + 1], R[1][c + 1], R[2][c + 1], R[3][c + 1], R[4][c + 1], R[5][c + 1], R[6][c + 1], R[7][c + 1], ob);
#pragma unroll
        for (int k = 0; k < 8; k++) {
            if (KIND == B200_IDCT_ADD) {
                const unsigned w = c < 4 ? dest_rows[k].x : dest_rows[k].y;
                oa[k] += (int)__byte_perm(w, 0, 0x4440 | (c & 3));
                ob[k] += (int)__byte_perm(w, 0, 0x4440 | ((c + 1) & 3));
            }
            const unsigned pr = __byte_perm((unsigned)oa[k], (unsigned)ob[k], 0x5410);     // (lo16(a), lo16(b))
            P[k][c >> 1] = KIND == B200_IDCT ? pr : __vimin_s16x2_relu(pr, 0x00ff00ffu);
        }
    }
#pragma unroll
    for (int k = 0; k < 8; k++) {
        if (KIND == B200_IDCT) {
            out_coef[k] = make_uint4(P[k][0], P[k][1], P[k][2], P[k][3]);
        } else {
            out_rows[k] = make_uint2(__byte_perm(P[k][0], P[k][1], 0x6420), __byte_perm(P[k][2], P[k][3], 0x6420));
        }
    }
}

constexpr int TPB_GEN = 128;        // blocks (= threads) per CTA, generic kernel

// generic destinations: dest + dest_off[b], rows stored straight to global memory (8-byte stores when aligned)
template <int KIND>
__global__ void __launch_bounds__(TPB_GEN)
idct_tpb_kernel(const int16_t *blocks, int16_t *blocks_out, long long nblocks, uint8_t *dest,
                const int64_t *__restrict__ dest_off, const int32_t *__restrict__ line_size, int uniform_ls)
{
    __shared__ uint4 sin[TPB_GEN * 8];
    const long long b0 = (long long)blockIdx.x * TPB_GEN;
    const int nb = (int)min((long long)TPB_GEN, nblocks - b0);
    const uint4 *g = reinterpret_cast<const uint4 *>(blocks) + b0 * 8;
    const unsigned s_in = smem_addr(sin);
    for (int i = threadIdx.x; i < nb * 8; i += TPB_GEN) {
        const int b = i >> 3, r = i & 7;
        cp_async16(s_in + (unsigned)(b * 8 + (r ^ (b & 7))) * 16u, g + i);
    }
    cp_async_wait_all();
    __syncthreads();
    const int t = threadIdx.x;
    const bool live = t < nb;
    uint2 drows[8], orows[8];
    uint4 ocoef[8];
    uint8_t *d = nullptr;
    long long ls = 0;
    if (live && KIND != B200_IDCT) {
        ls = line_size ? __ldg(line_size + b0 + t) : uniform_ls;
        d = dest + __ldg(dest_off + b0 + t);
    }
    const bool al8 = ((reinterpret_cast<uintptr_t>(d) | (unsigned long long)ls) & 7) == 0;
    if (live && KIND == B200_IDCT_ADD) {
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const uint8_t *p = d + k * ls;
            if (al8) drows[k] = *reinterpret_cast<const uint2 *>(p);
            else {
                drows[k].x = p[0] | (p[1] << 8) | (p[2] << 16) | ((unsigned)p[3] << 24);
                drows[k].y = p[4] | (p[5] << 8) | (p[6] << 16) | ((unsigned)p[7] << 24);
            }
        }
    }
    if (live) idct_block<KIND>(&sin[t * 8], t & 7, drows, orows, ocoef);
    if (KIND == B200_IDCT) {
        __syncthreads();                                   // everybody has consumed its input rows
        if (live) {
#pragma unroll
            for (int k = 0; k < 8; k++) sin[t * 8 + (k ^ (t & 7))] = ocoef[k];
        }
        __syncthreads();
        uint4 *go = reinterpret_cast<uint4 *>(blocks_out) + b0 * 8;
        for (int i = threadIdx.x; i < nb * 8; i += TPB_GEN) {
            const int b = i >> 3, r = i & 7;
            go[i] = sin[b * 8 + (r ^ (b & 7))];
        }
    } else if (live) {
#pragma unroll
        for (int k = 0; k < 8; k++) {
            uint8_t *p = d + k * ls;
            if (al8) *reinterpret_cast<uint2 *>(p) = orows[k];
            else {
#pragma unroll
                for (int i = 0; i < 4; i++) { p[i] = (uint8_t)(orows[k].x >> (8 * i)); p[4 + i] = (uint8_t)(orows[k].y >> (8 * i)); }
            }
        }
    }
}

// 4:2:0 macroblock stream.  blockDim.x = 48 * SEGS; segment = 8 consecutive macroblocks of one macroblock row.
// Grid: x over groups of SEGS segments of a row, y over macroblock rows, z over frames.
// Registers are kept low (4 CTAs per SM) by holding the row-pass result packed (32 words) and by sending every clamped
// pixel pair straight to the shared-memory tile (2-byte stores; for `add` the same 2 bytes are read first).
// Luma tile rows 8..15 are stored with their 64-byte halves swapped so that blocks Y0/Y2 (and Y1/Y3) of one
// macroblock, which sit 8 rows = 1024 B apart, do not share banks.
// ---- inverse quantisation fused in front of the transform (put_dct / add_dequant_dct, libavcodec/mpegvideo_dec.c:907-922): the
// arithmetic of mpv_unquant.cuh (libavcodec/mpegvideo_unquantize.c:50-276) that unquant.cu's kernel uses too, applied by the thread
// that owns the block to the eight rows it takes out of shared memory — the dequantised coefficients never exist in HBM (128 B read +
// 128 B written per block saved against the two-kernel sequence).  V = -1: no dequantisation (the plain IDCT kernels).
struct FusedUnquant : UnquantDev {        // passed by value (kernel parameter: every table index is a compile-time constant)
    const uint8_t *qscale;                // per block
    const int8_t *last_index;             // per block
};
// the eight rows of one block (row j in r[j], 8 int16 each) dequantised in place; n = block number inside its macroblock
template <int V>
__device__ __forceinline__ void fused_unquant_rows(uint4 (&r)[8], const FusedUnquant &P, int n, int qs, int last)
{
    const MpvBlock blk = mpv_block<V>(P, qs, last);
    int parity = 0;
#pragma unroll
    for (int row = 0; row < 8; row++) {
        unsigned w[4] = { r[row].x, r[row].y, r[row].z, r[row].w };
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const int j = 8 * row + k;
            int level = (k & 1) ? (int)w[k >> 1] >> 16 : (int)(short)(w[k >> 1] & 0xffffu);
            mpv_coef<V>(P, blk, n, j, mpv_matrix<V>(P, j), mpv_scanpos<V>(P, j), level, parity);
            if (MpvVariant<V>::MISMATCH && j == 63) level ^= (int)(1u ^ ((unsigned)parity & 1u));      // sum starts at -1: block[63] ^= sum & 1
            w[k >> 1] = (k & 1) ? (w[k >> 1] & 0xffffu) | ((unsigned)level << 16) : (w[k >> 1] & 0xffff0000u) | ((unsigned)level & 0xffffu);
        }
        r[row] = make_uint4(w[0], w[1], w[2], w[3]);
    }
}

constexpr int MAX_SEGS = 6;
__device__ __forceinline__ int luma_swz(int row) { return (row & 8) << 3; }               // 0 or 64

template <int KIND, int V = -1>
__global__ void __launch_bounds__(48 * MAX_SEGS, V < 0 ? 4 : 2)
idct_mb420_kernel(const int16_t *blocks, Mb420Geom g, int segs_per_cta, const __grid_constant__ FusedUnquant UQ)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint4 *sin = reinterpret_cast<uint4 *>(smem_raw);                                     // segs * 48 * 8 uint4
    unsigned char *tiles = smem_raw + (size_t)segs_per_cta * 48 * 128;                    // segs * 3072 B
    const int t = threadIdx.x, seg = t / 48, w = t - seg * 48;
    const int mby = blockIdx.y;
    const long long f = blockIdx.z;
    const int sx = blockIdx.x * segs_per_cta + seg;                                       // segment index within the row
    const int mbx0 = sx * 8;
    const int nmb = min(8, g.mb_w - mbx0);                                                // <= 0: segment beyond the row
    uint4 *my_in = sin + seg * 48 * 8;
    unsigned char *tile = tiles + seg * 3072;                                             // luma 16x128, U 8x64, V 8x64
    const int ls0 = g.linesize[0], ls1 = g.linesize[1], ls2 = g.linesize[2];
    uint8_t *py = g.plane[0] + f * g.frame_stride[0] + (long long)(mby * 16) * ls0 + mbx0 * 16;
    uint8_t *pu = g.plane[1] + f * g.frame_stride[1] + (long long)(mby * 8) * ls1 + mbx0 * 8;
    uint8_t *pv = g.plane[2] + f * g.frame_stride[2] + (long long)(mby * 8) * ls2 + mbx0 * 8;
    if (nmb > 0) {
        const long long blk0 = (((f * g.mb_h + mby) * g.mb_w) + mbx0) * 6;
        const uint4 *gsrc = reinterpret_cast<const uint4 *>(blocks) + blk0 * 8;
        {
            // chunk i = w + 48*it of the segment: block b = b0 + 6*it, row r = w & 7, swizzled slot r ^ (b & 7).
            // (b & 7) = (b0 + 2k) & 7 with k = (3*it) & 3, so four slot offsets cover all eight copies.
            const int r = w & 7, nb = nmb * 6, b0 = w >> 3;
            const unsigned s_in = smem_addr(my_in) + (unsigned)b0 * 128u;
            const uint4 *gp = gsrc + b0 * 8 + r;
            unsigned slot[4];
#pragma unroll
            for (int k = 0; k < 4; k++) slot[k] = (unsigned)(r ^ ((b0 + 2 * k) & 7)) * 16u;
#pragma unroll
            for (int it = 0; it < 8; it++)
                if (b0 + 6 * it < nb) cp_async16(s_in + (unsigned)it * 768u + slot[(3 * it) & 3], gp + it * 48);
        }
        if (KIND == B200_IDCT_ADD) {                                                      // stage the destination tile
            for (int i = w; i < 128; i += 48) {                                           // luma: 16 rows x 8 chunks of 16 B
                const int row = i >> 3, ch = i & 7;
                if (ch < nmb) cp_async16(smem_addr(tile) + (unsigned)(row * 128 + ((ch * 16) ^ luma_swz(row))), py + (long long)row * ls0 + ch * 16);
            }
            for (int i = w; i < 64; i += 48) {                                            // chroma: 8 rows x 8 chunks of 8 B each plane
                const int row = i >> 3, ch = i & 7;
                if (ch < nmb) {
                    *reinterpret_cast<uint2 *>(tile + 2048 + row * 64 + ch * 8) = *reinterpret_cast<const uint2 *>(pu + (long long)row * ls1 + ch * 8);
                    *reinterpret_cast<uint2 *>(tile + 2560 + row * 64 + ch * 8) = *reinterpret_cast<const uint2 *>(pv + (long long)row * ls2 + ch * 8);
                }
            }
        }
    }
    cp_async_wait_all();
    __syncthreads();
    const int m = w / 6, k = w - m * 6;                                                   // macroblock in segment, block in macroblock
    if (m < nmb) {
        unsigned char *trow; int tp;
        if (k < 4) { trow = tile + ((k >> 1) * 8) * 128 + ((m * 16 + (k & 1) * 8) ^ ((k >> 1) * 64)); tp = 128; }
        else       { trow = tile + (k == 4 ? 2048 : 2560) + m * 8; tp = 64; }
        const uint4 *rows = &my_in[w * 8];
        const int key = w & 7;
        unsigned R2[8][4];
        bool skip = false;
        if (V >= 0) {
            const long long bi = (((f * g.mb_h + mby) * g.mb_w) + mbx0 + m) * 6 + k;
            const int last = __ldg(UQ.last_index + bi);
            skip = KIND == B200_IDCT_ADD && last < 0;                                     // add_dequant_dct: block_last_index < 0 leaves the pixels alone
            uint4 rr[8];
#pragma unroll
            for (int j = 0; j < 8; j++) rr[j] = rows[j ^ key];
            fused_unquant_rows<V < 0 ? 0 : V>(rr, UQ, k, (int)__ldg(UQ.qscale + bi), last);
#pragma unroll
            for (int j = 0; j < 8; j++) row_pass<8>(rr[j], R2[j]);
        } else {
#pragma unroll
            for (int j = 0; j < 8; j++) row_pass<8>(rows[j ^ key], R2[j]);
        }
        if (!skip) {
#pragma unroll
        for (int half = 0; half < 2; half++) {             // four columns (one 32-bit tile word per row) at a time
            unsigned e0[8], e1[8], e2[8], e3[8];             // column sums before the >> 20 (rows in the order 0,1,2,3,4,5,6,7)
            const int c0 = 2 * half, c1 = 2 * half + 1;
            col_sums<8>(sx_lo(R2[0][c0]), sx_lo(R2[1][c0]), sx_lo(R2[2][c0]), sx_lo(R2[3][c0]),
                     sx_lo(R2[4][c0]), sx_lo(R2[5][c0]), sx_lo(R2[6][c0]), sx_lo(R2[7][c0]), e0);
            col_sums<8>(sx_hi(R2[0][c0]), sx_hi(R2[1][c0]), sx_hi(R2[2][c0]), sx_hi(R2[3][c0]),
                     sx_hi(R2[4][c0]), sx_hi(R2[5][c0]), sx_hi(R2[6][c0]), sx_hi(R2[7][c0]), e1);
            col_sums<8>(sx_lo(R2[0][c1]), sx_lo(R2[1][c1]), sx_lo(R2[2][c1]), sx_lo(R2[3][c1]),
                     sx_lo(R2[4][c1]), sx_lo(R2[5][c1]), sx_lo(R2[6][c1]), sx_lo(R2[7][c1]), e2);
            col_sums<8>(sx_hi(R2[0][c1]), sx_hi(R2[1][c1]), sx_hi(R2[2][c1]), sx_hi(R2[3][c1]),
                     sx_hi(R2[4][c1]), sx_hi(R2[5][c1]), sx_hi(R2[6][c1]), sx_hi(R2[7][c1]), e3);
#pragma unroll
            for (int r = 0; r < 8; r++) {
                unsigned *px = reinterpret_cast<unsigned *>(trow + r * tp + 4 * half);
                if (KIND == B200_IDCT_ADD) {
                    const unsigned dd = *px;
                    const int o0 = ((int)e0[r] >> 20) + (int)__byte_perm(dd, 0, 0x4440), o1 = ((int)e1[r] >> 20) + (int)__byte_perm(dd, 0, 0x4441);
                    const int o2 = ((int)e2[r] >> 20) + (int)__byte_perm(dd, 0, 0x4442), o3 = ((int)e3[r] >> 20) + (int)(dd >> 24);
                    const unsigned lo = __vimin_s16x2_relu(__byte_perm((unsigned)o0, (unsigned)o1, 0x5410), 0x00ff00ffu);
                    const unsigned hi = __vimin_s16x2_relu(__byte_perm((unsigned)o2, (unsigned)o3, 0x5410), 0x00ff00ffu);
                    *px = __byte_perm(lo, hi, 0x6420);
                } else {
                    // clip_u8(sum >> 20) == clamp(sum >> 16, 0, 4095) >> 4: take the high halves (PRMT), clamp both as s16x2,
                    // shift the pair once; bytes 0 and 2 of the shifted pair are the pixels
                    const unsigned lo = __vimin_s16x2_relu(__byte_perm(e0[r], e1[r], 0x7632), 0x0fff0fffu) >> 4;
                    const unsigned hi = __vimin_s16x2_relu(__byte_perm(e2[r], e3[r], 0x7632), 0x0fff0fffu) >> 4;
                    *px = __byte_perm(lo, hi, 0x6420);
                }
            }
        }
        }
    }
    __syncthreads();
    if (nmb > 0) {
        for (int i = w; i < 128; i += 48) {
            const int row = i >> 3, ch = i & 7;
            if (ch < nmb) *reinterpret_cast<uint4 *>(py + (long long)row * ls0 + ch * 16) =
                              *reinterpret_cast<const uint4 *>(tile + row * 128 + ((ch * 16) ^ luma_swz(row)));
        }
        for (int i = w; i < 64; i += 48) {
            const int row = i >> 3, ch = i & 7;
            if (ch < nmb) {
                *reinterpret_cast<uint2 *>(pu + (long long)row * ls1 + ch * 8) = *reinterpret_cast<const uint2 *>(tile + 2048 + row * 64 + ch * 8);
                *reinterpret_cast<uint2 *>(pv + (long long)row * ls2 + ch * 8) = *reinterpret_cast<const uint2 *>(tile + 2560 + row * 64 + ch * 8);
            }
        }
    }
}

// clamp helpers on one block (drop-in level only): kind 0 put, 1 put_signed, 2 add
__global__ void pixels_clamped_kernel(int kind, const int16_t *block, uint8_t *pix /* packed 8x8 */)
{
    const int i = threadIdx.x;
    const int b = block[i];
    if (kind == 0) pix[i] = (uint8_t)min(max(b, 0), 255);
    else if (kind == 1) pix[i] = b < -128 ? 0 : b > 127 ? 255 : (uint8_t)(b + 128);
    else pix[i] = (uint8_t)min(max((int)pix[i] + b, 0), 255);
}

template <int KIND, bool MB420>
int launch_idct(cudaStream_t st, const int16_t *blocks, int16_t *out, long long nblocks, uint8_t *dest,
                const int64_t *dest_off, const int32_t *line_size, int uls, const Mb420Geom &g)
{
    if (nblocks <= 0) return 0;
    const int threads = 256;                              // 8 warps = 32 blocks per CTA
    const long long ctas = (nblocks + 31) / 32;
    if (ctas > 0x7fffffffLL) return B200_EINVAL;
    idct8x8_kernel<KIND, MB420><<<(unsigned)ctas, threads, 0, st>>>(blocks, out, nblocks, dest, dest_off, line_size, uls, g);
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

template <int KIND>
int launch_tpb(cudaStream_t st, const int16_t *blocks, int16_t *out, long long nblocks, uint8_t *dest,
               const int64_t *dest_off, const int32_t *line_size, int uls)
{
    if (nblocks <= 0) return 0;
    const long long ctas = (nblocks + TPB_GEN - 1) / TPB_GEN;
    if (ctas > 0x7fffffffLL) return B200_EINVAL;
    idct_tpb_kernel<KIND><<<(unsigned)ctas, TPB_GEN, 0, st>>>(blocks, out, nblocks, dest, dest_off, line_size, uls);
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

// macroblock stream through the tiled kernel when planes/strides allow 16-byte (luma) and 8-byte (chroma) chunks
template <int KIND>
int launch_mb420(cudaStream_t st, const int16_t *blocks, const Mb420Geom &g, int nframes, bool *handled)
{
    *handled = false;
    const bool ok = (((uintptr_t)g.plane[0] | (uintptr_t)g.linesize[0] | (uintptr_t)g.frame_stride[0]) & 15) == 0 &&
                    (((uintptr_t)g.plane[1] | (uintptr_t)g.linesize[1] | (uintptr_t)g.frame_stride[1] |
                      (uintptr_t)g.plane[2] | (uintptr_t)g.linesize[2] | (uintptr_t)g.frame_stride[2]) & 7) == 0 &&
                    g.mb_h <= 65535 && g.linesize[0] > 0 && g.linesize[1] > 0 && g.linesize[2] > 0;
    if (!ok) return 0;
    const int segs_row = (g.mb_w + 7) / 8;
    int best = 4, waste = 1 << 30;
    for (int s = 3; s <= MAX_SEGS; s++) {                     // pick the CTA width that wastes the fewest idle segments
        const int wst = ((segs_row + s - 1) / s) * s - segs_row;
        if (wst < waste || (wst == waste && s > best)) { waste = wst; best = s; }
    }
    const size_t smem = (size_t)best * (48 * 128 + 3072);
    B200_CUDA_OK(cudaFuncSetAttribute(idct_mb420_kernel<KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    for (int f0 = 0; f0 < nframes; f0 += 65535) {
        const int nf = nframes - f0 < 65535 ? nframes - f0 : 65535;
        Mb420Geom gg = g;
        for (int i = 0; i < 3; i++) gg.plane[i] += (long long)f0 * g.frame_stride[i];
        dim3 grid((segs_row + best - 1) / best, g.mb_h, nf);
        idct_mb420_kernel<KIND><<<grid, 48 * best, smem, st>>>(blocks + (long long)f0 * g.mb_w * g.mb_h * 6 * 64, gg, best, FusedUnquant{});
        B200_LAUNCHED();
    }
    B200_CUDA_OK(cudaGetLastError());
    *handled = true;
    return 0;
}

// fused inverse quantiser + IDCT over the macroblock stream (aligned planes only: the tiled kernel)
template <int KIND, int V>
int launch_mb420_fused(cudaStream_t st, const int16_t *blocks, const Mb420Geom &g, int nframes, const FusedUnquant &UQ)
{
    const bool ok = (((uintptr_t)g.plane[0] | (uintptr_t)g.linesize[0] | (uintptr_t)g.frame_stride[0]) & 15) == 0 &&
                    (((uintptr_t)g.plane[1] | (uintptr_t)g.linesize[1] | (uintptr_t)g.frame_stride[1] |
                      (uintptr_t)g.plane[2] | (uintptr_t)g.linesize[2] | (uintptr_t)g.frame_stride[2]) & 7) == 0 &&
                    g.mb_h <= 65535 && g.linesize[0] > 0 && g.linesize[1] > 0 && g.linesize[2] > 0;
    if (!ok) { b200_set_error("unquant + idct: planes must be 16-byte (luma) / 8-byte (chroma) aligned with positive line sizes"); return B200_EINVAL; }
    if (nframes > 65535) return B200_EINVAL;
    const int segs_row = (g.mb_w + 7) / 8;
    int best = 4, waste = 1 << 30;
    for (int s = 3; s <= MAX_SEGS; s++) {
        const int wst = ((segs_row + s - 1) / s) * s - segs_row;
        if (wst < waste || (wst == waste && s > best)) { waste = wst; best = s; }
    }
    const size_t smem = (size_t)best * (48 * 128 + 3072);
    B200_CUDA_OK(cudaFuncSetAttribute(idct_mb420_kernel<KIND, V>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid((segs_row + best - 1) / best, g.mb_h, nframes);
    idct_mb420_kernel<KIND, V><<<grid, 48 * best, smem, st>>>(blocks, g, best, UQ);
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

int dispatch(cudaStream_t st, int kind, bool mb420, const int16_t *blocks, int16_t *out, long long n, uint8_t *dest,
             const int64_t *off, const int32_t *ls, int uls, const Mb420Geom &g, int nframes = 0)
{
    if (mb420) {
        bool handled = false;
        int ret = kind == B200_IDCT_PUT ? launch_mb420<B200_IDCT_PUT>(st, blocks, g, nframes, &handled)
                                        : launch_mb420<B200_IDCT_ADD>(st, blocks, g, nframes, &handled);
        if (ret < 0 || handled) return ret;
        // unaligned planes: the warp-cooperative kernel computes the implied destinations itself
        return kind == B200_IDCT_PUT ? launch_idct<B200_IDCT_PUT, true>(st, blocks, out, n, dest, off, ls, uls, g)
                                     : launch_idct<B200_IDCT_ADD, true>(st, blocks, out, n, dest, off, ls, uls, g);
    }
    switch (kind) {
    case B200_IDCT:     return launch_tpb<B200_IDCT>(st, blocks, out, n, dest, off, ls, uls);
    case B200_IDCT_PUT: return launch_tpb<B200_IDCT_PUT>(st, blocks, out, n, dest, off, ls, uls);
    case B200_IDCT_ADD: return launch_tpb<B200_IDCT_ADD>(st, blocks, out, n, dest, off, ls, uls);
    }
    return B200_EINVAL;
}

} // namespace

B200_API int b200_mpv_unquant_idct_mb420_device(B200Device *dev, int variant, const B200MpvUnquant *p, int kind, const int16_t *blocks,
                                                const uint8_t *qscale, const int8_t *last_index, int mb_w, int mb_h, int nframes,
                                                uint8_t *const planes[3], const int linesize[3], const int64_t frame_stride[3])
{
    if (!dev || !p || !blocks || !qscale || !last_index || !planes || !linesize || !frame_stride || mb_w <= 0 || mb_h <= 0 || nframes < 0)
        return B200_EINVAL;
    if (kind != B200_IDCT_PUT && kind != B200_IDCT_ADD) return B200_EINVAL;
    if (variant < 0 || variant > B200_UNQUANT_H263_INTER) return B200_EINVAL;
    if (((uintptr_t)blocks) & 15) return B200_EINVAL;
    if (nframes == 0) return 0;
    FusedUnquant U;
    if (!mpv_unquant_params(p, &U)) { b200_set_error("b200_mpv_unquant_idct: permutated[] is not a permutation of 0..63"); return B200_EINVAL; }
    U.qscale = qscale; U.last_index = last_index;
    if (int r = b200_use_device(dev)) return r;
    Mb420Geom g{};
    g.mb_w = mb_w; g.mb_h = mb_h;
    for (int i = 0; i < 3; i++) { g.plane[i] = planes[i]; g.linesize[i] = linesize[i]; g.frame_stride[i] = frame_stride[i]; }
    cudaStream_t st = dev->stream;
    int ret = B200_EINVAL;
    switch (variant * 2 + (kind == B200_IDCT_ADD)) {
#define CASE(V) case (V) * 2: ret = launch_mb420_fused<B200_IDCT_PUT, V>(st, blocks, g, nframes, U); break; \
                case (V) * 2 + 1: ret = launch_mb420_fused<B200_IDCT_ADD, V>(st, blocks, g, nframes, U); break;
    CASE(B200_UNQUANT_MPEG1_INTRA) CASE(B200_UNQUANT_MPEG1_INTER) CASE(B200_UNQUANT_MPEG2_INTRA)
    CASE(B200_UNQUANT_MPEG2_INTRA_BITEXACT) CASE(B200_UNQUANT_MPEG2_INTER) CASE(B200_UNQUANT_H263_INTRA) CASE(B200_UNQUANT_H263_INTER)
#undef CASE
    }
    return ret;
}

B200_API int b200_idct_batch_device(B200Device *dev, int kind, int16_t *blocks, int64_t nblocks, uint8_t *dest,
                                    const int64_t *dest_off, const int32_t *line_size, int uniform_line_size)
{
    if (!dev || !blocks || nblocks < 0) return B200_EINVAL;
    if (kind != B200_IDCT && (!dest || !dest_off)) return B200_EINVAL;
    if (((uintptr_t)blocks) & 15) { b200_set_error("idct: coefficient blocks must be 16-byte aligned"); return B200_EINVAL; }
    if (int r = b200_use_device(dev)) return r;
    Mb420Geom g{};
    return dispatch(dev->stream, kind, false, blocks, blocks, nblocks, dest, dest_off, line_size, uniform_line_size, g);
}

B200_API int b200_idct_mb420_device(B200Device *dev, int kind, const int16_t *blocks, int mb_w, int mb_h, int nframes,
                                    uint8_t *const planes[3], const int linesize[3], const int64_t frame_stride[3])
{
    if (!dev || !blocks || !planes || !linesize || !frame_stride || mb_w <= 0 || mb_h <= 0 || nframes < 0) return B200_EINVAL;
    if (kind != B200_IDCT_PUT && kind != B200_IDCT_ADD) return B200_EINVAL;
    if (((uintptr_t)blocks) & 15) return B200_EINVAL;
    if (int r = b200_use_device(dev)) return r;
    Mb420Geom g{};
    g.mb_w = mb_w; g.mb_h = mb_h;
    for (int i = 0; i < 3; i++) { g.plane[i] = planes[i]; g.linesize[i] = linesize[i]; g.frame_stride[i] = frame_stride[i]; }
    const long long n = (long long)mb_w * mb_h * 6 * nframes;
    return dispatch(dev->stream, kind, true, blocks, nullptr, n, nullptr, nullptr, nullptr, 0, g, nframes);
}

B200_API int b200_idct_mb420_host(B200Device *dev, int kind, const int16_t *blocks, int mb_w, int mb_h, int nframes,
                                  uint8_t *const planes[3], const int linesize[3], const int64_t frame_stride[3])
{
    if (!dev || !blocks || !planes || !linesize || !frame_stride || mb_w <= 0 || mb_h <= 0 || nframes < 0) return B200_EINVAL;
    if (kind != B200_IDCT_PUT && kind != B200_IDCT_ADD) return B200_EINVAL;
    B200_CUDA_OK(cudaSetDevice(dev->ordinal));
    // device-side packed frames: Y (16*mb_w x 16*mb_h), U, V (8*mb_w x 8*mb_h), pitch = width rounded to 256
    const int W[3] = { mb_w * 16, mb_w * 8, mb_w * 8 }, H[3] = { mb_h * 16, mb_h * 8, mb_h * 8 };
    size_t pitch[3], off[3], frameBytes = 0;
    for (int i = 0; i < 3; i++) { pitch[i] = ((size_t)W[i] + 255) & ~(size_t)255; off[i] = frameBytes; frameBytes += pitch[i] * H[i]; }
    const size_t coefBytes = (size_t)mb_w * mb_h * 6 * 128;
    const size_t perFrame = coefBytes + frameBytes;
    int chunk = (int)(((size_t)256 << 20) / perFrame);
    if (chunk < 1) chunk = 1;
    if (chunk > nframes) chunk = nframes > 0 ? nframes : 1;
    const int K = B200Device::kPipe;
    B200_LOCK_DEVICE(dev);      // scratch + stream are per device: one host-pointer call at a time (released on return)
    uint8_t *scr = (uint8_t *)b200_scratch(dev, perFrame * chunk * K);
    if (!scr) return B200_ENOMEM;
    B200_CUDA_OK(cudaStreamSynchronize(dev->stream));
    int slot = 0;
    for (int f0 = 0; f0 < nframes; f0 += chunk, slot = (slot + 1) % K) {
        const int nf = nframes - f0 < chunk ? nframes - f0 : chunk;
        cudaStream_t st = dev->pipe[slot];
        uint8_t *cbase = scr + (size_t)slot * perFrame * chunk;
        uint8_t *pbase = cbase + coefBytes * chunk;
        B200_CUDA_OK(cudaMemcpyAsync(cbase, (const uint8_t *)blocks + (size_t)f0 * coefBytes, coefBytes * nf, cudaMemcpyHostToDevice, st));
        if (kind == B200_IDCT_ADD)
            for (int f = 0; f < nf; f++)
                for (int i = 0; i < 3; i++)
                    B200_CUDA_OK(cudaMemcpy2DAsync(pbase + (size_t)f * frameBytes + off[i], pitch[i],
                                                   planes[i] + (int64_t)(f0 + f) * frame_stride[i], (size_t)linesize[i],
                                                   W[i], H[i], cudaMemcpyHostToDevice, st));
        Mb420Geom g{};
        g.mb_w = mb_w; g.mb_h = mb_h;
        for (int i = 0; i < 3; i++) { g.plane[i] = pbase + off[i]; g.linesize[i] = (int)pitch[i]; g.frame_stride[i] = (long long)frameBytes; }
        int ret = dispatch(st, kind, true, (const int16_t *)cbase, nullptr, (long long)mb_w * mb_h * 6 * nf, nullptr, nullptr, nullptr, 0, g, nf);
        if (ret < 0) return ret;
        for (int f = 0; f < nf; f++)
            for (int i = 0; i < 3; i++)
                B200_CUDA_OK(cudaMemcpy2DAsync(planes[i] + (int64_t)(f0 + f) * frame_stride[i], (size_t)linesize[i],
                                               pbase + (size_t)f * frameBytes + off[i], pitch[i], W[i], H[i],
                                               cudaMemcpyDeviceToHost, st));
    }
    for (int i = 0; i < K; i++) B200_CUDA_OK(cudaStreamSynchronize(dev->pipe[i]));
    return 0;
}

// ------------------------------------------------------------------------------------------------ drop-in pointer table
// The reference's per-block entry points carry no context argument, so they use the process-wide default device.
// Each call moves one block through the device: this level exists for parity and for un-modified callers, the
// batched entry points above are the fast path.
namespace {

void one_block(const char *feature, int kind, uint8_t *dest, ptrdiff_t line_size, int16_t *block)
{
    B200HostCall call(feature, nullptr, 256);
    int16_t *dblk = (int16_t *)call.scratch;
    uint8_t *dpix = call.scratch + 128;      // packed 8x8, line size 8
    int64_t *doff = (int64_t *)(call.scratch + 192);
    cudaStream_t st = call.stream;
    call.check(cudaMemcpyAsync(dblk, block, 128, cudaMemcpyHostToDevice, st), "h2d block");
    if (kind == B200_IDCT_ADD) call.check(b200_h2d_rows(dpix, 8, dest, line_size, 8, 8, st), "h2d dest");
    call.check(cudaMemsetAsync(doff, 0, 8, st), "memset");
    Mb420Geom g{};
    call.launched(dispatch(st, kind, false, dblk, dblk, 1, dpix, doff, nullptr, 8, g));
    if (kind == B200_IDCT) call.check(cudaMemcpyAsync(block, dblk, 128, cudaMemcpyDeviceToHost, st), "d2h block");
    else call.check(b200_d2h_rows(dest, line_size, dpix, 8, 8, 8, st), "d2h dest");
    call.sync();
}

void one_clamp(const char *feature, int kind, const int16_t *block, uint8_t *pixels, ptrdiff_t line_size)
{
    B200HostCall call(feature, nullptr, 256);
    uint8_t *scr = call.scratch;
    cudaStream_t st = call.stream;
    call.check(cudaMemcpyAsync(scr, block, 128, cudaMemcpyHostToDevice, st), "h2d block");
    if (kind == 2) call.check(b200_h2d_rows(scr + 128, 8, pixels, line_size, 8, 8, st), "h2d pixels");
    pixels_clamped_kernel<<<1, 64, 0, st>>>(kind, (const int16_t *)scr, scr + 128);
    B200_LAUNCHED();
    call.launched();
    call.check(b200_d2h_rows(pixels, line_size, scr + 128, 8, 8, 8, st), "d2h pixels");
    call.sync();
}

void tab_idct(int16_t *block) { one_block("idct", B200_IDCT, nullptr, 0, block); }
void tab_idct_put(uint8_t *dest, ptrdiff_t ls, int16_t *block) { one_block("idct_put", B200_IDCT_PUT, dest, ls, block); }
void tab_idct_add(uint8_t *dest, ptrdiff_t ls, int16_t *block) { one_block("idct_add", B200_IDCT_ADD, dest, ls, block); }
void tab_put_clamped(const int16_t *b, uint8_t *p, ptrdiff_t ls) { one_clamp("put_pixels_clamped", 0, b, p, ls); }
void tab_put_signed_clamped(const int16_t *b, uint8_t *p, ptrdiff_t ls) { one_clamp("put_signed_pixels_clamped", 1, b, p, ls); }
void tab_add_clamped(const int16_t *b, uint8_t *p, ptrdiff_t ls) { one_clamp("add_pixels_clamped", 2, b, p, ls); }

} // namespace

B200_API int b200_idctdsp_init(B200IDCTDSPContext *c, int idct_algo, int bits_per_raw_sample, int lowres)
{
    if (!c) return B200_EINVAL;
    // ff_idctdsp_init, libavcodec/idctdsp.c:228-314: FF_IDCT_AUTO (0) and FF_IDCT_SIMPLE (2) at <= 8 bits select simple_idct
    if (lowres != 0 || bits_per_raw_sample > 8 || (idct_algo != 0 && idct_algo != 2)) return B200_ENOSYS;
    if (!b200_default_device()) return B200_ENODEV;
    memset(c, 0, sizeof(*c));
    c->put_pixels_clamped = tab_put_clamped;
    c->put_signed_pixels_clamped = tab_put_signed_clamped;
    c->add_pixels_clamped = tab_add_clamped;
    c->idct = tab_idct;
    c->idct_put = tab_idct_put;
    c->idct_add = tab_idct_add;
    for (int i = 0; i < 64; i++) c->idct_permutation[i] = (uint8_t)i;       // FF_IDCT_PERM_NONE, idctdsp.c:287
    c->perm_type = 0;
    return 0;
}
