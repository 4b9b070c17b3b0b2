// emu.h — TEST INFRASTRUCTURE ONLY.  A few dozen lines that let the device code of the kernels written without GPU access
// compile and run on the host, one CUDA thread after the other (a real OS thread per lane where a kernel uses a warp
// collective), so their arithmetic and indexing can be compared with the checker before they ever see a GPU.
// It emulates only what those kernels use: built-in index variables, __ldg, the round-to-nearest float intrinsics, min / max,
// uint4, __reduce_xor_sync.  It does not model memory spaces, races or performance.
#pragma once
#include <cstdint>
#include <cstddef>
#include <algorithm>
#include <barrier>
#include <thread>
#include <vector>
#include <functional>
#include <memory>
#include <cstring>

struct dim3 { unsigned x, y, z; dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {} };
struct uint4 { unsigned x, y, z, w; };
struct uint2 { unsigned x, y; };
struct int2 { int x, y; };
struct int4 { int x, y, z, w; };
static inline int4 make_int4(int a, int b, int c, int d) { int4 r = { a, b, c, d }; return r; }
static inline uint2 make_uint2(unsigned a, unsigned b) { uint2 r = { a, b }; return r; }
static inline int2 make_int2(int a, int b) { int2 r = { a, b }; return r; }
static inline uint4 make_uint4(unsigned a, unsigned b, unsigned c, unsigned d) { uint4 r = { a, b, c, d }; return r; }
struct float2 { float x, y; };
static inline float2 make_float2(float a, float b) { float2 r = { a, b }; return r; }
struct double2 { double x, y; };
static inline double2 make_double2(double a, double b) { double2 r = { a, b }; return r; }
static thread_local dim3 threadIdx, blockIdx, blockDim, gridDim;

#define __global__
#define __host__
#define __device__
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __constant__ static const
#define __restrict__
#define __grid_constant__

template <typename T> static inline T __ldg(const T *p) { return *p; }
using std::min;
using std::max;
static inline float  __fmul_rn(float a, float b)   { volatile float r = a * b; return r; }      // volatile: no contraction into an fma
static inline float  __fadd_rn(float a, float b)   { volatile float r = a + b; return r; }
static inline double __dmul_rn(double a, double b) { volatile double r = a * b; return r; }
static inline double __dadd_rn(double a, double b) { volatile double r = a + b; return r; }

// integer SIMD-in-a-word intrinsics of the swscale kernels, by their PTX definitions
static inline unsigned __byte_perm(unsigned x, unsigned y, unsigned s)          // PRMT, default mode: nibble n picks byte n of {y,x}; bit 3 = replicate its sign
{
    const unsigned long long v = ((unsigned long long)y << 32) | x;
    unsigned r = 0;
    for (int i = 0; i < 4; i++) {
        const unsigned sel = (s >> (4 * i)) & 0xF;
        unsigned b = (unsigned)(v >> (8 * (sel & 7))) & 0xFF;
        if (sel & 8) b = (b & 0x80) ? 0xFF : 0x00;
        r |= b << (8 * i);
    }
    return r;
}
static inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned sh)   // SHF.R.WRAP: low word of {hi,lo} >> (sh & 31)
{
    return (unsigned)(((((unsigned long long)hi) << 32) | lo) >> (sh & 31));
}
static inline int atomicAdd(int *p, int v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
static inline int __mulhi(int a, int b) { return (int)(((long long)a * (long long)b) >> 32); }
static inline int __vimin_s32_relu(int a, int b) { const int m = a < b ? a : b; return m < 0 ? 0 : m; }
static inline unsigned __vimin_s16x2_relu(unsigned a, unsigned b)               // per signed halfword: max(min(a, b), 0)
{
    unsigned r = 0;
    for (int i = 0; i < 2; i++) {
        const int x = (int16_t)(a >> (16 * i)), y = (int16_t)(b >> (16 * i));
        int m = x < y ? x : y;
        if (m < 0) m = 0;
        r |= ((unsigned)m & 0xFFFF) << (16 * i);
    }
    return r;
}
// dp2a.{lo,hi}.s32.u32 d, a, b, c with a as two signed halfwords and b as unsigned bytes (what the two asm helpers of sws.cu emit):
// d = c + a.h0 * b.byte[0 | 2] + a.h1 * b.byte[1 | 3]
static inline int emu_dp2a_su(int a, unsigned b, int c, int hi)
{
    const int h0 = (int16_t)(a & 0xFFFF), h1 = (int16_t)((unsigned)a >> 16);
    const int b0 = (b >> (hi ? 16 : 0)) & 0xFF, b1 = (b >> (hi ? 24 : 8)) & 0xFF;
    return (int)((unsigned)c + (unsigned)(h0 * b0) + (unsigned)(h1 * b1));
}

// warp collective for kernels launched with emu_launch_warps: every lane is an OS thread, the barrier makes them meet
struct EmuWarp { std::barrier<> *bar; unsigned slots[32]; };
static thread_local EmuWarp *emu_warp = nullptr;
static inline unsigned __reduce_xor_sync(unsigned, unsigned v)
{
    EmuWarp *w = emu_warp;
    w->slots[threadIdx.x & 31] = v;
    w->bar->arrive_and_wait();
    unsigned r = 0;
    for (int i = 0; i < 32; i++) r ^= w->slots[i];
    w->bar->arrive_and_wait();
    return r;
}

// block-synchronous kernels (dynamic shared memory + __syncthreads): every thread of a block is an OS thread, one block at a time;
// a thread that returns drops out of the barrier like an exited CUDA thread
static thread_local std::barrier<> *emu_block_bar = nullptr;
static thread_local void *emu_smem = nullptr;
static inline void __syncthreads() { emu_block_bar->arrive_and_wait(); }
// warps inside a block launch (1-D blocks whose size is a multiple of 32, no thread leaves before the last collective): a barrier and
// 32 x 8 exchange words per warp
struct EmuBlockWarp { std::barrier<> *bar; unsigned slots[32][8]; };
static thread_local EmuBlockWarp *emu_bwarp = nullptr;
static inline unsigned emu_warp_xchg(unsigned v, int from_lane)
{
    EmuBlockWarp *w = emu_bwarp;
    w->slots[threadIdx.x & 31][0] = v;
    w->bar->arrive_and_wait();
    const unsigned r = w->slots[from_lane & 31][0];
    w->bar->arrive_and_wait();
    return r;
}
static inline int __shfl_xor_sync(unsigned, int v, int m) { return (int)emu_warp_xchg((unsigned)v, (threadIdx.x & 31) ^ m); }
static inline unsigned __shfl_xor_sync(unsigned, unsigned v, int m) { return emu_warp_xchg(v, (threadIdx.x & 31) ^ m); }
// mma.sync.aligned.m16n8k32.row.col.s32.u8.{s8,u8}.s32 by the PTX ISA fragment layouts: lane = 4 * groupID + tig;
//   A (16 x 32 u8): reg0 row groupID, k 4*tig..+3; reg1 row groupID + 8; reg2 / reg3 the same rows, k + 16
//   B (32 x 8):     reg0 k 4*tig..+3, column groupID; reg1 k + 16
//   D (16 x 8 s32): d0, d1 row groupID, columns 2*tig, 2*tig + 1; d2, d3 row groupID + 8
static inline void emu_mma_m16n8k32(int (&d)[4], const unsigned (&a)[4], unsigned b0, unsigned b1, bool b_signed)
{
    EmuBlockWarp *w = emu_bwarp;
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    for (int i = 0; i < 4; i++) w->slots[lane][i] = a[i];
    w->slots[lane][4] = b0; w->slots[lane][5] = b1;
    w->bar->arrive_and_wait();
    for (int i = 0; i < 4; i++) {
        const int row = g + (i >= 2 ? 8 : 0), col = 2 * t + (i & 1);
        long long acc = d[i];
        for (int k = 0; k < 32; k++) {
            const int al = (row & 7) * 4 + ((k & 15) >> 2), ar = (row >= 8 ? 1 : 0) + (k >= 16 ? 2 : 0);
            const int av = (w->slots[al][ar] >> (8 * (k & 3))) & 0xFF;
            const int bl = col * 4 + ((k & 15) >> 2);
            int bv = (w->slots[bl][4 + (k >= 16 ? 1 : 0)] >> (8 * (k & 3))) & 0xFF;
            if (b_signed && bv >= 128) bv -= 256;
            acc += (long long)av * bv;
        }
        d[i] = (int)acc;
    }
    w->bar->arrive_and_wait();
}
template <typename F> static void emu_launch_blocks(dim3 grid, dim3 block, size_t smem, F body)
{
    std::vector<unsigned char> shared(smem + 64);
    const unsigned nthreads = block.x * block.y * block.z, nwarps = (nthreads + 31) / 32;
    for (unsigned bz = 0; bz < grid.z; bz++) for (unsigned by = 0; by < grid.y; by++) for (unsigned bx = 0; bx < grid.x; bx++) {
        std::barrier<> bar(nthreads);
        std::vector<std::unique_ptr<std::barrier<>>> wbars;
        std::vector<EmuBlockWarp> warps(nwarps);
        for (unsigned wi = 0; wi < nwarps; wi++) {
            wbars.emplace_back(new std::barrier<>(std::min(32u, nthreads - 32 * wi)));
            warps[wi].bar = wbars.back().get();
        }
        std::vector<std::thread> th;
        for (unsigned tz = 0; tz < block.z; tz++) for (unsigned ty = 0; ty < block.y; ty++) for (unsigned tx = 0; tx < block.x; tx++)
            th.emplace_back([&, tx, ty, tz] {
                gridDim = grid; blockDim = block; blockIdx = dim3(bx, by, bz); threadIdx = dim3(tx, ty, tz);
                emu_block_bar = &bar; emu_smem = shared.data();
                emu_bwarp = &warps[(tx + block.x * (ty + block.y * tz)) / 32];
                body();
                bar.arrive_and_drop();
            });
        for (auto &t : th) t.join();
    }
}

// sequential launch: kernels without collectives or shared memory
template <typename F> static void emu_launch(dim3 grid, dim3 block, F body)
{
    gridDim = grid; blockDim = block;
    for (unsigned bz = 0; bz < grid.z; bz++) for (unsigned by = 0; by < grid.y; by++) for (unsigned bx = 0; bx < grid.x; bx++) {
        blockIdx = dim3(bx, by, bz);
        for (unsigned tz = 0; tz < block.z; tz++) for (unsigned ty = 0; ty < block.y; ty++) for (unsigned tx = 0; tx < block.x; tx++) {
            threadIdx = dim3(tx, ty, tz);
            body();
        }
    }
}

// one OS thread per lane, warp by warp (1-D blocks): for kernels that use __reduce_xor_sync
template <typename F> static void emu_launch_warps(dim3 grid, dim3 block, F body)
{
    for (unsigned bx = 0; bx < grid.x; bx++)
        for (unsigned w0 = 0; w0 < block.x; w0 += 32) {
            std::barrier<> bar(32);
            EmuWarp warp{ &bar, { 0 } };
            std::vector<std::thread> lanes;
            for (unsigned l = 0; l < 32; l++)
                lanes.emplace_back([&, l] {
                    gridDim = grid; blockDim = block; blockIdx = dim3(bx, 0, 0); threadIdx = dim3(w0 + l, 0, 0);
                    emu_warp = &warp;
                    body();
                });
            for (auto &t : lanes) t.join();
        }
}
