// hevcintra.cu — HEVC intra reconstruction of a whole picture on sm_90a: every intra TU of a picture, all three components, in decode
// order in one call, each TU's intra_pred (hevc/pred_template.c, hevcpred_dev.cuh) fused with the residual hls_transform_unit adds after
// it (hevc/cabac.c:1550-1592 and add_residual, hevcidct_dev.cuh).
//
// Picture kernel: one warp per op, 4 warps per CTA, each with its own shared memory and no CTA-wide barrier.  A warp takes ops by an
// atomicAdd ticket in decode order, so every op it waits on has a smaller ticket and is held by a warp that is already running: the
// smallest unfinished op can always proceed, whatever else shares the GPU.  A marking launch first records, per 4x4 cell of each plane,
// the op that writes it (-1: not written by an op of this call; TUs are at least 4x4 and 4-aligned in every chroma format).  Op t then
// waits, with acquire loads, only on the earlier ops of its plane that own a cell of what it reads: the left column from y - 1 down to
// the clipped bottom-left run when CAND_BL / L / UL is set, the top row from x - 1 to the clipped top-right run when CAND_U / UR / UL is
// set (constrained intra prediction only clears flags and substitutes inside these runs).  It then runs the five prediction stages with
// the edges read through L2, stores the predicted block, and, when the TU has a residual, runs the two transform passes in shared memory
// and adds and clips row by row over the block it stored.  A fence and a release store publish the op.  Every wait is bounded by about
// one second of %globaltimer: a scheduling mistake gives wrong samples, never a hung GPU, and each wait that runs out is counted for
// b200_hevc_intra_timeouts().
#include "common.h"
#include "hevcidct_dev.cuh"
#include "hevcpred_dev.cuh"
#include "wait_timeouts.h"
#include <cstring>

namespace {

constexpr int kWarps = 4;                                    // ops in flight per CTA
constexpr int kMaxCtas = 2048;                               // enough to fill the GPU; further warps would only find the tickets gone
constexpr unsigned long long kWaitNs = 1000000000ull;        // bound of one wait

struct ReconArgs {
    uint8_t *plane[3];
    long long ls[3];                                         // bytes
    PredPlane g[3];
    const B200HevcIntraReconOp *ops;
    const int16_t *coef;
    int *sync;                                               // [0] ticket, [1 + k] op k published
    int *owner[3];                                           // per plane, cell (cy, cx) at [cy * cw + cx]: the op that writes it, or -1
    int *timeouts;                                           // waits that ran out (b200_hevc_intra_timeouts)
    int cw[3];                                               // cells per row
    int nops, nplanes;
};

// ---- inter-warp progress
__device__ __forceinline__ int ld_acquire(const int *p)
{
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release(int *p, int v)
{
    asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long globaltimer()
{
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// ---- end of inter-warp progress

// the residual fields of an op as the shared passes read them
struct TuView {
    int col_limit, flags;
};

// the checks that make an op write nothing (those of both batch entries, plus the plane index and 4-aligned positions)
__device__ __forceinline__ bool recon_ok(const ReconArgs &a, const B200HevcIntraReconOp &op)
{
    if (op.plane >= a.nplanes || (op.x & 3) || (op.y & 3)) return false;
    if (!pred_op_ok(a.g[op.plane], op.x, op.y, op.log2_size, op.mode, op.flags)) return false;
    if (op.tu_kind == B200_HEVC_TU_NONE) return true;
    return op.tu_kind <= K_BYPASS && (op.tu_kind != K_DST4 || op.log2_size == 2) && op.coef_off >= 0 && !(op.coef_off & 7);
}

// the marking launch: each valid op's cells get its index.  The ops of a call write disjoint blocks (decode order gives that); where a
// caller's ops overlap anyway, the cell keeps the largest index, so the marks do not depend on which thread runs last
__global__ void hevc_recon_mark_kernel(const __grid_constant__ ReconArgs a)
{
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= a.nops) return;
    const B200HevcIntraReconOp op = a.ops[k];
    if (!recon_ok(a, op)) return;
    const int p = op.plane, n4 = 1 << (op.log2_size - 2);
    for (int cy = op.y >> 2; cy < (op.y >> 2) + n4; cy++)
        for (int cx = op.x >> 2; cx < (op.x >> 2) + n4; cx++) atomicMax(a.owner[p] + (long long)cy * a.cw[p] + cx, (int)k);
}

template <typename P, int N>
__device__ __forceinline__ void residual(const TuView &tv, int kind, int16_t *A, int16_t *B, P *dst, long long st, int depth, int lane)
{
    if (lane < N) pass1_col<N>(tv, kind, lane, A, B, depth);
    __syncwarp();
    if (lane < N) {
        int y[N];
        pass2_row<N>(tv, kind, lane, A, B, depth, y);
        P *d = dst + (long long)lane * st;
        const int maxv = (1 << depth) - 1;
#pragma unroll
        for (int j = 0; j < N; j += 4) add4<P>(d + j, y + j, maxv);
    }
}

template <typename P>
__global__ void __launch_bounds__(32 * kWarps) hevc_recon_kernel(const __grid_constant__ ReconArgs a)
{
    __shared__ int sE[kWarps][kWarpInts];
    __shared__ __align__(16) int16_t sA[kWarps][32 * 32];
    __shared__ int16_t sB[kWarps][32 * 34];
    __shared__ int sTicket[kWarps];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (;;) {
        if (lane == 0) sTicket[w] = atomicAdd(a.sync, 1);
        __syncwarp();
        const int t = sTicket[w];
        __syncwarp();
        if (t >= a.nops) break;
        const B200HevcIntraReconOp op = a.ops[t];
        if (recon_ok(a, op)) {
            const int p = op.plane, log2 = op.log2_size, size = 1 << log2, x = op.x, y = op.y, f = op.flags;
            const PredPlane &g = a.g[p];
            // wait for the ops that own the cells this op reads: the left column, then the top row (cell runs clipped to the plane)
            {
                const bool lft = f & (B200_HEVC_INTRA_CAND_BL | B200_HEVC_INTRA_CAND_L | B200_HEVC_INTRA_CAND_UL);
                const bool abv = f & (B200_HEVC_INTRA_CAND_UL | B200_HEVC_INTRA_CAND_U | B200_HEVC_INTRA_CAND_UR);
                const int l0 = max(y - 1, 0) >> 2, l1 = (min(y + 2 * size, g.ph) - 1) >> 2;
                const int t0 = max(x - 1, 0) >> 2, t1 = (min(x + 2 * size, g.pw) - 1) >> 2;
                const int nl = lft ? l1 - l0 + 1 : 0, nt = abv ? t1 - t0 + 1 : 0;
                for (int i = lane; i < nl + nt; i += 32) {
                    const int cy = i < nl ? l0 + i : (y - 1) >> 2, cx = i < nl ? (x - 1) >> 2 : t0 + i - nl;
                    const int o = a.owner[p][(long long)cy * a.cw[p] + cx];
                    if (o >= 0 && o < t && !ld_acquire(a.sync + 1 + o)) {
                        const unsigned long long start = globaltimer();
                        unsigned ns = 32;
                        while (!ld_acquire(a.sync + 1 + o) && globaltimer() - start < kWaitNs) {
                            __nanosleep(ns);
                            ns = min(ns * 2, 1024u);
                        }
                        if (!ld_acquire(a.sync + 1 + o)) atomicAdd(a.timeouts, 1);
                    }
                }
            }
            __syncwarp();
            const long long st = a.ls[p] / (long long)sizeof(P);
            P *src = reinterpret_cast<P *>(a.plane[p] + (long long)y * a.ls[p]) + x;
            intra_pred_op<P>(true, g, x, y, log2, op.mode, f, src, st, sE[w], lane, [] { __syncwarp(); },
                             [](const P *q) { return (int)__ldcg(q); });
            __syncwarp();                                    // the lanes' stores of the prediction before the add reads them
            if (op.tu_kind != B200_HEVC_TU_NONE) {
                int16_t *A = sA[w];
                const int16_t *c = a.coef + op.coef_off;
                for (int e = 8 * lane; e < size * size; e += 8 * 32)
                    *reinterpret_cast<int4 *>(A + e) = *reinterpret_cast<const int4 *>(c + e);
                __syncwarp();
                const TuView tv = { op.col_limit, op.tu_flags };
                switch (log2) {
                case 2:  residual<P, 4>(tv, op.tu_kind, A, sB[w], src, st, g.depth, lane); break;
                case 3:  residual<P, 8>(tv, op.tu_kind, A, sB[w], src, st, g.depth, lane); break;
                case 4:  residual<P, 16>(tv, op.tu_kind, A, sB[w], src, st, g.depth, lane); break;
                default: residual<P, 32>(tv, op.tu_kind, A, sB[w], src, st, g.depth, lane); break;
                }
            }
        }
        __threadfence();
        __syncwarp();
        // the ticket is read back from shared memory rather than kept in a register across the op: at the 32-point residual pass that
        // register is what ptxas would otherwise spill (168 registers either way)
        if (lane == 0) st_release(a.sync + 1 + sTicket[w], 1);
    }
}

bool depth_ok(int d) { return d == 8 || d == 9 || d == 10 || d == 12; }

} // namespace

B200_API int b200_hevc_intra_recon_picture_device(B200Device *dev, int bit_depth, int chroma_format_idc, int width, int height,
                                                  uint8_t *const planes[3], ptrdiff_t ls_y, ptrdiff_t ls_uv, int64_t nops,
                                                  const B200HevcIntraReconOp *ops, const int16_t *coef, const uint8_t *intra_map,
                                                  ptrdiff_t map_stride, int log2_min_pu_size)
{
    if (!depth_ok(bit_depth)) { b200_set_error("hevc intra picture: bit depth %d is not 8, 9, 10 or 12", bit_depth); return B200_EINVAL; }
    if (chroma_format_idc < 0 || chroma_format_idc > 3) { b200_set_error("hevc intra picture: chroma_format_idc %d", chroma_format_idc); return B200_EINVAL; }
    const int np = chroma_format_idc ? 3 : 1;
    if (!planes) { b200_set_error("hevc intra picture: NULL planes"); return B200_EINVAL; }
    for (int p = 0; p < np; p++)
        if (!planes[p]) { b200_set_error("hevc intra picture: NULL plane %d", p); return B200_EINVAL; }
    if (width < 1 || height < 1 || width > 65536 || height > 65536) { b200_set_error("hevc intra picture: %dx%d picture", width, height); return B200_EINVAL; }
    if (nops < 0 || nops > (1LL << 30)) { b200_set_error("hevc intra picture: nops %lld outside 0 .. 2^30", (long long)nops); return B200_EINVAL; }
    const int bps = bit_depth > 8 ? 2 : 1;
    const int hs = chroma_format_idc == 1 || chroma_format_idc == 2, vs = chroma_format_idc == 1;
    for (int p = 0; p < np; p++) {
        const long long ls = p ? ls_uv : ls_y, pw = p ? width >> hs : width;
        if (ls < pw * bps || ls % (4 * bps)) {
            b200_set_error("hevc intra picture: line size of plane %d shorter than a row or not a multiple of 4 samples", p);
            return B200_EINVAL;
        }
        if ((uintptr_t)planes[p] % (4 * bps)) { b200_set_error("hevc intra picture: plane %d not aligned to 4 samples", p); return B200_EINVAL; }
    }
    if (intra_map && (log2_min_pu_size < 2 || log2_min_pu_size > 6 || map_stride < (width >> log2_min_pu_size))) {
        b200_set_error("hevc intra picture: log2_min_pu_size %d or map_stride %lld does not fit the picture", log2_min_pu_size, (long long)map_stride);
        return B200_EINVAL;
    }
    if (nops == 0) return 0;
    if (!ops || !coef || ((uintptr_t)ops & 15) || ((uintptr_t)coef & 15)) {
        b200_set_error("hevc intra picture: ops / coef NULL or not aligned to 16 bytes");
        return B200_EINVAL;
    }
    if (int r = b200_use_device(dev)) return r;
    B200_LOCK_DEVICE(dev);
    int *timeouts = b200_wait_timeouts_word(dev->ordinal, B200_WAIT_HEVC_INTRA, true);
    if (!timeouts) { b200_set_error("hevc intra picture: no timeout counter for device %d", dev->ordinal); return B200_ENOMEM; }
    ReconArgs a;
    memset(&a, 0, sizeof(a));
    // scratch: the ticket and one published flag per op, then the cell maps
    size_t cells[3] = { 0, 0, 0 }, bytes = sizeof(int) * (((size_t)nops + 1 + 3) & ~(size_t)3);
    const size_t sync_bytes = bytes;
    for (int p = 0; p < np; p++) {
        PredPlane &g = a.g[p];
        g.map = intra_map; g.mstride = (long long)map_stride;
        g.W = width; g.H = height; g.hs = p ? hs : 0; g.vs = p ? vs : 0; g.pw = width >> g.hs; g.ph = height >> g.vs;
        g.log2_pu = intra_map ? log2_min_pu_size : 2;
        g.mpw = width >> g.log2_pu; g.mph = height >> g.log2_pu; g.depth = bit_depth;
        a.cw[p] = (g.pw + 3) >> 2;
        cells[p] = (size_t)a.cw[p] * (size_t)((g.ph + 3) >> 2);
        bytes += sizeof(int) * ((cells[p] + 3) & ~(size_t)3);
    }
    int *scr = (int *)b200_scratch(dev, bytes);
    if (!scr) return B200_ENOMEM;
    size_t off = sync_bytes / sizeof(int);
    for (int p = 0; p < np; p++) {
        a.plane[p] = planes[p];
        a.ls[p] = p ? ls_uv : ls_y;
        a.owner[p] = scr + off;
        off += (cells[p] + 3) & ~(size_t)3;
    }
    a.ops = ops;
    a.coef = coef;
    a.sync = scr;
    a.timeouts = timeouts;
    a.nops = (int)nops;
    a.nplanes = np;
    B200_CUDA_OK(cudaMemsetAsync(scr, 0, sync_bytes, dev->stream));
    B200_CUDA_OK(cudaMemsetAsync(a.owner[0], 0xFF, bytes - sync_bytes, dev->stream));
    hevc_recon_mark_kernel<<<(unsigned)((nops + 255) / 256), 256, 0, dev->stream>>>(a);
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    const long long ctas = (nops + kWarps - 1) / kWarps;
    const unsigned grid = (unsigned)(ctas < kMaxCtas ? ctas : kMaxCtas);
    if (bit_depth == 8) hevc_recon_kernel<uint8_t><<<grid, 32 * kWarps, 0, dev->stream>>>(a);
    else hevc_recon_kernel<uint16_t><<<grid, 32 * kWarps, 0, dev->stream>>>(a);
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

B200_API int b200_hevc_intra_timeouts(B200Device *dev, int64_t *count)
{
    if (!count) { b200_set_error("hevc intra timeouts: NULL pointer"); return B200_EINVAL; }
    if (int r = b200_use_device(dev)) return r;
    B200_CUDA_OK(cudaStreamSynchronize(dev->stream));
    int v = 0;
    int *w = b200_wait_timeouts_word(dev->ordinal, B200_WAIT_HEVC_INTRA, false);
    if (w) B200_CUDA_OK(cudaMemcpy(&v, w, sizeof(int), cudaMemcpyDeviceToHost));
    *count = v;
    return 0;
}
