// hevcpred.cu — HEVC intra prediction on sm_90a: the members of HEVCPredContext (libavcodec/hevc/pred.h) that ff_hevc_pred_init fills
// (pred_planar[4], pred_dc, pred_angular[4], ref_filter_3tap[3], ref_filter_strong; intra_pred[] takes decoder structs and stays NULL)
// for 8, 9, 10 and 12 bit samples, and a batched entry that runs intra_pred (hevc/pred_template.c) for a set of independent TUs.
//
// Per op, the kernel follows intra_pred's data flow (hevcpred_dev.cuh, shared with hevcintra.cu), bit for bit (checked against the reference's own intra_pred, tests/test_hevc_pred.py):
//   1. neighbours: the left column left[-1..2 * size - 1] and the top row top[-1..2 * size - 1] in shared memory, taken from the plane
//      where the op's CAND_* flags allow (the bottom-left and top-right runs clipped to the picture and extended with their last sample);
//   2. constrained intra prediction (intra_map given): the PU checks that can clear a flag, the arrays preset to the byte 128, and the
//      substitution over the intra / inter map, lane-serial (CIP streams are rare), with the reference's quirks;
//   3. the substitution of unavailable runs, in closed form: in the scan order bottom-left, left, corner, top, top-right, an unavailable
//      run takes the last sample of the nearest available run before it, or the first sample of the first available run when none is
//      before it, and every sample is 1 << (depth - 1) when no run is available (the reference's if-chain, pred_template.c:296-332);
//   4. the filter decision and the 3-tap or strong filter;
//   5. planar / DC / angular, each lane computing runs of 4 samples and storing them as one word where aligned.
// A CTA of 4 warps takes 4 ops, one warp each.
#include "common.h"
#include "hevcpred_dev.cuh"
#include <cstring>
#include <type_traits>

namespace {

constexpr int kOpsPerCta = 4;
struct IntraArgs {
    uint8_t *pix;
    long long stride;                            // bytes
    const B200HevcIntraOp *ops;
    long long nops;
    PredPlane g;
};

// 10 CTAs per SM: the register budget of 48 the kernel had before its stages moved to hevcpred_dev.cuh; left to itself ptxas now
// settles on 40 and spills a predicate
template <typename P>
__global__ void __launch_bounds__(32 * kOpsPerCta, 10) hevc_intra_kernel(IntraArgs a)
{
    extern __shared__ int ipred_smem[];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long o = (long long)blockIdx.x * kOpsPerCta + w;
    B200HevcIntraOp op;
    memset(&op, 0, sizeof(op));
    if (o < a.nops) {
        const uint4 raw = __ldg(reinterpret_cast<const uint4 *>(a.ops + o));
        memcpy(&op, &raw, sizeof(op));
    }
    const int log2 = op.log2_size, mode = op.mode, f = op.flags;
    const bool act = o < a.nops && pred_op_ok(a.g, op.x, op.y, log2, mode, f);
    const long long st = a.stride / (long long)sizeof(P);
    P *src = act ? reinterpret_cast<P *>(a.pix + (long long)op.y * a.stride) + op.x : nullptr;
    intra_pred_op<P>(act, a.g, op.x, op.y, log2, mode, f, src, st, ipred_smem + w * kWarpInts, lane, [] { __syncthreads(); },
                     [](const P *p) { return (int)*p; });
}

// the prediction stage alone, for the members: one warp, top / left staged as int arrays of kArr elements (index -1 at kPad)
template <typename P>
__global__ void __launch_bounds__(32) hevc_pred_member_kernel(const int *staged, P *dst, long long st, int log2, int mode, int luma, int depth)
{
    extern __shared__ int ipred_smem[];
    int *left = ipred_smem + kPad + 1, *top = left + kArr, *R = top + kArr;
    for (int i = threadIdx.x; i < 2 * kArr; i += 32) ipred_smem[i] = staged[i];
    __syncthreads();
    predict<P>(true, top, left, R, dst, st, log2, mode, luma != 0, depth, threadIdx.x, [] { __syncthreads(); });
}

bool depth_ok(int d) { return d == 8 || d == 9 || d == 10 || d == 12; }

constexpr long long kChunkOps = 1LL << 24;
constexpr size_t kSmem = (size_t)kOpsPerCta * kWarpInts * sizeof(int);

cudaError_t launch_batch(IntraArgs a, cudaStream_t st)
{
    const long long nops = a.nops;
    const B200HevcIntraOp *ops = a.ops;
    for (long long b = 0; b < nops; b += kChunkOps) {
        a.ops = ops + b;
        a.nops = nops - b < kChunkOps ? nops - b : kChunkOps;
        const unsigned grid = (unsigned)((a.nops + kOpsPerCta - 1) / kOpsPerCta);
        if (a.g.depth == 8) hevc_intra_kernel<uint8_t><<<grid, 32 * kOpsPerCta, kSmem, st>>>(a);
        else hevc_intra_kernel<uint16_t><<<grid, 32 * kOpsPerCta, kSmem, st>>>(a);
        B200_LAUNCHED();
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// ---- prediction members (host pointers): top[t0..t1) and left[t0..t1) staged (index -1 = the corner), the block predicted into a
// scratch block and copied back.  `stride` is in samples, as intra_pred passes it (linesize / sizeof(pixel)).
template <int D>
void member_run(uint8_t *dst, ptrdiff_t stride, const uint8_t *top_, const uint8_t *left_, int log2, int mode, int c_idx, int t0, int t1)
{
    typedef typename std::conditional<D == 8, uint8_t, uint16_t>::type P;
    const P *top = reinterpret_cast<const P *>(top_), *left = reinterpret_cast<const P *>(left_);
    const int size = 1 << log2;
    int staged[2 * kArr];
    memset(staged, 0, sizeof(staged));
    for (int i = t0; i < t1; i++) {
        staged[kPad + 1 + i] = left[i];
        staged[kArr + kPad + 1 + i] = top[i];
    }
    const size_t blk = (size_t)size * size * sizeof(P);
    B200HostCall call("hevc intra prediction", nullptr, sizeof(staged) + blk);
    uint8_t *scr = call.scratch;
    cudaStream_t st = call.stream;
    call.check(cudaMemcpyAsync(scr, staged, sizeof(staged), cudaMemcpyHostToDevice, st), "h2d edges");
    P *sdst = reinterpret_cast<P *>(scr + sizeof(staged));
    hevc_pred_member_kernel<P><<<1, 32, (2 * kArr + kRef) * sizeof(int), st>>>((const int *)scr, sdst, size, log2, mode, c_idx == 0, D);
    B200_LAUNCHED();
    call.launched();
    call.check(b200_d2h_rows(dst, stride * (ptrdiff_t)sizeof(P), sdst, (size_t)size * sizeof(P), (size_t)size * sizeof(P), (size_t)size, st), "d2h block");
    call.sync();
}

template <int D, int L2>
void m_planar(uint8_t *src, const uint8_t *top, const uint8_t *left, ptrdiff_t stride)
{
    member_run<D>(src, stride, top, left, L2, 0, 0, 0, (1 << L2) + 1);
}

template <int D>
void m_dc(uint8_t *src, const uint8_t *top, const uint8_t *left, ptrdiff_t stride, int log2_size, int c_idx)
{
    if (log2_size < 2 || log2_size > 5) { b200_set_error("hevc pred_dc: log2_size %d is not 2..5", log2_size); return; }
    member_run<D>(src, stride, top, left, log2_size, 1, c_idx, 0, 1 << log2_size);
}

template <int D, int L2>
void m_angular(uint8_t *src, const uint8_t *top, const uint8_t *left, ptrdiff_t stride, int c_idx, int mode)
{
    if (mode < 2 || mode > 34) { b200_set_error("hevc pred_angular: mode %d is not 2..34", mode); return; }
    member_run<D>(src, stride, top, left, L2, mode, c_idx, -1, 2 << L2);
}

// ---- filter members: host only, the kernel's filter functions
template <int D>
void m_filter_3tap(uint8_t *filtered_left, uint8_t *filtered_top, const uint8_t *left_, const uint8_t *top_, int size)
{
    typedef typename std::conditional<D == 8, uint8_t, uint16_t>::type P;
    P *fl = reinterpret_cast<P *>(filtered_left), *ft = reinterpret_cast<P *>(filtered_top);
    const P *left = reinterpret_cast<const P *>(left_), *top = reinterpret_cast<const P *>(top_);
    const int n = 2 * size;
    fl[n - 1] = left[n - 1];
    ft[n - 1] = top[n - 1];
    for (int i = n - 2; i >= 0; i--) fl[i] = (P)filt3(left, i, n);
    ft[-1] = fl[-1] = (P)filt3_corner(left, top);
    for (int i = n - 2; i >= 0; i--) ft[i] = (P)filt3(top, i, n);
}

template <int D>
void m_filter_strong(uint8_t *filtered_top, uint8_t *left_, const uint8_t *top_)
{
    typedef typename std::conditional<D == 8, uint8_t, uint16_t>::type P;
    P *ft = reinterpret_cast<P *>(filtered_top), *left = reinterpret_cast<P *>(left_);
    const P *top = reinterpret_cast<const P *>(top_);
    ft[-1] = top[-1];
    ft[63] = top[63];
    for (int i = 0; i < 63; i++) ft[i] = (P)strong_at(top, i);
    for (int i = 0; i < 63; i++) left[i] = (P)strong_at(left, i);
}

template <int D>
void fill(B200HEVCPredContext *h)
{
    h->pred_planar[0] = m_planar<D, 2>;
    h->pred_planar[1] = m_planar<D, 3>;
    h->pred_planar[2] = m_planar<D, 4>;
    h->pred_planar[3] = m_planar<D, 5>;
    h->pred_dc = m_dc<D>;
    h->pred_angular[0] = m_angular<D, 2>;
    h->pred_angular[1] = m_angular<D, 3>;
    h->pred_angular[2] = m_angular<D, 4>;
    h->pred_angular[3] = m_angular<D, 5>;
    for (int k = 0; k < 3; k++) h->ref_filter_3tap[k] = m_filter_3tap<D>;
    h->ref_filter_strong = m_filter_strong<D>;
}

} // namespace

B200_API int b200_hevc_pred_init(B200HEVCPredContext *hpc, int bit_depth)
{
    if (!hpc) return B200_EINVAL;
    if (!depth_ok(bit_depth)) return B200_ENOSYS;
    if (!b200_default_device()) return B200_ENODEV;
    memset(hpc, 0, sizeof(*hpc));                                        // intra_pred[] stays NULL
    switch (bit_depth) {
    case 8:  fill<8>(hpc); break;
    case 9:  fill<9>(hpc); break;
    case 10: fill<10>(hpc); break;
    default: fill<12>(hpc); break;
    }
    return 0;
}

B200_API int b200_hevc_intra_pred_batch_device(B200Device *dev, int bit_depth, uint8_t *pix, ptrdiff_t stride, int width, int height, int hshift,
                                               int vshift, int64_t nops, const B200HevcIntraOp *ops, const uint8_t *intra_map,
                                               ptrdiff_t map_stride, int log2_min_pu_size)
{
    if (!depth_ok(bit_depth)) { b200_set_error("hevc intra batch: bit depth %d is not 8, 9, 10 or 12", bit_depth); return B200_EINVAL; }
    if (nops < 0) { b200_set_error("hevc intra batch: nops %lld < 0", (long long)nops); return B200_EINVAL; }
    if (width < 1 || height < 1) { b200_set_error("hevc intra batch: %dx%d is empty", width, height); return B200_EINVAL; }
    if ((hshift != 0 && hshift != 1) || (vshift != 0 && vshift != 1)) {
        b200_set_error("hevc intra batch: shifts %d, %d are not 0 or 1", hshift, vshift);
        return B200_EINVAL;
    }
    const int bps = bit_depth > 8 ? 2 : 1;
    if (stride < (ptrdiff_t)(width >> hshift) * bps || stride % bps) {
        b200_set_error("hevc intra batch: stride shorter than a plane row or not a whole number of samples");
        return B200_EINVAL;
    }
    if (intra_map && (log2_min_pu_size < 2 || log2_min_pu_size > 6 || map_stride < (width >> log2_min_pu_size))) {
        b200_set_error("hevc intra batch: log2_min_pu_size %d or map_stride %lld does not fit the picture", log2_min_pu_size, (long long)map_stride);
        return B200_EINVAL;
    }
    if (nops == 0) return 0;
    if (!pix || !ops || (uintptr_t)pix % bps || (uintptr_t)ops % 16) {
        b200_set_error("hevc intra batch: NULL pix / ops, pix not aligned to a sample or ops not aligned to 16 bytes");
        return B200_EINVAL;
    }
    if (int r = b200_use_device(dev)) return r;
    IntraArgs a;
    a.pix = pix; a.stride = (long long)stride; a.ops = ops; a.nops = nops;
    PredPlane &g = a.g;
    g.map = intra_map; g.mstride = (long long)map_stride;
    g.W = width; g.H = height; g.hs = hshift; g.vs = vshift; g.pw = width >> hshift; g.ph = height >> vshift;
    g.log2_pu = intra_map ? log2_min_pu_size : 2;
    g.mpw = width >> g.log2_pu; g.mph = height >> g.log2_pu; g.depth = bit_depth;
    B200_CUDA_OK(launch_batch(a, dev->stream));
    return 0;
}
