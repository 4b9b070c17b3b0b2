// hevcidct.cu — HEVC residual reconstruction on sm_90a: the transform members of HEVCDSPContext (libavcodec/hevc/dsp.h:47-125:
// add_residual[4], dequant, transform_rdpcm, transform_4x4_luma, idct[4], idct_dc[4]) as ff_hevc_dsp_init fills them for 8, 9, 10 and
// 12 bit samples (hevc/dsp.c:198-215), and a batched device entry that runs the decoder's per-transform-unit sequence
// (hevc/cabac.c:1550-1592) followed by add_residual.
//
// Reference semantics reproduced bit for bit (checker: oracle/hevcidct_oracle.c), hevc/dsp_template.c:46-309:
//   idct N x N:  column pass then row pass, each clip16((sum + add) >> shift), shifts 7 and 20 - depth.  col_limit masks the odd inputs
//                of the partial butterflies: column c of the first pass sums odd rows j < L(c), L(0) = L0 = min(col_limit + 4, N),
//                L(c >= 1) = L0 - 4 ((c - 1) / 4) while below N (the reference's running limit2); every row of the second pass sums odd
//                columns j < min(col_limit, N); at 32 points the inner 16-point butterfly gets end / 2, which also masks j = 2 (mod 4)
//                by j / 2 < end / 2.  The 4x4 ignores col_limit.  Exact int32 sums, so the partial butterfly of the inputs with those
//                terms zeroed is the reference's result.
//   idct_dc:     every coefficient = (((c0 + 1) >> 1) + add) >> (14 - depth)
//   4x4 luma:    the DST butterfly TR_4x4_LUMA with the idct's shifts and clips
//   dequant:     (c + 2^(s - 1)) >> s, s = 15 - depth - log2; nothing for s == 0; (int16)((uint16)c << -s) for s < 0 (12 bit)
//   rdpcm:       running sums along rows (mode 0) or down columns (mode != 0), int16 wrap at every step
//   add:         dst = clip(dst + res, 0, 2^depth - 1)
//
// Kernel: a CTA of 256 threads takes a run of 1-256 ops (chosen from the batch size) and walks it in rounds of at most kCap
// coefficients.  A round loads its ops' coefficients into shared memory as 16-byte vectors, then runs two line passes over all its
// ops at once: pass 1 gives every thread one column of one op (the whole column transform in registers, clipped into a second shared
// array whose rows are padded to an odd number of words), pass 2 one row of one op (the row transform in registers, fused with the
// add, the clip and a store of whole 4-sample words of the destination).  A 32x32 TU is thus 32 threads' work per pass, a 4x4 TU four
// threads', and a run of small TUs fills the CTA as well as a few large ones do.  Nothing goes to global memory between the passes.
#include "common.h"
#include "hevcidct_dev.cuh"
#include <cstring>

namespace {

constexpr int kThreads = 256;
constexpr int kMaxOps = 256;                                 // ops per CTA
constexpr int kCap = 8192;                                   // coefficients per round
constexpr int kBCap = kCap + kCap / 2;                       // pass-1 array: N x (N + 2) per op, at most 1.5 N^2 (N = 4)
constexpr int kHead = 2 * (kMaxOps + 1) + 2 * kMaxOps + 2;  // ints in front of the coefficients (a multiple of 4: 16-byte aligned)
constexpr size_t kSmem = 4 * kHead + 2 * (kCap + kBCap);
struct TuArgs {
    const B200HevcTuOp *ops;
    long long nops;
    const int16_t *coef;
    uint8_t *dst;
    long long dst_stride;
    int16_t *res;                        // drop-in members: the int16 result goes here (at coef_off, N x N row-major) instead of dst
    int depth, ops_per_cta;
};

template <int N>
__device__ __forceinline__ void pass1(const B200HevcTuOp &op, int kind, int c, const int16_t *A, int16_t *B, int depth)
{
    pass1_col<N>(op, kind, c, A, B, depth);
}

template <typename P, int N>
__device__ __forceinline__ void pass2(const B200HevcTuOp &op, int kind, int r, const int16_t *A, const int16_t *B, const TuArgs &a)
{
    int y[N];
    pass2_row<N>(op, kind, r, A, B, a.depth, y);
    if (a.res) {
        int16_t *o = a.res + op.coef_off + r * N;
#pragma unroll
        for (int j = 0; j < N; j += 4)
            *reinterpret_cast<uint2 *>(o + j) = make_uint2((unsigned)(uint16_t)y[j] | (unsigned)y[j + 1] << 16,
                                                          (unsigned)(uint16_t)y[j + 2] | (unsigned)y[j + 3] << 16);
        return;
    }
    P *d = reinterpret_cast<P *>(a.dst + op.dst_off + (long long)r * a.dst_stride);
    const int maxv = (1 << a.depth) - 1;
#pragma unroll
    for (int j = 0; j < N; j += 4) add4<P>(d + j, y + j, maxv);
}

// the device-side guard: an op it refuses writes nothing
template <typename P>
__device__ __forceinline__ bool op_ok(const B200HevcTuOp &op, bool res_mode)
{
    if (op.log2_size < 2 || op.log2_size > 5 || op.kind > K_BYPASS || (op.kind == K_DST4 && op.log2_size != 2)) return false;
    if (op.coef_off & 7) return false;
    return res_mode || (op.dst_off & (4 * sizeof(P) - 1)) == 0;
}

// largest i in [lo, hi) with v[i] <= x (v non-decreasing, v[lo] <= x)
__device__ __forceinline__ int find(const int *v, int lo, int hi, int x)
{
    while (hi - lo > 1) {
        const int m = (lo + hi) >> 1;
        if (v[m] <= x) lo = m;
        else hi = m;
    }
    return lo;
}

template <typename P>
__global__ void __launch_bounds__(kThreads) hevc_tu_kernel(TuArgs a)
{
    extern __shared__ int4 hevc_tu_smem[];
    int *S = reinterpret_cast<int *>(hevc_tu_smem);          // [i] = first coefficient of op i in the CTA's run, [n] = total
    int *L = S + kMaxOps + 1;                                // [i] = first line of op i
    int *meta = L + kMaxOps + 1;                             // log2 | kind << 8, -1 for a refused op
    int *boff = meta + kMaxOps;                              // first element of op i in Bs, relative to its round
    int16_t *As = reinterpret_cast<int16_t *>(S + kHead), *Bs = As + kCap;
    const int tid = threadIdx.x;
    const long long o0 = (long long)blockIdx.x * a.ops_per_cta;
    const int n = (int)(a.nops - o0 < a.ops_per_cta ? a.nops - o0 : a.ops_per_cta);
    const B200HevcTuOp *ops = a.ops + o0;
    if (tid < n) {
        const B200HevcTuOp &op = ops[tid];
        const bool ok = op_ok<P>(op, a.res != nullptr);
        meta[tid] = ok ? op.log2_size | op.kind << 8 : -1;
        S[tid + 1] = ok ? 1 << (2 * op.log2_size) : 0;
        L[tid + 1] = ok ? 1 << op.log2_size : 0;
    }
    if (tid == 0) S[0] = L[0] = 0;
    __syncthreads();
    for (int d = 1; d < n; d <<= 1) {                        // inclusive scan of S[1..n], L[1..n]
        int s = 0, l = 0;
        if (tid < n && tid >= d) s = S[tid + 1 - d], l = L[tid + 1 - d];
        __syncthreads();
        if (tid < n && tid >= d) S[tid + 1] += s, L[tid + 1] += l;
        __syncthreads();
    }
    for (int r0 = 0; r0 < n;) {
        const int r1 = find(S, r0, n + 1, S[r0] + kCap);    // ops r0 .. r1 - 1 fit in a round (r1 > r0: an op is at most 1024)
        const int sa = S[r0], la = L[r0];
        for (int i = r0 + tid; i < r1; i += kThreads) boff[i] = S[i] - sa + 2 * (L[i] - la);
        const int nv = (S[r1] - sa) >> 3;
        for (int v = tid; v < nv; v += kThreads) {
            const int s = sa + 8 * v, i = find(S, r0, r1, s);
            const int4 q = *reinterpret_cast<const int4 *>(a.coef + ops[i].coef_off + (s - S[i]));
            *reinterpret_cast<int4 *>(As + (s - sa)) = q;
        }
        __syncthreads();
        const int nl = L[r1] - la;
        for (int t = tid; t < nl; t += kThreads) {
            const int i = find(L, r0, r1, la + t), m = meta[i], c = la + t - L[i];
            const int16_t *A = As + (S[i] - sa);
            int16_t *B = Bs + boff[i];
            switch (m & 0xFF) {
            case 2:  pass1<4>(ops[i], m >> 8, c, A, B, a.depth); break;
            case 3:  pass1<8>(ops[i], m >> 8, c, A, B, a.depth); break;
            case 4:  pass1<16>(ops[i], m >> 8, c, A, B, a.depth); break;
            default: pass1<32>(ops[i], m >> 8, c, A, B, a.depth); break;
            }
        }
        __syncthreads();
        for (int t = tid; t < nl; t += kThreads) {
            const int i = find(L, r0, r1, la + t), m = meta[i], r = la + t - L[i];
            const int16_t *A = As + (S[i] - sa), *B = Bs + boff[i];
            switch (m & 0xFF) {
            case 2:  pass2<P, 4>(ops[i], m >> 8, r, A, B, a); break;
            case 3:  pass2<P, 8>(ops[i], m >> 8, r, A, B, a); break;
            case 4:  pass2<P, 16>(ops[i], m >> 8, r, A, B, a); break;
            default: pass2<P, 32>(ops[i], m >> 8, r, A, B, a); break;
            }
        }
        __syncthreads();
        r0 = r1;
    }
}

constexpr long long kChunkOps = 1LL << 20;                   // ops per launch

bool depth_ok(int d) { return d == 8 || d == 9 || d == 10 || d == 12; }

cudaError_t launch(TuArgs a, cudaStream_t st)
{
    const long long nops = a.nops;
    const long long per = (nops + 1055) / 1056;             // about 8 CTAs per SM for a frame; 1 op per CTA for a few ops
    a.ops_per_cta = (int)(per < 1 ? 1 : per > kMaxOps ? kMaxOps : per);
    const B200HevcTuOp *ops = a.ops;
    for (long long b = 0; b < nops; b += kChunkOps) {
        a.ops = ops + b;
        a.nops = nops - b < kChunkOps ? nops - b : kChunkOps;
        const unsigned grid = (unsigned)((a.nops + a.ops_per_cta - 1) / a.ops_per_cta);
        if (a.depth == 8) hevc_tu_kernel<uint8_t><<<grid, kThreads, kSmem, st>>>(a);
        else hevc_tu_kernel<uint16_t><<<grid, kThreads, kSmem, st>>>(a);
        B200_LAUNCHED();
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// ---- drop-in members (host pointers): one op through the device scratch.  res != nullptr: the members that work in place on the
// coefficients (the kernel's int16 result is copied back over them); else add_residual (the block of dst is staged and copied back).
void member_host(int depth, int log2, int kind, int flags, int col_limit, int16_t *coeffs, const int16_t *res, uint8_t *dst, ptrdiff_t stride)
{
    const int N = 1 << log2, bps = depth > 8 ? 2 : 1;
    const size_t cbytes = (size_t)N * N * sizeof(int16_t), dpitch = (size_t)N * bps;
    B200HostCall call("hevc transform", nullptr, 256 + 3 * 2048);
    uint8_t *scr = call.scratch;
    cudaStream_t st = call.stream;
    uint8_t *dop = scr, *dcoef = scr + 256, *dres = dcoef + 2048, *ddst = dres + 2048;
    B200HevcTuOp op;
    memset(&op, 0, sizeof(op));
    op.log2_size = (uint8_t)log2;
    op.kind = (uint8_t)kind;
    op.flags = (uint8_t)flags;
    op.col_limit = col_limit;
    call.check(cudaMemcpyAsync(dop, &op, sizeof(op), cudaMemcpyHostToDevice, st), "h2d op");
    call.check(cudaMemcpyAsync(dcoef, coeffs ? coeffs : res, cbytes, cudaMemcpyHostToDevice, st), "h2d coefficients");
    if (!coeffs) call.check(b200_h2d_rows(ddst, dpitch, dst, stride, dpitch, (size_t)N, st), "h2d block");
    TuArgs a = { (const B200HevcTuOp *)dop, 1, (const int16_t *)dcoef, ddst, (long long)dpitch, coeffs ? (int16_t *)dres : nullptr, depth, 1 };
    call.check(launch(a, st), "launch");
    if (coeffs) call.check(cudaMemcpyAsync(coeffs, dres, cbytes, cudaMemcpyDeviceToHost, st), "d2h coefficients");
    else call.check(b200_d2h_rows(dst, stride, ddst, dpitch, dpitch, (size_t)N, st), "d2h block");
    call.sync();
}

bool log2_ok(int log2, const char *who)
{
    if (log2 >= 2 && log2 <= 5) return true;
    b200_set_error("hevc %s: log2_size %d outside 2..5, nothing written", who, log2);
    return false;
}

template <int D, int LOG2>
void m_add_residual(uint8_t *dst, const int16_t *res, ptrdiff_t stride) { member_host(D, LOG2, K_BYPASS, 0, 0, nullptr, res, dst, stride); }
template <int D>
void m_dequant(int16_t *coeffs, int16_t log2)
{
    if (log2_ok(log2, "dequant")) member_host(D, log2, K_SKIP, 0, 0, coeffs, nullptr, nullptr, 0);
}
template <int D>
void m_rdpcm(int16_t *coeffs, int16_t log2, int mode)
{
    if (log2_ok(log2, "transform_rdpcm"))
        member_host(D, log2, K_BYPASS, B200_HEVC_TU_RDPCM | (mode ? B200_HEVC_TU_RDPCM_VER : 0), 0, coeffs, nullptr, nullptr, 0);
}
template <int D>
void m_dst4(int16_t *coeffs) { member_host(D, 2, K_DST4, 0, 0, coeffs, nullptr, nullptr, 0); }
template <int D, int LOG2>
void m_idct(int16_t *coeffs, int col_limit) { member_host(D, LOG2, K_IDCT, 0, col_limit, coeffs, nullptr, nullptr, 0); }
template <int D, int LOG2>
void m_idct_dc(int16_t *coeffs) { member_host(D, LOG2, K_DC, 0, 0, coeffs, nullptr, nullptr, 0); }

template <int D, int LOG2>
void fill_size(B200HEVCDSPContext *c)
{
    c->add_residual[LOG2 - 2] = m_add_residual<D, LOG2>;
    c->idct[LOG2 - 2] = m_idct<D, LOG2>;
    c->idct_dc[LOG2 - 2] = m_idct_dc<D, LOG2>;
}
// hevc/dsp.c:198-215
template <int D>
void fill(B200HEVCDSPContext *c)
{
    fill_size<D, 2>(c);
    fill_size<D, 3>(c);
    fill_size<D, 4>(c);
    fill_size<D, 5>(c);
    c->dequant = m_dequant<D>;
    c->transform_rdpcm = m_rdpcm<D>;
    c->transform_4x4_luma = m_dst4<D>;
}

} // namespace

B200_API int b200_hevc_dsp_init_transform(B200HEVCDSPContext *c, int bit_depth)
{
    if (!c) return B200_EINVAL;
    if (!depth_ok(bit_depth)) return B200_ENOSYS;
    if (!b200_default_device()) return B200_ENODEV;
    switch (bit_depth) {
    case 8:  fill<8>(c); break;
    case 9:  fill<9>(c); break;
    case 10: fill<10>(c); break;
    default: fill<12>(c); break;
    }
    return 0;
}

B200_API int b200_hevc_transform_add_batch_device(B200Device *dev, int bit_depth, int64_t nops, const B200HevcTuOp *ops, const int16_t *coef,
                                                  uint8_t *dst, ptrdiff_t dst_stride)
{
    if (nops < 0) { b200_set_error("hevc transform batch: negative nops"); return B200_EINVAL; }
    if (!depth_ok(bit_depth)) { b200_set_error("hevc transform batch: bit depth %d is not 8, 9, 10 or 12", bit_depth); return B200_EINVAL; }
    const int bps = bit_depth > 8 ? 2 : 1;
    if (dst_stride % (4 * bps)) { b200_set_error("hevc transform batch: dst_stride not a multiple of 4 samples"); return B200_EINVAL; }
    if (nops == 0) return 0;
    if (!ops || !coef || !dst || ((uintptr_t)ops & 15) || ((uintptr_t)coef & 15) || ((uintptr_t)dst % (4 * bps))) {
        b200_set_error("hevc transform batch: NULL or misaligned pointer");
        return B200_EINVAL;
    }
    if (int r = b200_use_device(dev)) return r;
    TuArgs a = { ops, (long long)nops, coef, dst, (long long)dst_stride, nullptr, bit_depth, 1 };
    B200_CUDA_OK(launch(a, dev->stream));
    return 0;
}
