// vp9itxfm.cu — VP9 residual reconstruction on sm_90a: the itxfm_add[5][4] members of VP9DSPContext (libavcodec/vp9dsp.h:40-122) as
// vp9dsp_itxfm_init fills them for 8, 10 and 12 bit samples (vp9dsp_template.c:1755-1778), and a batched device entry that runs one
// member call per transform block, which is inter_recon's residual loop (vp9recon.c:608-652).
//
// Reference semantics reproduced bit for bit for any coefficient values (checker: oracle/vp9itxfm_oracle.c), vp9dsp_template.c:1155-1753:
//   [tx 0..2][type]  pass 1 = type a on every column of the dense sz x sz block, pass 2 = type b on every column of pass 1's result, with
//                    DCT_DCT idct / idct, DCT_ADST iadst / idct, ADST_DCT idct / iadst, ADST_ADST iadst / iadst; [3][*] idct / idct at
//                    32 points, [4][*] the Walsh-Hadamard transform (pass 1 takes its inputs >> 2, pass 2 as they are)
//   storage          8 bit: coefficients and both passes' results int16, arithmetic in 32 bits (wrapping: the multiplications are
//                    unsigned in the reference); 10 / 12 bit: int32 coefficients and results, arithmetic in int64 (no overflow for any
//                    int32 input).  The Walsh-Hadamard transform works in 32-bit ints at every depth.
//   add              output j of pass 2 for column i goes to dst row j, column i: clip(dst + ((int)(out + 2^(bits - 1)) >> bits)),
//                    bits 4 / 5 / 6 / 6 by size, no shift for the Walsh-Hadamard transform
//   DC only          idct / idct at 4..16 and every 32x32 slot with eob == 1: t = ((c0 * 11585 + 2^13) >> 14) * 11585 + 2^13) >> 14
//                    truncated to int, added to every sample; only c0 is read (and cleared by the members)
// The butterflies follow the VP9 bitstream specification's inverse DCT (an N-point DCT is the N/2-point DCT of the even inputs plus an
// odd part of rotations by cospi_k_64 = round(2^14 cos(k pi / 64))) and inverse ADST (rotations by cospi_k_64, rounded after the
// sums, and the 4-point ADST from sinpi_k_9), with every rounding (x + 2^13) >> 14 where the reference rounds.
//
// Kernel: hevcidct.cu's work distribution.  A CTA of 256 threads takes a run of 1-256 ops (chosen from the batch size) and walks it in
// rounds of at most kCap coefficients.  A round loads its ops' coefficients into shared memory as 16-byte vectors (only the first
// vector of a DC-only op), then runs three line passes over all its ops at once: pass 1 gives every thread one column of one op (the
// whole 1-D transform in registers, truncated to the storage type into a second shared array whose rows are padded to an odd number of
// words); pass 2 one column of that result (the second transform in registers, the rounding shift, the residual written back over the
// op's coefficients, which pass 1 has consumed); pass 3 one destination row (the add, the clip and a store of whole 4-sample words).
// Pass 2's thread owns a destination column (the reference adds output j of column i to row j), so the residual goes through shared
// memory once more to be stored row by row in whole words.  Nothing goes to global memory between the passes.
#include "common.h"
#include "vp9itxfm_dev.cuh"
#include <cstring>

namespace {

constexpr int kThreads = 256;
constexpr int kMaxOps = 256;                                 // ops per CTA
constexpr int kHead = 2 * (kMaxOps + 1) + 2 * kMaxOps + 2;  // ints in front of the coefficients (a multiple of 4: 16-byte aligned)
template <typename P> constexpr int bcap() { return Store<P>::kCap + Store<P>::kCap / 4 * Store<P>::kPad; }   // N (N + pad) <= this share
template <typename P> constexpr size_t smem_bytes()
{
    return 4 * kHead + sizeof(typename Store<P>::C) * Store<P>::kCap + sizeof(typename Store<P>::Tmp) * bcap<P>();
}

struct ItxArgs {
    const B200Vp9TxOp *ops;
    long long nops;
    const void *coef;
    uint8_t *dst;
    long long dst_stride;
    int depth, ops_per_cta;
};

// meta of an op: log2 size | type a << 8 | type b << 10 | DC only << 12 | bits << 13; -1 for an op the guard refuses
__host__ __device__ __forceinline__ bool dc_only(int tx, int type, int eob) { return eob == 1 && (tx == 3 || (tx < 3 && type == 0)); }

template <typename P>
__device__ __forceinline__ int op_meta(const B200Vp9TxOp &op)
{
    if (op.tx > 4 || op.type > 3 || (op.coef_off & 15) || (op.dst_off & (4 * sizeof(P) - 1))) return -1;
    const int tx = op.tx;
    if (tx == 4) return 2 | T_WHT << 8 | T_WHT << 10;
    const int ta = tx == 3 ? T_DCT : (op.type & 1) ? T_ADST : T_DCT;
    const int tb = tx == 3 ? T_DCT : (op.type & 2) ? T_ADST : T_DCT;
    return (tx + 2) | ta << 8 | tb << 10 | (dc_only(tx, op.type, op.eob) ? 1 << 12 : 0) | (tx < 2 ? 4 + tx : 6) << 13;
}

template <typename P, int N>
__device__ __forceinline__ void pass1(int m, int c, const typename Store<P>::C *A, typename Store<P>::Tmp *B)
{
    using C = typename Store<P>::C;
    constexpr int pitch = N + Store<P>::kPad;
    C x[N];
    typename Store<P>::Tmp y[N];
#pragma unroll
    for (int k = 0; k < N; k++) x[k] = A[k * N + c];
    tx1d<P, N>((m >> 8) & 3, true, x, y);
#pragma unroll
    for (int k = 0; k < N; k++) B[k * pitch + c] = y[k];          // row k of B = output k of every column
}

template <typename P, int N>
__device__ __forceinline__ void pass2(int m, int i, typename Store<P>::C *A, const typename Store<P>::Tmp *B)
{
    using C = typename Store<P>::C;
    constexpr int pitch = N + Store<P>::kPad;
    typename Store<P>::Tmp x[N], y[N];
#pragma unroll
    for (int k = 0; k < N; k++) x[k] = B[i * pitch + k];          // output i of column k of pass 1
    tx1d<P, N>((m >> 10) & 3, false, x, y);
    const int bits = m >> 13;
#pragma unroll
    for (int j = 0; j < N; j++)
        A[j * N + i] = bits ? (C)((int)((unsigned)(int)y[j] + (1u << (bits - 1))) >> bits) : y[j];
}

// one destination word of 4 samples: load, add (32-bit wrapping, as the reference's int sum), clip, store
template <typename P>
__device__ __forceinline__ void add4(P *d, const int *r, int maxv)
{
    auto px = [maxv](int s, int v) { return (unsigned)min(max((int)((unsigned)s + (unsigned)v), 0), maxv); };
    if constexpr (sizeof(P) == 1) {
        const unsigned w = *reinterpret_cast<const unsigned *>(d);
        unsigned o = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) o |= px((w >> (8 * k)) & 0xFF, r[k]) << (8 * k);
        *reinterpret_cast<unsigned *>(d) = o;
    } else {
        const uint2 w = *reinterpret_cast<const uint2 *>(d);
        uint2 o;
        o.x = px(w.x & 0xFFFF, r[0]) | px(w.x >> 16, r[1]) << 16;
        o.y = px(w.y & 0xFFFF, r[2]) | px(w.y >> 16, r[3]) << 16;
        *reinterpret_cast<uint2 *>(d) = o;
    }
}

template <typename P, int N>
__device__ __forceinline__ void pass3(int m, int j, long long dst_off, const typename Store<P>::C *A, const ItxArgs &a)
{
    using T = typename Store<P>::T;
    int r[N];
    if (m & (1 << 12)) {
        const T t1 = r14(mul((T)A[0], 11585));
        const int t = (int)r14(mul(t1, 11585));                   // the reference's `const int t`
        const int bits = m >> 13;
        const int v = (int)((unsigned)t + (1u << (bits - 1))) >> bits;
#pragma unroll
        for (int k = 0; k < N; k++) r[k] = v;
    } else {
#pragma unroll
        for (int k = 0; k < N; k++) r[k] = A[j * N + k];
    }
    P *d = reinterpret_cast<P *>(a.dst + dst_off + (long long)j * a.dst_stride);
    const int maxv = (1 << a.depth) - 1;
#pragma unroll
    for (int k = 0; k < N; k += 4) add4<P>(d + k, r + k, maxv);
}

// largest i in [lo, hi) with v[i] <= x (v non-decreasing, v[lo] <= x)
__device__ __forceinline__ int find(const int *v, int lo, int hi, int x)
{
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (v[mid] <= x) lo = mid;
        else hi = mid;
    }
    return lo;
}

template <typename P>
__global__ void __launch_bounds__(kThreads) vp9_itx_kernel(ItxArgs a)
{
    using C = typename Store<P>::C;
    constexpr int kCap = Store<P>::kCap, kPad = Store<P>::kPad, kVec = 16 / sizeof(C);
    extern __shared__ int4 vp9_itx_smem[];
    int *S = reinterpret_cast<int *>(vp9_itx_smem);          // [i] = first coefficient of op i in the CTA's run, [n] = total
    int *L = S + kMaxOps + 1;                                // [i] = first line of op i
    int *meta = L + kMaxOps + 1;                             // op_meta
    int *boff = meta + kMaxOps;                              // first element of op i in Bs, relative to its round
    using Tmp = typename Store<P>::Tmp;
    C *As = reinterpret_cast<C *>(S + kHead);
    Tmp *Bs = reinterpret_cast<Tmp *>(As + kCap);
    const C *coef = reinterpret_cast<const C *>(a.coef);
    const int tid = threadIdx.x;
    const long long o0 = (long long)blockIdx.x * a.ops_per_cta;
    const int n = (int)(a.nops - o0 < a.ops_per_cta ? a.nops - o0 : a.ops_per_cta);
    const B200Vp9TxOp *ops = a.ops + o0;
    if (tid < n) {
        const int m = op_meta<P>(ops[tid]);
        const int l2 = m < 0 ? 0 : m & 0xFF;
        meta[tid] = m;
        S[tid + 1] = m < 0 ? 0 : 1 << (2 * l2);
        L[tid + 1] = m < 0 ? 0 : 1 << l2;
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
        for (int i = r0 + tid; i < r1; i += kThreads) boff[i] = S[i] - sa + kPad * (L[i] - la);
        const int nv = (S[r1] - sa) / kVec;
        for (int v = tid; v < nv; v += kThreads) {
            const int s = sa + kVec * v, i = find(S, r0, r1, s);
            if ((meta[i] & (1 << 12)) && s != S[i]) continue;   // a DC-only op reads its first coefficient
            const int4 q = *reinterpret_cast<const int4 *>(coef + ops[i].coef_off + (s - S[i]));
            *reinterpret_cast<int4 *>(As + (s - sa)) = q;
        }
        __syncthreads();
        const int nl = L[r1] - la;
        for (int t = tid; t < nl; t += kThreads) {
            const int i = find(L, r0, r1, la + t), m = meta[i], c = la + t - L[i];
            if (m & (1 << 12)) continue;
            const C *A = As + (S[i] - sa);
            Tmp *B = Bs + boff[i];
            switch (m & 0xFF) {
            case 2:  pass1<P, 4>(m, c, A, B); break;
            case 3:  pass1<P, 8>(m, c, A, B); break;
            case 4:  pass1<P, 16>(m, c, A, B); break;
            default: pass1<P, 32>(m, c, A, B); break;
            }
        }
        __syncthreads();
        for (int t = tid; t < nl; t += kThreads) {
            const int i = find(L, r0, r1, la + t), m = meta[i], c = la + t - L[i];
            if (m & (1 << 12)) continue;
            C *A = As + (S[i] - sa);
            const Tmp *B = Bs + boff[i];
            switch (m & 0xFF) {
            case 2:  pass2<P, 4>(m, c, A, B); break;
            case 3:  pass2<P, 8>(m, c, A, B); break;
            case 4:  pass2<P, 16>(m, c, A, B); break;
            default: pass2<P, 32>(m, c, A, B); break;
            }
        }
        __syncthreads();
        for (int t = tid; t < nl; t += kThreads) {
            const int i = find(L, r0, r1, la + t), m = meta[i], j = la + t - L[i];
            const C *A = As + (S[i] - sa);
            const long long off = ops[i].dst_off;
            switch (m & 0xFF) {
            case 2:  pass3<P, 4>(m, j, off, A, a); break;
            case 3:  pass3<P, 8>(m, j, off, A, a); break;
            case 4:  pass3<P, 16>(m, j, off, A, a); break;
            default: pass3<P, 32>(m, j, off, A, a); break;
            }
        }
        __syncthreads();
        r0 = r1;
    }
}

constexpr long long kChunkOps = 1LL << 20;                   // ops per launch

bool depth_ok(int d) { return d == 8 || d == 10 || d == 12; }

cudaError_t launch(ItxArgs a, cudaStream_t st)
{
    const long long nops = a.nops;
    const long long per = (nops + 1055) / 1056;             // about 8 CTAs per SM for a frame; 1 op per CTA for a few ops
    a.ops_per_cta = (int)(per < 1 ? 1 : per > kMaxOps ? kMaxOps : per);
    const B200Vp9TxOp *ops = a.ops;
    for (long long b = 0; b < nops; b += kChunkOps) {
        a.ops = ops + b;
        a.nops = nops - b < kChunkOps ? nops - b : kChunkOps;
        const unsigned grid = (unsigned)((a.nops + a.ops_per_cta - 1) / a.ops_per_cta);
        if (a.depth == 8) vp9_itx_kernel<uint8_t><<<grid, kThreads, smem_bytes<uint8_t>(), st>>>(a);
        else vp9_itx_kernel<uint16_t><<<grid, kThreads, smem_bytes<uint16_t>(), st>>>(a);
        B200_LAUNCHED();
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// ---- drop-in members (host pointers): the block's coefficients and the sz x sz block of dst through the device scratch, one op, the
// block back; the coefficients are then left as the reference leaves them (only block[0] cleared on the DC-only path, all else zeroed)
void member_host(int depth, int tx, int type, uint8_t *dst, ptrdiff_t stride, int16_t *block, int eob)
{
    const int N = tx == 4 ? 4 : 4 << tx, bps = depth > 8 ? 2 : 1, cs = depth > 8 ? 4 : 2;
    const size_t cbytes = (size_t)N * N * cs, dpitch = (size_t)N * bps;
    B200HostCall call("vp9 inverse transform", nullptr, 256 + 4096 + 2048);
    uint8_t *scr = call.scratch;
    cudaStream_t st = call.stream;
    uint8_t *dop = scr, *dcoef = scr + 256, *ddst = dcoef + 4096;
    B200Vp9TxOp op;
    memset(&op, 0, sizeof(op));
    op.tx = (uint8_t)tx;
    op.type = (uint8_t)type;
    op.eob = (uint16_t)(eob == 1);   // only eob == 1 means anything to the members; any other int runs the full transform
    call.check(cudaMemcpyAsync(dop, &op, sizeof(op), cudaMemcpyHostToDevice, st), "h2d op");
    call.check(cudaMemcpyAsync(dcoef, block, cbytes, cudaMemcpyHostToDevice, st), "h2d coefficients");
    call.check(b200_h2d_rows(ddst, dpitch, dst, stride, dpitch, (size_t)N, st), "h2d block");
    ItxArgs a = { (const B200Vp9TxOp *)dop, 1, dcoef, ddst, (long long)dpitch, depth, 1 };
    call.check(launch(a, st), "launch");
    call.check(b200_d2h_rows(dst, stride, ddst, dpitch, dpitch, (size_t)N, st), "d2h block");
    call.sync();
    memset(block, 0, dc_only(tx, type, eob) ? (size_t)cs : cbytes);
}

template <int D, int TX, int TYPE>
void m_itxfm(uint8_t *dst, ptrdiff_t stride, int16_t *block, int eob) { member_host(D, TX, TYPE, dst, stride, block, eob); }

// vp9dsp_template.c:1755-1778: four functions per size at 4..16, one for every 32x32 slot, one for every lossless slot
template <int D, int TX>
void fill_size(B200VP9DSPContext *c)
{
    if constexpr (TX < 3) {
        c->itxfm_add[TX][0] = m_itxfm<D, TX, 0>;
        c->itxfm_add[TX][1] = m_itxfm<D, TX, 1>;
        c->itxfm_add[TX][2] = m_itxfm<D, TX, 2>;
        c->itxfm_add[TX][3] = m_itxfm<D, TX, 3>;
    } else {
        c->itxfm_add[TX][0] = c->itxfm_add[TX][1] = c->itxfm_add[TX][2] = c->itxfm_add[TX][3] = m_itxfm<D, TX, 0>;
    }
}
template <int D>
void fill(B200VP9DSPContext *c)
{
    fill_size<D, 0>(c); fill_size<D, 1>(c); fill_size<D, 2>(c); fill_size<D, 3>(c); fill_size<D, 4>(c);
}

} // namespace

B200_API int b200_vp9_dsp_init_itxfm(B200VP9DSPContext *c, int bit_depth)
{
    if (!c) return B200_EINVAL;
    if (!depth_ok(bit_depth)) return B200_ENOSYS;
    if (!b200_default_device()) return B200_ENODEV;
    switch (bit_depth) {
    case 8:  fill<8>(c); break;
    case 10: fill<10>(c); break;
    default: fill<12>(c); break;
    }
    return 0;
}

B200_API int b200_vp9_itxfm_add_batch_device(B200Device *dev, int bit_depth, int64_t nops, const B200Vp9TxOp *ops, const void *coef,
                                             uint8_t *dst, ptrdiff_t dst_stride)
{
    if (nops < 0) { b200_set_error("vp9 itxfm batch: negative nops"); return B200_EINVAL; }
    if (!depth_ok(bit_depth)) { b200_set_error("vp9 itxfm batch: bit depth %d is not 8, 10 or 12", bit_depth); return B200_EINVAL; }
    const int bps = bit_depth > 8 ? 2 : 1;
    if (dst_stride % (4 * bps)) { b200_set_error("vp9 itxfm batch: dst_stride not a multiple of 4 samples"); return B200_EINVAL; }
    if (nops == 0) return 0;
    if (!ops || !coef || !dst || ((uintptr_t)ops & 7) || ((uintptr_t)coef & 15) || ((uintptr_t)dst % (4 * bps))) {
        b200_set_error("vp9 itxfm batch: NULL or misaligned pointer");
        return B200_EINVAL;
    }
    if (int r = b200_use_device(dev)) return r;
    ItxArgs a = { ops, (long long)nops, coef, dst, (long long)dst_stride, bit_depth, 1 };
    B200_CUDA_OK(launch(a, dev->stream));
    return 0;
}
