// tx_int32.cu — libavutil/tx 32-bit fixed-point transforms on sm_90a: AV_TX_INT32_FFT and AV_TX_INT32_MDCT, power-of-two lengths
// (the fixed-point AAC / AC-3 decoders' transforms).
//
// Reference semantics reproduced bit for bit (checker: oracle/txi_oracle.c): the TX_INT32 instantiation of libavutil/tx_template.c
// (libavutil/tx_int32.c) with the macros of libavutil/tx_priv.h:113-155 — sums wrap modulo 2^32, products are 64-bit and rounded
// ((a*b - c*d + 2^30) >> 31), tables are clip(llrintf((float)(x * 2^31))), the forward MDCT folds its input with (a + b + 32) >> 6.
//   tables tx_template.c:65-77; butterflies / transform / combine :540-586; base cases :631-704; recursion :615-629; FFT wrapper :763-778;
//   MDCT :1223-1342; twiddles :2107-2134; permutation libavutil/tx.c:125-154.
//
// One CTA per transform, the transform in shared memory (as tx.cu's float kernels): the reference's recursion
// fft(S) = fft(S/2) | fft(S/4) | fft(S/4) ; combine(S) is flattened into levels — all blocks of one size are independent — and the
// CTA sweeps S = 2, 4, ..., n with one barrier per size; the hard-coded sizes 4, 8, 16 follow the same rule except that their j = 0
// butterfly skips the multiplication by (1, 0).  Every sum wraps modulo 2^32 and every product is rounded exactly as the reference
// does it, so the schedule does not matter for the bits.  IMAD.WIDE carries the 64-bit products.
#include "tx_int32.h"
#include <vector>
#include <cmath>
#include <cstring>

namespace {

// [device-code tx_int32] (tests/cuda_emu runs this block on the CPU against the checker; comment markers only)
struct TxiDev {
    const int *map;                 // FFT: gather permutation; MDCT: the same, doubled for the inverse (positions in floats)
    const int2 *exp;                // MDCT twiddles (inverse: pre-shuffled copy first, natural order after it)
    const int *tabs[18];            // tabs[k]: cosine table of the 2^k-point transform
    int n, log2n, len;              // n: complex points of the FFT that runs
    const int *blk;                 // offsets of the split-radix blocks, level after level
    int lvl_start[18], lvl_cnt[18]; // level L (block size 2^L): blk[lvl_start[L] .. + lvl_cnt[L])
};

__device__ __forceinline__ int mulr(long long accu) { return (int)((accu + 0x40000000LL) >> 31); }
// CMUL(dre, dim, are, aim, bre, bim)
__device__ __forceinline__ void cmul(unsigned &dre, unsigned &dim, int are, int aim, int bre, int bim)
{
    dre = (unsigned)mulr((long long)bre * are - (long long)bim * aim);
    dim = (unsigned)mulr((long long)bim * are + (long long)bre * aim);
}
__device__ __forceinline__ void butterflies(int2 &a0, int2 &a1, int2 &a2, int2 &a3, unsigned t1, unsigned t2, unsigned t5, unsigned t6)
{
    const unsigned r0 = a0.x, i0 = a0.y, r1 = a1.x, i1 = a1.y;
    const unsigned t3 = t5 - t1; t5 = t5 + t1;
    a2.x = (int)(r0 - t5); a0.x = (int)(r0 + t5);
    a3.y = (int)(i1 - t3); a1.y = (int)(i1 + t3);
    const unsigned t4 = t2 - t6; t6 = t2 + t6;
    a3.x = (int)(r1 - t4); a1.x = (int)(r1 + t4);
    a2.y = (int)(i0 - t6); a0.y = (int)(i0 + t6);
}
__device__ __forceinline__ void transform(int2 &a0, int2 &a1, int2 &a2, int2 &a3, int wre, int wim)
{
    unsigned t1, t2, t5, t6;
    cmul(t1, t2, a2.x, a2.y, wre, -wim);
    cmul(t5, t6, a3.x, a3.y, wre, wim);
    butterflies(a0, a1, a2, a3, t1, t2, t5, t6);
}
__device__ __forceinline__ int PADI(int i) { return i + (i >> 4); }
// all levels of one transform held in z[PADI(0 .. n)) (shared memory)
__device__ void i32_levels(const TxiDev &P, int2 *z)
{
    for (int L = 1; L <= P.log2n; L++) {
        const int *off = P.blk + P.lvl_start[L];
        const int cnt = P.lvl_cnt[L];
        if (L == 1) {
            for (int b = threadIdx.x; b < cnt; b += blockDim.x) {
                const int o = off[b];
                const int2 s0 = z[PADI(o)], s1 = z[PADI(o + 1)];
                z[PADI(o)] = make_int2((int)((unsigned)s0.x + (unsigned)s1.x), (int)((unsigned)s0.y + (unsigned)s1.y));
                z[PADI(o + 1)] = make_int2((int)((unsigned)s0.x - (unsigned)s1.x), (int)((unsigned)s0.y - (unsigned)s1.y));
            }
        } else {
            const int lq = L - 2, q = 1 << lq, total = cnt << lq;
            const int *tab = P.tabs[L];
            for (int r = threadIdx.x; r < total; r += blockDim.x) {
                const int o = off[r >> lq], j = r & (q - 1);
                const int i0 = PADI(o + j), i1 = PADI(o + q + j), i2 = PADI(o + 2 * q + j), i3 = PADI(o + 3 * q + j);
                int2 a0 = z[i0], a1 = z[i1], a2 = z[i2], a3 = z[i3];
                if (L <= 4 && j == 0) butterflies(a0, a1, a2, a3, (unsigned)a2.x, (unsigned)a2.y, (unsigned)a3.x, (unsigned)a3.y);
                else transform(a0, a1, a2, a3, tab[j], tab[q - j]);
                z[i0] = a0; z[i1] = a1; z[i2] = a2; z[i3] = a3;
            }
        }
        __syncthreads();
    }
}

__device__ __forceinline__ int fold(int x, int y) { return (int)((unsigned)x + (unsigned)y + 32u) >> 6; }

// kind 0: FFT, 1: inverse MDCT, 2: forward MDCT.  One CTA per transform (CTAs stride over the batch).
constexpr int I32_THREADS = 128;
template <int KIND>
__global__ void __launch_bounds__(I32_THREADS)
tx_i32_kernel(const TxiDev P, int *out, const int *in, long long stride, long long out_step, long long in_step, long long count)
{
    extern __shared__ int2 i32_z[];
    int2 *z = i32_z;
    const int len2 = P.len >> 1, len4 = P.len >> 2;
    for (long long tr = blockIdx.x; tr < count; tr += gridDim.x) {
        int *dst = reinterpret_cast<int *>(reinterpret_cast<char *>(out) + tr * out_step);
        const int *src = reinterpret_cast<const int *>(reinterpret_cast<const char *>(in) + tr * in_step);
        const int2 *e = P.exp;
        if (KIND == 0) {
            const int2 *s = reinterpret_cast<const int2 *>(src);
            for (int j = threadIdx.x; j < P.n; j += blockDim.x) z[PADI(j)] = s[P.map[j]];
        } else if (KIND == 1) {
            const int *in1 = src, *in2 = src + (len2 * 2 - 1) * stride;
            for (int i = threadIdx.x; i < len2; i += blockDim.x) {
                const int k = P.map[i];
                unsigned re, im;
                cmul(re, im, in2[-k * stride], in1[k * stride], e[i].x, e[i].y);
                z[PADI(i)] = make_int2((int)re, (int)im);
            }
        } else {
            const int len3 = len2 * 3;
            for (int i = threadIdx.x; i < len2; i += blockDim.x) {
                const int k = 2 * i, idx = P.map[i];
                int re, im;
                if (k < len2) { re = fold(-src[len2 + k], src[1 * len2 - 1 - k]); im = fold(-src[len3 + k], -src[1 * len3 - 1 - k]); }
                else          { re = fold(-src[len2 + k], -src[5 * len2 - 1 - k]); im = fold(src[-len2 + k], -src[1 * len3 - 1 - k]); }
                unsigned a, b;
                cmul(a, b, re, im, e[i].x, e[i].y);
                z[PADI(idx)] = make_int2((int)b, (int)a);
            }
        }
        __syncthreads();
        i32_levels(P, z);
        if (KIND == 0) {
            int2 *d = reinterpret_cast<int2 *>(dst);
            for (int j = threadIdx.x; j < P.n; j += blockDim.x) d[j] = z[PADI(j)];
        } else if (KIND == 1) {
            int2 *d = reinterpret_cast<int2 *>(dst);
            e += len2;
            for (int i = threadIdx.x; i < len4; i += blockDim.x) {
                const int i0 = len4 + i, i1 = len4 - i - 1;
                const int2 z1 = z[PADI(i1)], z0 = z[PADI(i0)];
                const int2 s1 = make_int2(z1.y, z1.x), s0 = make_int2(z0.y, z0.x);
                unsigned a, b, c2, d2;
                cmul(a, b, s1.x, s1.y, e[i1].y, e[i1].x);            // z[i1].re, z[i0].im
                cmul(c2, d2, s0.x, s0.y, e[i0].y, e[i0].x);          // z[i0].re, z[i1].im
                d[i1] = make_int2((int)a, (int)d2);
                d[i0] = make_int2((int)c2, (int)b);
            }
        } else {
            for (int i = threadIdx.x; i < len4; i += blockDim.x) {
                const int i0 = len4 + i, i1 = len4 - i - 1;
                const int2 s1 = z[PADI(i1)], s0 = z[PADI(i0)];
                unsigned a, b;
                cmul(a, b, s0.x, s0.y, e[i0].y, e[i0].x); dst[(2 * i1 + 1) * stride] = (int)a; dst[2 * i0 * stride] = (int)b;
                cmul(a, b, s1.x, s1.y, e[i1].y, e[i1].x); dst[(2 * i0 + 1) * stride] = (int)a; dst[2 * i1 * stride] = (int)b;
            }
        }
        __syncthreads();                                   // the buffer is reused by the next transform of this CTA
    }
}
// [/device-code tx_int32]

int sr_perm(int i, int len, int inv)
{
    len >>= 1;
    if (len <= 1) return i & 1;
    if (!(i & len)) return sr_perm(i, len, inv) * 2;
    len >>= 1;
    return sr_perm(i, len, inv) * 4 + 1 - 2 * (!(i & len) ^ inv);
}
int32_t rescale(double x)                                           // RESCALE of tx_priv.h:140 for TX_INT32
{
    const float f = (float)(x * 2147483648.0);
    long long v = llrintf(f);
    if (v < INT32_MIN) v = INT32_MIN;
    if (v > INT32_MAX) v = INT32_MAX;
    return (int32_t)v;
}

} // namespace

struct TxI32 {
    B200Device *dev = nullptr;
    int type = 0, inv = 0, len = 0;
    TxiDev d{};
    void *blob = nullptr;
    size_t smem = 0;
    int grid_cap = 0;
};

bool tx_i32_length_ok(int type, int len)
{
    if (len < 2 || (len & (len - 1))) return false;
    const int n = type == B200_TX_INT32_FFT ? len : len >> 1;
    return n >= 1 && n <= 4096 && (type == B200_TX_INT32_FFT || len >= 4);
}

// host tables, flattened: [map n][exp 2 * (inv ? 2n : n) (MDCT only)][cos tables k = 3 .. log2 n]; layout4 = word offsets + log2 n
static int i32_host_tables(std::vector<int32_t> &w, int32_t lay[4], int type, int inv, int len, float scale)
{
    const int n = type == B200_TX_INT32_FFT ? len : len >> 1;
    int k = 0;
    while ((1 << k) < n) k++;
    std::vector<int> map(n);
    const bool scatter = type == B200_TX_INT32_MDCT && !inv;
    for (int i = 0; i < n; i++) {
        const int p = n == 1 ? 0 : (-sr_perm(i, n, inv)) & (n - 1);
        if (scatter) map[p] = i; else map[i] = p;
    }
    w.clear();
    lay[0] = 0;
    lay[1] = n;
    std::vector<int32_t> exp;
    if (type == B200_TX_INT32_MDCT) {
        const int len4 = len >> 1;
        const double theta = (scale < 0 ? len4 : 0) + 1.0 / 8.0, sc = sqrt(fabs((double)scale));
        std::vector<int32_t> full(2 * (size_t)len4);
        for (int i = 0; i < len4; i++) {
            const double alpha = M_PI_2 * (i + theta) / len4;
            full[2 * i] = rescale(cos(alpha) * sc);
            full[2 * i + 1] = rescale(sin(alpha) * sc);
        }
        if (inv) {
            exp.assign(4 * (size_t)len4, 0);
            memcpy(&exp[2 * (size_t)len4], full.data(), sizeof(int32_t) * 2 * len4);
            for (int i = 0; i < len4; i++) { exp[2 * i] = full[2 * map[i]]; exp[2 * i + 1] = full[2 * map[i] + 1]; }
            for (int i = 0; i < len4; i++) map[i] <<= 1;            // "saves multiplies in loops", tx_template.c:1266-1268
        } else
            exp = full;
    }
    for (int x : map) w.push_back(x);
    for (int32_t x : exp) w.push_back(x);
    lay[2] = (int32_t)w.size();
    for (int kk = 3; kk <= k; kk++) {
        const int nn = 1 << kk;
        const double freq = 2 * M_PI / nn;
        for (int i = 0; i < nn / 4; i++) w.push_back(rescale(cos(i * freq)));
        w.push_back(0);
    }
    lay[3] = k;
    {   // after the cosine tables: 18 level starts, 18 level counts, then the block offsets of every level
        std::vector<std::vector<int>> lv(18);
        struct R { static void go(std::vector<std::vector<int>> &lv, int L, int off) {
            if (L < 1) return;
            lv[L].push_back(off);
            const int S = 1 << L;
            go(lv, L - 1, off);
            if (L >= 2) { go(lv, L - 2, off + S / 2); go(lv, L - 2, off + 3 * S / 4); }
        } };
        R::go(lv, k, 0);
        int start = 0;
        for (int L = 0; L < 18; L++) { w.push_back(start); start += (int)lv[L].size(); }
        for (int L = 0; L < 18; L++) w.push_back((int)lv[L].size());
        for (int L = 0; L < 18; L++) for (int o : lv[L]) w.push_back(o);
    }
    return (int)w.size();
}

B200_API int b200_tx_i32_tables(int type, int inv, int len, float scale, int32_t *words, int cap, int32_t *layout4)
{
    if ((type != B200_TX_INT32_FFT && type != B200_TX_INT32_MDCT) || !tx_i32_length_ok(type, len)) return B200_ENOSYS;
    std::vector<int32_t> w;
    int32_t lay[4];
    const int nw = i32_host_tables(w, lay, type, !!inv, len, scale);
    if (layout4) memcpy(layout4, lay, sizeof(lay));
    if (words && cap >= nw) memcpy(words, w.data(), (size_t)nw * 4);
    return nw;
}

TxI32 *tx_i32_create(B200Device *dev, int type, int inv, int len, float scale)
{
    if (!tx_i32_length_ok(type, len)) return nullptr;
    std::vector<int32_t> w;
    int32_t lay[4];
    const int nw = i32_host_tables(w, lay, type, inv, len, scale);
    TxI32 *p = new (std::nothrow) TxI32();
    if (!p) return nullptr;
    p->dev = dev; p->type = type; p->inv = inv; p->len = len;
    if (cudaMalloc(&p->blob, (size_t)nw * 4 + 16) != cudaSuccess || cudaMemcpy(p->blob, w.data(), (size_t)nw * 4, cudaMemcpyHostToDevice) != cudaSuccess) {
        b200_set_error("tx_i32_create: device tables");
        if (p->blob) cudaFree(p->blob);
        delete p;
        return nullptr;
    }
    const int32_t *b = (const int32_t *)p->blob;
    TxiDev &d = p->d;
    d.n = type == B200_TX_INT32_FFT ? len : len >> 1; d.log2n = lay[3]; d.len = len;
    d.map = b + lay[0];
    d.exp = (const int2 *)(b + lay[1]);
    const int32_t *c = b + lay[2];
    for (int k = 0; k < 18; k++) d.tabs[k] = nullptr;
    for (int k = 3; k <= d.log2n; k++) { d.tabs[k] = c; c += (1 << k) / 4 + 1; }
    d.blk = c + 36;
    for (int L = 0; L < 18; L++) { d.lvl_start[L] = w[(size_t)(c - b) + L]; d.lvl_cnt[L] = w[(size_t)(c - b) + 18 + L]; }
    p->smem = (size_t)(d.n + (d.n >> 4) + 1) * sizeof(int2);
    if (p->smem > 48 * 1024 &&
        (cudaFuncSetAttribute(tx_i32_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->smem) != cudaSuccess ||
         cudaFuncSetAttribute(tx_i32_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->smem) != cudaSuccess ||
         cudaFuncSetAttribute(tx_i32_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->smem) != cudaSuccess)) {
        cudaFree(p->blob);
        delete p;
        return nullptr;
    }
    p->grid_cap = (dev && dev->sm_count > 0 ? dev->sm_count : 132) * 8;
    return p;
}

void tx_i32_free(TxI32 *p)
{
    if (!p) return;
    if (p->blob) cudaFree(p->blob);
    delete p;
}

int tx_i32_launch(TxI32 *p, cudaStream_t st, void *out, const void *in, ptrdiff_t stride, int64_t count, ptrdiff_t out_step, ptrdiff_t in_step)
{
    if (count <= 0) return 0;
    // the kernels move complex values as 8-byte words: the complex side(s) of a transform must be 8-byte aligned (the reference
    // asks for 32 unless AV_TX_UNALIGNED), the real side 4
    const uintptr_t oa = reinterpret_cast<uintptr_t>(out) | (uintptr_t)out_step, ia = reinterpret_cast<uintptr_t>(in) | (uintptr_t)in_step;
    const bool cplx_out = p->type == B200_TX_INT32_FFT || p->inv, cplx_in = p->type == B200_TX_INT32_FFT;
    if ((oa & (cplx_out ? 7 : 3)) || (ia & (cplx_in ? 7 : 3))) {
        b200_set_error("b200_tx_batch_device: int32 transform pointers and steps must be multiples of 8 bytes on the complex side, 4 on the real side");
        return B200_EINVAL;
    }
    const unsigned nb = (unsigned)(count < p->grid_cap ? count : p->grid_cap);
    const long long sf = (long long)(stride / 4);
    if (p->type == B200_TX_INT32_FFT) tx_i32_kernel<0><<<nb, I32_THREADS, p->smem, st>>>(p->d, (int *)out, (const int *)in, sf, out_step, in_step, count);
    else if (p->inv)                  tx_i32_kernel<1><<<nb, I32_THREADS, p->smem, st>>>(p->d, (int *)out, (const int *)in, sf, out_step, in_step, count);
    else                              tx_i32_kernel<2><<<nb, I32_THREADS, p->smem, st>>>(p->d, (int *)out, (const int *)in, sf, out_step, in_step, count);
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

void tx_i32_host_fn(TxI32 *p, void *out, void *in, ptrdiff_t stride)
{
    const size_t len = p->len;
    const bool mdct = p->type == B200_TX_INT32_MDCT;
    const size_t in_elems = !mdct ? 2 * len : p->inv ? len : 2 * len, out_elems = !mdct ? 2 * len : len;        // 32-bit words
    B200HostCall call("av_tx_fn (int32)", p->dev, (in_elems + out_elems) * 4 + 512);
    int32_t *din = (int32_t *)call.scratch, *dout = din + ((in_elems + 63) & ~(size_t)63);
    cudaStream_t st = call.stream;
    cudaError_t e;
    const bool strided_in = mdct && p->inv && stride != 4, strided_out = mdct && !p->inv && stride != 4;
    if (strided_in) e = cudaMemcpy2DAsync(din, 4, in, (size_t)stride, 4, in_elems, cudaMemcpyHostToDevice, st);
    else e = cudaMemcpyAsync(din, in, in_elems * 4, cudaMemcpyHostToDevice, st);
    call.check(e, "h2d");
    call.launched(tx_i32_launch(p, st, dout, din, 4, 1, 0, 0));
    if (strided_out) e = cudaMemcpy2DAsync(out, (size_t)stride, dout, 4, 4, out_elems, cudaMemcpyDeviceToHost, st);
    else e = cudaMemcpyAsync(out, dout, out_elems * 4, cudaMemcpyDeviceToHost, st);
    call.check(e, "d2h");
    call.sync();
}
