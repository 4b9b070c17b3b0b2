// tx_double.cu — libavutil/tx in double precision on sm_90a: AV_TX_DOUBLE_FFT and AV_TX_DOUBLE_MDCT, power-of-two lengths (libavutil/tx_double.c
// instantiates tx_template.c with TXSample = double; what the audio filters afir / afftdn / adeclick / dialoguenhance ask for).
//
// Reference semantics reproduced bit for bit (checker: oracle/txd_oracle.c, pinned on the compiled reference), libavutil/tx_template.c:
//   :65-77 cosine tables (double), :540-586 butterflies / transform / split-radix combine, :615-704 recursion and base cases,
//   tx.c:125-154 permutation, :1223-1342 ff_tx_mdct_init / _fwd / _inv, :2107-2134 ff_tx_mdct_gen_exp (scale: const double *).
// Every product and sum is rounded on its own (library built with --fmad=false), in the reference's order.
//
// Plain version: one CTA per transform, the samples in shared memory as double2, the split-radix recursion flattened level by level
// like the compound transforms of tx_pfa.cu (all blocks of one size are independent).  These transforms do
// FP64 arithmetic, which the GPU runs at a fraction of its FP32 rate; the float path carries the tuned kernels.
#include "common.h"
#include "tx_double.h"
#include <cmath>
#include <cstring>
#include <vector>

namespace {

// (tests/test_cuda_emu.py compiles this whole file, host code included, against the stand-in runtime)
struct DblDev {
    const int *map;                            // FFT: gather permutation; inverse MDCT: doubled gather positions; forward MDCT: scatter positions
    const double2 *exp;                        // MDCT twiddles (inverse: pre-shuffled copy first, natural order after it)
    const double *tabs[18];                    // tabs[k]: cosine table of the 2^k-point transform
    int n, logn, len;                          // complex points, their log2, av_tx length
    const int *blk;                            // offsets of the split-radix blocks of an n-point transform, level after level
    int lvl_start[18], lvl_cnt[18];
};

__device__ __forceinline__ int DPAD(int i) { return i + (i >> 4); }

__device__ __forceinline__ void dbutterflies(double2 &a0, double2 &a1, double2 &a2, double2 &a3, double t1, double t2, double t5, double t6)
{
    const double r0 = a0.x, i0 = a0.y, r1 = a1.x, i1 = a1.y;
    const double t3 = t5 - t1; t5 = t5 + t1;
    a2.x = r0 - t5; a0.x = r0 + t5;
    a3.y = i1 - t3; a1.y = i1 + t3;
    const double t4 = t2 - t6; t6 = t2 + t6;
    a3.x = r1 - t4; a1.x = r1 + t4;
    a2.y = i0 - t6; a0.y = i0 + t6;
}

__device__ __forceinline__ void dtransform(double2 &a0, double2 &a1, double2 &a2, double2 &a3, double wre, double wim)
{
    const double t1 = a2.x * wre - a2.y * (-wim);
    const double t2 = a2.x * (-wim) + a2.y * wre;
    const double t5 = a3.x * wre - a3.y * wim;
    const double t6 = a3.x * wim + a3.y * wre;
    dbutterflies(a0, a1, a2, a3, t1, t2, t5, t6);
}

// fft(S) = fft(S/2) | fft(S/4) | fft(S/4) ; combine(S), flattened: the CTA sweeps S = 2, 4, ..., n with one barrier per size.  The hard-coded
// sizes 4, 8, 16 of the reference are instances of the same rule except that their j = 0 butterfly skips the multiplication by (1, 0).
__device__ void dbl_fft(const DblDev &P, double2 *z)
{
    for (int L = 1; L <= P.logn; L++) {
        const int *off = P.blk + P.lvl_start[L];
        const int cnt = P.lvl_cnt[L];
        if (L == 1) {
            for (int it = threadIdx.x; it < cnt; it += blockDim.x) {
                const int o = off[it];
                double2 &a = z[DPAD(o)], &b = z[DPAD(o + 1)];
                const double2 s0 = a, s1 = b;
                a = make_double2(s0.x + s1.x, s0.y + s1.y);
                b = make_double2(s0.x - s1.x, s0.y - s1.y);
            }
        } else {
            const int lq = L - 2, q = 1 << lq, per = cnt << lq;
            const double *tab = P.tabs[L];
            for (int r = threadIdx.x; r < per; r += blockDim.x) {
                const int o = off[r >> lq], jj = r & (q - 1);
                const int i0 = DPAD(o + jj), i1 = DPAD(o + q + jj), i2 = DPAD(o + 2 * q + jj), i3 = DPAD(o + 3 * q + jj);
                double2 a0 = z[i0], a1 = z[i1], a2 = z[i2], a3 = z[i3];
                if (L <= 4 && jj == 0) dbutterflies(a0, a1, a2, a3, a2.x, a2.y, a3.x, a3.y);
                else dtransform(a0, a1, a2, a3, tab[jj], tab[q - jj]);
                z[i0] = a0; z[i1] = a1; z[i2] = a2; z[i3] = a3;
            }
        }
        __syncthreads();
    }
}

constexpr int DBL_THREADS = 128;

// ff_tx_fft (tx_template.c:763-778): dst[i] = src[map[i]], then the in-place transform.  Everything is read before anything is stored.
__global__ void __launch_bounds__(DBL_THREADS)
tx_dbl_fft_kernel(const DblDev P, double2 *out, const double2 *in, long long out_step, long long in_step, long long count)
{
    extern __shared__ double2 dbl_z[];
    for (long long tr = blockIdx.x; tr < count; tr += gridDim.x) {
        const double2 *src = reinterpret_cast<const double2 *>(reinterpret_cast<const char *>(in) + tr * in_step);
        double2 *dst = reinterpret_cast<double2 *>(reinterpret_cast<char *>(out) + tr * out_step);
        for (int i = threadIdx.x; i < P.n; i += blockDim.x) dbl_z[DPAD(i)] = src[P.map[i]];
        __syncthreads();
        dbl_fft(P, dbl_z);
        for (int i = threadIdx.x; i < P.n; i += blockDim.x) dst[i] = dbl_z[DPAD(i)];
        __syncthreads();
    }
}

// ff_tx_mdct_inv (tx_template.c:1299-1342): len doubles with a stride (in doubles) in, len doubles (len / 2 complex) out
__global__ void __launch_bounds__(DBL_THREADS)
tx_dbl_mdct_inv_kernel(const DblDev P, double *out, const double *in, long long stride, long long out_step, long long in_step, long long count)
{
    extern __shared__ double2 dbl_z[];
    const int len2 = P.len >> 1, len4 = P.len >> 2;
    for (long long tr = blockIdx.x; tr < count; tr += gridDim.x) {
        const double *src = reinterpret_cast<const double *>(reinterpret_cast<const char *>(in) + tr * in_step);
        double2 *z = reinterpret_cast<double2 *>(reinterpret_cast<char *>(out) + tr * out_step);
        const double *in1 = src, *in2 = src + (len2 * 2 - 1) * stride;
        for (int i = threadIdx.x; i < len2; i += blockDim.x) {
            const int k = P.map[i];
            const double are = in2[-k * stride], aim = in1[k * stride];
            const double2 e = P.exp[i];
            dbl_z[DPAD(i)] = make_double2(are * e.x - aim * e.y, are * e.y + aim * e.x);
        }
        __syncthreads();
        dbl_fft(P, dbl_z);
        const double2 *e = P.exp + len2;
        for (int i = threadIdx.x; i < len4; i += blockDim.x) {
            const int i0 = len4 + i, i1 = len4 - i - 1;
            const double2 t1 = dbl_z[DPAD(i1)], t0 = dbl_z[DPAD(i0)];
            const double2 s1 = make_double2(t1.y, t1.x), s0 = make_double2(t0.y, t0.x);
            double2 o1, o0;
            o1.x = s1.x * e[i1].y - s1.y * e[i1].x;
            o0.y = s1.x * e[i1].x + s1.y * e[i1].y;
            o0.x = s0.x * e[i0].y - s0.y * e[i0].x;
            o1.y = s0.x * e[i0].x + s0.y * e[i0].y;
            z[i1] = o1; z[i0] = o0;
        }
        __syncthreads();
    }
}

// ff_tx_mdct_fwd (tx_template.c:1254-1297): 2 * len doubles in, len doubles with a stride (in doubles) out
__global__ void __launch_bounds__(DBL_THREADS)
tx_dbl_mdct_fwd_kernel(const DblDev P, double *out, const double *in, long long stride, long long out_step, long long in_step, long long count)
{
    extern __shared__ double2 dbl_z[];
    const int len2 = P.len >> 1, len4 = P.len >> 2, len3 = len2 * 3;
    for (long long tr = blockIdx.x; tr < count; tr += gridDim.x) {
        const double *src = reinterpret_cast<const double *>(reinterpret_cast<const char *>(in) + tr * in_step);
        double *dst = reinterpret_cast<double *>(reinterpret_cast<char *>(out) + tr * out_step);
        for (int i = threadIdx.x; i < len2; i += blockDim.x) {
            const int k = 2 * i, idx = P.map[i];
            double re, im;
            if (k < len2) { re = -src[len2 + k] + src[1 * len2 - 1 - k]; im = -src[len3 + k] + -src[1 * len3 - 1 - k]; }
            else          { re = -src[len2 + k] + -src[5 * len2 - 1 - k]; im = src[-len2 + k] + -src[1 * len3 - 1 - k]; }
            const double2 e = P.exp[i];
            dbl_z[DPAD(idx)] = make_double2(re * e.y + im * e.x, re * e.x - im * e.y);
        }
        __syncthreads();
        dbl_fft(P, dbl_z);
        const double2 *e = P.exp;
        for (int i = threadIdx.x; i < len4; i += blockDim.x) {
            const int i0 = len4 + i, i1 = len4 - i - 1;
            const double2 s1 = dbl_z[DPAD(i1)], s0 = dbl_z[DPAD(i0)];
            dst[(2 * i1 + 1) * stride] = s0.x * e[i0].y - s0.y * e[i0].x;
            dst[2 * i0 * stride]       = s0.x * e[i0].x + s0.y * e[i0].y;
            dst[(2 * i0 + 1) * stride] = s1.x * e[i1].y - s1.y * e[i1].x;
            dst[2 * i1 * stride]       = s1.x * e[i1].x + s1.y * e[i1].y;
        }
        __syncthreads();
    }
}


int dsr_perm(int i, int len, int inv)                              // split_radix_permutation, libavutil/tx.c:125-134
{
    len >>= 1;
    if (len <= 1) return i & 1;
    if (!(i & len)) return dsr_perm(i, len, inv) * 2;
    len >>= 1;
    return dsr_perm(i, len, inv) * 4 + 1 - 2 * (!(i & len) ^ inv);
}

void collect_blocks(std::vector<std::vector<int>> &lv, int L, int off)   // block of size 2^L at `off` and everything below it
{
    if (L < 1) return;
    lv[L].push_back(off);
    const int S = 1 << L;
    collect_blocks(lv, L - 1, off);
    if (L >= 2) {
        collect_blocks(lv, L - 2, off + S / 2);
        collect_blocks(lv, L - 2, off + 3 * S / 4);
    }
}

} // namespace

struct TxDbl {
    B200Device *dev = nullptr;
    int type = 0, inv = 0, len = 0;
    DblDev d{};
    void *blob = nullptr;
    size_t smem = 0;
    int grid_cap = 0;
};

bool tx_dbl_length_ok(int type, int len)
{
    if (len < 2 || (len & (len - 1))) return false;
    const int n = type == B200_TX_DOUBLE_FFT ? len : len >> 1;
    if (type == B200_TX_DOUBLE_MDCT && len < 4) return false;      // len 2: the reference falls back to its naive MDCT
    return n >= 1 && n <= 8192;                                    // one transform must fit a CTA's shared memory (16 bytes per point)
}

TxDbl *tx_dbl_create(B200Device *dev, int type, int inv, int len, double scale)
{
    if (!tx_dbl_length_ok(type, len)) return nullptr;
    const bool mdct = type == B200_TX_DOUBLE_MDCT;
    const int n = mdct ? len >> 1 : len;
    int logn = 0;
    while ((1 << logn) < n) logn++;
    std::vector<int> perm(n), map(n);
    const bool scatter = mdct && !inv;                             // ff_tx_mdct_init: map_dir = !inv ? SCATTER : GATHER
    for (int i = 0; i < n; i++) {
        const int p = n == 1 ? 0 : (-dsr_perm(i, n, inv)) & (n - 1);
        if (scatter) perm[p] = i; else perm[i] = p;
    }
    std::vector<double> exp;
    if (mdct) {                                                    // ff_tx_mdct_gen_exp, tx_template.c:2107-2134
        const double theta = (scale < 0 ? n : 0) + 1.0 / 8.0, sc = sqrt(fabs(scale));
        std::vector<double> full(2 * (size_t)n);
        for (int i = 0; i < n; i++) {
            const double alpha = M_PI_2 * (i + theta) / n;
            full[2 * i] = cos(alpha) * sc; full[2 * i + 1] = sin(alpha) * sc;
        }
        if (inv) {
            exp.assign(4 * (size_t)n, 0.0);
            memcpy(&exp[2 * (size_t)n], full.data(), sizeof(double) * 2 * n);
            for (int i = 0; i < n; i++) { exp[2 * i] = full[2 * perm[i]]; exp[2 * i + 1] = full[2 * perm[i] + 1]; }
        } else
            exp = full;
    }
    for (int i = 0; i < n; i++) map[i] = mdct && inv ? perm[i] << 1 : perm[i];
    std::vector<std::vector<int>> lv(18);
    collect_blocks(lv, logn, 0);
    std::vector<int> blk;
    int lvl_start[18] = { 0 }, lvl_cnt[18] = { 0 };
    for (int L = 0; L < 18; L++) { lvl_start[L] = (int)blk.size(); lvl_cnt[L] = (int)lv[L].size(); blk.insert(blk.end(), lv[L].begin(), lv[L].end()); }
    std::vector<std::vector<double>> cosk(18);
    for (int k = 3; k <= logn; k++) {                              // ff_tx_init_tab_N, tx_template.c:65-77
        const int nn = 1 << k;
        cosk[k].assign(nn / 4 + 1, 0.0);
        const double freq = 2 * M_PI / nn;
        for (int i = 0; i < nn / 4; i++) cosk[k][i] = cos(i * freq);
    }
    auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
    size_t off = 0;
    const size_t o_map = off; off += al(sizeof(int) * n);
    const size_t o_exp = off; off += al(sizeof(double) * exp.size() + 16);
    const size_t o_blk = off; off += al(sizeof(int) * blk.size() + 4);
    size_t o_cos[18] = { 0 };
    for (int k = 3; k <= logn; k++) { o_cos[k] = off; off += al(sizeof(double) * cosk[k].size()); }
    std::vector<uint8_t> host(off + 256, 0);
    memcpy(&host[o_map], map.data(), sizeof(int) * n);
    if (!exp.empty()) memcpy(&host[o_exp], exp.data(), sizeof(double) * exp.size());
    if (!blk.empty()) memcpy(&host[o_blk], blk.data(), sizeof(int) * blk.size());
    for (int k = 3; k <= logn; k++) memcpy(&host[o_cos[k]], cosk[k].data(), sizeof(double) * cosk[k].size());
    TxDbl *p = new (std::nothrow) TxDbl();
    if (!p) return nullptr;
    p->dev = dev; p->type = type; p->inv = inv; p->len = len;
    if (cudaMalloc(&p->blob, host.size()) != cudaSuccess || cudaMemcpy(p->blob, host.data(), host.size(), cudaMemcpyHostToDevice) != cudaSuccess) {
        b200_set_error("tx_dbl_create: device tables");
        if (p->blob) cudaFree(p->blob);
        delete p;
        return nullptr;
    }
    uint8_t *b = (uint8_t *)p->blob;
    DblDev &d = p->d;
    d.map = (const int *)(b + o_map); d.exp = (const double2 *)(b + o_exp); d.blk = (const int *)(b + o_blk);
    for (int k = 0; k < 18; k++) d.tabs[k] = k >= 3 && k <= logn ? (const double *)(b + o_cos[k]) : nullptr;
    d.n = n; d.logn = logn; d.len = len;
    for (int L = 0; L < 18; L++) { d.lvl_start[L] = lvl_start[L]; d.lvl_cnt[L] = lvl_cnt[L]; }
    p->smem = (size_t)(n + (n >> 4) + 1) * sizeof(double2);
    if (p->smem > 48 * 1024 &&
        (cudaFuncSetAttribute(tx_dbl_fft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->smem) != cudaSuccess ||
         cudaFuncSetAttribute(tx_dbl_mdct_inv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->smem) != cudaSuccess ||
         cudaFuncSetAttribute(tx_dbl_mdct_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->smem) != cudaSuccess)) {
        b200_set_error("tx_dbl_create: %zu bytes of shared memory per transform", p->smem);
        cudaFree(p->blob);
        delete p;
        return nullptr;
    }
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev->ordinal);
    p->grid_cap = (sms > 0 ? sms : 132) * 8;
    return p;
}

void tx_dbl_free(TxDbl *p)
{
    if (!p) return;
    if (p->blob) cudaFree(p->blob);
    delete p;
}

int tx_dbl_launch(TxDbl *p, cudaStream_t st, void *out, const void *in, ptrdiff_t stride, int64_t count, ptrdiff_t out_step, ptrdiff_t in_step)
{
    if (count <= 0) return 0;
    const bool mdct = p->type == B200_TX_DOUBLE_MDCT;
    const int oa = (!mdct || p->inv) ? 15 : 7;                     // complex stores (16 bytes) except for the forward MDCT
    const int ia = mdct ? 7 : 15;
    if (((reinterpret_cast<uintptr_t>(out) | (uintptr_t)out_step) & oa) || ((reinterpret_cast<uintptr_t>(in) | (uintptr_t)in_step) & ia)) {
        b200_set_error("b200_tx_batch_device: double transform pointers and steps must be multiples of 16 bytes on the complex side, 8 on the real side");
        return B200_EINVAL;
    }
    if (mdct && ((stride & 7) || stride <= 0)) return B200_EINVAL;
    const unsigned nb = (unsigned)(count < p->grid_cap ? count : p->grid_cap);
    if (!mdct)       tx_dbl_fft_kernel<<<nb, DBL_THREADS, p->smem, st>>>(p->d, (double2 *)out, (const double2 *)in, out_step, in_step, count);
    else if (p->inv) tx_dbl_mdct_inv_kernel<<<nb, DBL_THREADS, p->smem, st>>>(p->d, (double *)out, (const double *)in, (long long)(stride / 8), out_step, in_step, count);
    else             tx_dbl_mdct_fwd_kernel<<<nb, DBL_THREADS, p->smem, st>>>(p->d, (double *)out, (const double *)in, (long long)(stride / 8), out_step, in_step, count);
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

// av_tx_fn shaped entry: HOST pointers, one transform
void tx_dbl_host_fn(TxDbl *p, void *out, void *in, ptrdiff_t stride)
{
    const size_t len = p->len;
    const bool mdct = p->type == B200_TX_DOUBLE_MDCT;
    const size_t in_elems = !mdct ? 2 * len : p->inv ? len : 2 * len, out_elems = !mdct ? 2 * len : len;        // doubles
    B200HostCall call("av_tx_fn (double)", p->dev, (in_elems + out_elems) * 8 + 1024);
    double *din = (double *)call.scratch, *dout = din + ((in_elems + 63) & ~(size_t)63);
    cudaStream_t st = call.stream;
    cudaError_t e;
    const bool strided_in = mdct && p->inv && stride != 8, strided_out = mdct && !p->inv && stride != 8;
    if (strided_in) e = cudaMemcpy2DAsync(din, 8, in, (size_t)stride, 8, in_elems, cudaMemcpyHostToDevice, st);
    else e = cudaMemcpyAsync(din, in, in_elems * 8, cudaMemcpyHostToDevice, st);
    call.check(e, "h2d");
    call.launched(tx_dbl_launch(p, st, dout, din, 8, 1, 0, 0));
    if (strided_out) e = cudaMemcpy2DAsync(out, (size_t)stride, dout, 8, 8, out_elems, cudaMemcpyDeviceToHost, st);
    else e = cudaMemcpyAsync(out, dout, out_elems * 8, cudaMemcpyDeviceToHost, st);
    call.check(e, "d2h");
    call.sync();
}
