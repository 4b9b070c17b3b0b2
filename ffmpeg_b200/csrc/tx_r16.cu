// tx_r16.cu — power-of-two float FFT / inverse MDCT with register-resident split-radix passes (sm_90a).
//
// Same arithmetic, in the same order per output, as the reference's *_float_c codelets (libavutil/tx_template.c:540-722 split-radix
// codelets and ff_tx_fft_sr_combine, :1312-1342 ff_tx_mdct_inv; checker: oracle/tx_oracle.c), so results stay bit-identical; only
// the schedule is different from tx.cu's level-by-level kernels:
//
//  * The reference's recursion  fft(S) = fft(S/2) | fft(S/4) | fft(S/4) ; combine(S)  only ever connects elements whose indices
//    differ by multiples of S/4.  All combines of the levels (a, a+3] therefore close over the 16 elements  m*C + j + t*q
//    (C = 2^(a+3), q = 2^(a-1), t < 16): one thread holds them in registers and does up to nine butterflies before anything goes
//    back to shared memory.  An aligned chunk of C elements is either one block of level a+3 or two blocks of level a+2 (the two
//    quarter blocks of a level-a+4 block are adjacent), so every thread always owns 16 elements: n/16 threads per transform,
//    3 exchanges through shared memory for 1024 points (levels 1-4 | 5-7 | 8-10) instead of 7.
//  * The work of a thread is the same for every transform (persistent CTAs): its butterfly factors and shared-memory offsets are
//    loaded once into registers; nothing but samples moves inside the loop.
//  * Input: one cp.async.bulk (1-D TMA, UBLKCP in SASS) per transform into a two-deep ring per thread group, completion on an
//    mbarrier; the split-radix permutation (and the MDCT pre-rotation) is applied on the shared-memory -> register read.  Output:
//    the last pass stores straight from registers (256 contiguous bytes per warp instruction); the MDCT post-rotation swaps its
//    mirrored partner values inside the warp with one shuffle per sample (thread -> column mapping chosen for that).
//
// Algorithmic HBM bytes: 8n in + 8n out per complex FFT, 4*len + 4*len per inverse MDCT (n = len/2).
#include "common.h"
#include "tx_r16.h"
#include <vector>
#include <cmath>
#include <cstring>

namespace {

// ------------------------------------------------------------------------------------------------ arithmetic (as tx.cu)
__device__ __forceinline__ void butterflies(float2 &a0, float2 &a1, float2 &a2, float2 &a3, float t1, float t2, float t5, float t6)
{
    const float r0 = a0.x, i0 = a0.y, r1 = a1.x, i1 = a1.y;
    const float t3 = t5 - t1; t5 = t5 + t1;
    a2.x = r0 - t5; a0.x = r0 + t5;
    a3.y = i1 - t3; a1.y = i1 + t3;
    const float t4 = t2 - t6; t6 = t2 + t6;
    a3.x = r1 - t4; a1.x = r1 + t4;
    a2.y = i0 - t6; a0.y = i0 + t6;
}
__device__ __forceinline__ void fft2r(float2 &a, float2 &b)
{
    const float2 s0 = a, s1 = b;
    a = make_float2(s0.x + s1.x, s0.y + s1.y);
    b = make_float2(s0.x - s1.x, s0.y - s1.y);
}
__device__ __forceinline__ void bfly_nomul(float2 &a0, float2 &a1, float2 &a2, float2 &a3) { butterflies(a0, a1, a2, a3, a2.x, a2.y, a3.x, a3.y); }
__device__ __forceinline__ void bfly_mul(float2 &a0, float2 &a1, float2 &a2, float2 &a3, float wre, float wim)
{
    const float t1 = a2.x * wre - a2.y * (-wim);
    const float t2 = a2.x * (-wim) + a2.y * wre;
    const float t5 = a3.x * wre - a3.y * wim;
    const float t6 = a3.x * wim + a3.y * wre;
    butterflies(a0, a1, a2, a3, t1, t2, t5, t6);
}
__device__ __forceinline__ void bfly_w(float2 &a0, float2 &a1, float2 &a2, float2 &a3, float2 w) { bfly_mul(a0, a1, a2, a3, w.x, w.y); }

// one aligned chunk of 16 samples: a size-16 block (ff_tx_fft16_ns, tx_template.c:681-704) or two size-8 blocks (ff_tx_fft8_ns,
// :660-679); the part the two cases share is done once so that a warp holding both kinds diverges over five butterflies only
__device__ __forceinline__ void leaf16(float2 *v, bool full, float c8, float c1, float c2, float c3)
{
    fft2r(v[0], v[1]); fft2r(v[4], v[5]); fft2r(v[6], v[7]);
    bfly_nomul(v[0], v[1], v[2], v[3]);
    bfly_nomul(v[0], v[2], v[4], v[6]);
    bfly_mul(v[1], v[3], v[5], v[7], c8, c8);
    fft2r(v[8], v[9]);
    bfly_nomul(v[8], v[9], v[10], v[11]);
    fft2r(v[12], v[13]);
    if (full) {
        bfly_nomul(v[12], v[13], v[14], v[15]);
        bfly_nomul(v[0], v[4], v[8], v[12]);
        bfly_mul(v[2], v[6], v[10], v[14], c2, c2);
        bfly_mul(v[1], v[5], v[9], v[13], c1, c3);
        bfly_mul(v[3], v[7], v[11], v[15], c3, c1);
    } else {
        fft2r(v[14], v[15]);
        bfly_nomul(v[8], v[10], v[12], v[14]);
        bfly_mul(v[9], v[11], v[13], v[15], c8, c8);
    }
}

// combines of NL levels on one item (16 samples for NL = 3, 8 for NL = 2); tw: level a+1 {0}, a+2 {1, 2}, a+3 {3..6}
template <int NL>
__device__ __forceinline__ void combine_item(float2 *x, const float2 *tw, bool full)
{
    bfly_w(x[0], x[1], x[2], x[3], tw[0]);
    if (NL == 3) {
        bfly_w(x[0], x[2], x[4], x[6], tw[1]);
        bfly_w(x[1], x[3], x[5], x[7], tw[2]);
        bfly_w(x[8], x[9], x[10], x[11], tw[0]);
        if (full) {
            bfly_w(x[12], x[13], x[14], x[15], tw[0]);
#pragma unroll
            for (int u = 0; u < 4; u++) bfly_w(x[u], x[u + 4], x[u + 8], x[u + 12], tw[3 + u]);
        } else {
            bfly_w(x[8], x[10], x[12], x[14], tw[1]);
            bfly_w(x[9], x[11], x[13], x[15], tw[2]);
        }
    } else {
        if (full) {
            bfly_w(x[0], x[2], x[4], x[6], tw[1]);
            bfly_w(x[1], x[3], x[5], x[7], tw[2]);
        } else {
            bfly_w(x[4], x[5], x[6], x[7], tw[0]);
        }
    }
}

// ------------------------------------------------------------------------------------------------ async-copy plumbing
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t a, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(a), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t a, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(a), "r"(bytes) : "memory"); }
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t mbar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(dst), "l"(src), "r"(bytes), "r"(mbar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t a, uint32_t parity)
{
    uint32_t ok;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(a), "r"(parity) : "memory");
    } while (!ok);
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

template <int G>
__device__ __forceinline__ void group_sync(int group)
{
    if (G == 32) __syncwarp();
    else if (G == 256) __syncthreads();
    else asm volatile("bar.sync %0, %1;" :: "r"(group + 1), "n"(G) : "memory");
}

// ------------------------------------------------------------------------------------------------ plan layout (words per thread)
__host__ __device__ constexpr int ntw(int nl) { return nl == 3 ? 7 : 3; }
__host__ __device__ constexpr int items(int nl) { return nl == 3 ? 1 : 2; }
__host__ __device__ constexpr int pass_words(int nl) { return nl == 0 ? 0 : items(nl) * (3 + 2 * ntw(nl)); }
constexpr int LEAF_WORDS = 13;          // 8 packed source offsets, kind, c8, c1, c2, c3

template <int NL>
struct PassRegs {
    int base[items(NL)], kind[items(NL)], gidx[items(NL)];
    float2 tw[items(NL)][ntw(NL)];
    __device__ __forceinline__ void load(const uint32_t *plan, int w0, int G, int tg)
    {
#pragma unroll
        for (int s = 0; s < items(NL); s++) {
            const uint32_t *p = plan + (size_t)(w0 + s * (3 + 2 * ntw(NL))) * G + tg;
            base[s] = (int)p[0]; kind[s] = (int)p[G]; gidx[s] = (int)p[2 * G];
#pragma unroll
            for (int k = 0; k < ntw(NL); k++)
                tw[s][k] = make_float2(__uint_as_float(p[(size_t)(3 + 2 * k) * G]), __uint_as_float(p[(size_t)(4 + 2 * k) * G]));
        }
    }
};

// shared-memory index (in float2) of sample t of an item: z index e lives at e + (e >> 4)
template <int Q>
__device__ __forceinline__ int zidx(int base, int t) { return Q >= 16 ? base + t * (Q + Q / 16) : base + 8 * t + (t >> 1); }

// a pass that is not the last one: shared memory -> registers -> combines -> shared memory (in place: no barrier in between)
template <int NL, int Q>
__device__ __forceinline__ void mid_pass(float2 *buf, const PassRegs<NL> &r)
{
    constexpr int E = 2 << NL;
#pragma unroll
    for (int s = 0; s < items(NL); s++) {
        float2 x[E];
#pragma unroll
        for (int t = 0; t < E; t++) x[t] = buf[zidx<Q>(r.base[s], t)];
        combine_item<NL>(x, r.tw[s], r.kind[s] != 0);
#pragma unroll
        for (int t = 0; t < E; t++) buf[zidx<Q>(r.base[s], t)] = x[t];
    }
}

// the last pass: results go to global memory; MODE 1 applies the MDCT post-rotation (tx_template.c:1333-1341):
// out[e].re = z[e].im * exp[e].im - z[e].re * exp[e].re,  out[e].im = z[e'].im * exp[e'].re + z[e'].re * exp[e'].im with e' = n-1-e,
// and e' is sample E-1-t of the same item slot of lane 31 - lane (host-side column mapping)
template <int NL, int Q, int MODE>
__device__ __forceinline__ void last_pass(const float2 *buf, const PassRegs<NL> &r, float2 *dst, const float2 *expS, int lane)
{
    constexpr int E = 2 << NL;
#pragma unroll
    for (int s = 0; s < items(NL); s++) {
        float2 x[E];
#pragma unroll
        for (int t = 0; t < E; t++) x[t] = buf[zidx<Q>(r.base[s], t)];
        combine_item<NL>(x, r.tw[s], r.kind[s] != 0);
        if (MODE == 1) {
            float b[E];
#pragma unroll
            for (int t = 0; t < E; t++) {
                const float2 e = expS[r.gidx[s] + t * Q];
                const float a = x[t].y * e.y - x[t].x * e.x;
                b[t] = x[t].y * e.x + x[t].x * e.y;
                x[t].x = a;
            }
#pragma unroll
            for (int t = 0; t < E; t++) x[t].y = __shfl_sync(0xffffffffu, b[E - 1 - t], 31 - lane);
        }
#pragma unroll
        for (int t = 0; t < E; t++) dst[r.gidx[s] + t * Q] = x[t];
    }
}

// LOGN: log2 of the complex points; MODE 0 FFT, 1 inverse MDCT; NL1..NL3: levels per pass after the leaf pass (0 = no such pass)
template <int LOGN, int MODE, int NL1, int NL2, int NL3>
__global__ void __launch_bounds__(256, 2)
tx_r16_kernel(const uint32_t *__restrict__ plan, const float2 *__restrict__ exp_nat, char *__restrict__ out, const char *__restrict__ in,
              long long out_step, long long in_step, long long count, int leaf_perm)
{
    constexpr int N = 1 << LOGN, G = N / 16, GROUPS = 256 / G, ZS = N + N / 16;
    constexpr int Q1 = 8, Q2 = 1 << (4 + NL1 - 1), Q3 = 1 << (4 + NL1 + NL2 - 1);
    constexpr int W1 = LEAF_WORDS, W2 = W1 + pass_words(NL1), W3 = W2 + pass_words(NL2);
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float2 *zbuf = reinterpret_cast<float2 *>(smem_raw);                                   // [GROUPS][2][ZS]
    float2 *expS = zbuf + (size_t)GROUPS * 2 * ZS;                                         // [N] (MODE 1)
    uint64_t *mbar = reinterpret_cast<uint64_t *>(expS + (MODE == 1 ? N : 0));             // [GROUPS][2]

    const int g = threadIdx.x / G, tg = threadIdx.x % G, lane = threadIdx.x & 31;
    // loop-invariant per-thread state.  Leaf chunk of this thread: the 16 lanes of a half-warp take chunks whose low four bits AND
    // whose top four bits are all different -- the permuted source samples of chunk c sit at (roughly bit-reversed c) + k N/16, so the
    // top bits of c pick the bank of the reads while the low bits pick the bank of the 17-strided writes; consecutive chunks per warp
    // made the reads an 8-way (N = 2048) / 4-way (N = 1024) bank conflict
    const int lt = (G > 16 && leaf_perm) ? (tg & 15) + 16 * (((tg & 15) ^ (tg >> 4)) & (G / 16 - 1)) : tg;
    uint32_t off[8];
#pragma unroll
    for (int k = 0; k < 8; k++) off[k] = plan[(size_t)k * G + lt];
    const bool leaf_full = plan[(size_t)8 * G + lt] != 0;
    const float c8 = __uint_as_float(plan[(size_t)9 * G + lt]), c1 = __uint_as_float(plan[(size_t)10 * G + lt]),
                c2 = __uint_as_float(plan[(size_t)11 * G + lt]), c3 = __uint_as_float(plan[(size_t)12 * G + lt]);
    PassRegs<NL1> r1; r1.load(plan, W1, G, tg);
    PassRegs<NL2> r2; r2.load(plan, W2, G, tg);
    PassRegs<NL3 ? NL3 : 2> r3;
    if constexpr (NL3 != 0) r3.load(plan, W3, G, tg);

    if (MODE == 1)
        for (int i = threadIdx.x; i < N; i += 256) expS[i] = exp_nat[i];
    float2 *buf0 = zbuf + (size_t)(g * 2) * ZS, *buf1 = buf0 + ZS;
    const uint32_t mb0 = smem_u32(mbar + g * 2), mb1 = mb0 + 8;
    if (tg == 0) { mbar_init(mb0, 1); mbar_init(mb1, 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
    __syncthreads();

    const long long stride = (long long)gridDim.x * GROUPS;
    long long t = (long long)blockIdx.x * GROUPS + g;
    constexpr uint32_t BYTES = N * 8;
    if (tg == 0) {
        if (t < count)          { mbar_expect_tx(mb0, BYTES); bulk_g2s(smem_u32(buf0), in + t * in_step, BYTES, mb0); }
        if (t + stride < count) { mbar_expect_tx(mb1, BYTES); bulk_g2s(smem_u32(buf1), in + (t + stride) * in_step, BYTES, mb1); }
    }
    for (int it = 0; t < count; t += stride, it++) {
        float2 *buf = (it & 1) ? buf1 : buf0;
        const uint32_t mb = (it & 1) ? mb1 : mb0;
        mbar_wait(mb, (it >> 1) & 1);
        // ---- leaf pass: permuted read (and MDCT pre-rotation, tx_template.c:1322-1327), sizes 2..16 in registers
        float2 v[16];
        {
            const char *src = reinterpret_cast<const char *>(buf);
#pragma unroll
            for (int i = 0; i < 16; i++) {
                const uint32_t o = (i & 1) ? (off[i >> 1] >> 16) : (off[i >> 1] & 0xffffu);
                if (MODE == 0) {
                    v[i] = *reinterpret_cast<const float2 *>(src + o);
                } else {
                    const float aim = *reinterpret_cast<const float *>(src + o);                       // in1[2m]
                    const float are = *reinterpret_cast<const float *>(src + (8 * N - 4) - o);         // in2[-2m] = src[len - 1 - 2m]
                    const float2 w = *reinterpret_cast<const float2 *>(reinterpret_cast<const char *>(expS) + o);
                    v[i] = make_float2(are * w.x - aim * w.y, are * w.y + aim * w.x);
                }
            }
        }
        group_sync<G>(g);                              // everybody has its samples: the buffer can now hold z
        leaf16(v, leaf_full, c8, c1, c2, c3);
#pragma unroll
        for (int i = 0; i < 16; i++) buf[17 * lt + i] = v[i];
        group_sync<G>(g);
        // ---- passes over levels 5 and up
        char *dstb = out + t * out_step;
        mid_pass<NL1, Q1>(buf, r1);
        group_sync<G>(g);
        if constexpr (NL3 != 0) {
            mid_pass<NL2, Q2>(buf, r2);
            group_sync<G>(g);
            last_pass<NL3 ? NL3 : 2, Q3, MODE>(buf, r3, reinterpret_cast<float2 *>(dstb), expS, lane);
        } else {
            last_pass<NL2, Q2, MODE>(buf, r2, reinterpret_cast<float2 *>(dstb), expS, lane);
        }
        group_sync<G>(g);                              // the buffer is free again: fetch the transform two rounds ahead into it
        if (tg == 0 && t + 2 * stride < count) {
            fence_proxy_async();
            mbar_expect_tx(mb, BYTES);
            bulk_g2s(smem_u32(buf), in + (t + 2 * stride) * in_step, BYTES, mb);
        }
    }
}

// ------------------------------------------------------------------------------------------------ host: plan
void collect_blocks(std::vector<std::vector<int>> &lv, int L, int off)
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

bool has(const std::vector<int> &v, int x) { for (int y : v) if (y == x) return true; return false; }

std::vector<float> cos_tab(int L)               // ff_tx_init_tab_N (tx_template.c:65-77): N/4 cosines in double, rounded, then 0
{
    const int N = 1 << L;
    std::vector<float> t;
    const double freq = 2 * M_PI / N;
    for (int i = 0; i < N / 4; i++) t.push_back((float)cos(i * freq));
    t.push_back(0.0f);
    return t;
}

uint32_t fbits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

} // namespace

struct TxR16 {
    int mode = 0, n = 0, logn = 0, G = 0, groups = 0, grid_cap = 0, leaf_perm = 1;
    size_t smem = 0;
    uint32_t *plan = nullptr;
    float2 *exp_nat = nullptr;
    void (*kernel)(const uint32_t *, const float2 *, char *, const char *, long long, long long, long long, int) = nullptr;
};

template <int LOGN, int MODE, int A, int B, int C>
static int r16_bind(TxR16 *p, int sm_count)
{
    p->kernel = tx_r16_kernel<LOGN, MODE, A, B, C>;
    if (cudaFuncSetAttribute(p->kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->smem) != cudaSuccess) return -1;
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, p->kernel, 256, p->smem) != cudaSuccess || per_sm < 1) return -1;
    p->grid_cap = per_sm * sm_count;
    return 0;
}

// the per-thread words of a transform (layout: word w of thread tg at plan[w * G + tg]); empty when the size is not covered
static std::vector<uint32_t> r16_plan(int n, const int *gather, int *logn_out)
{
    std::vector<uint32_t> none;
    int logn = 0;
    while ((1 << logn) < n) logn++;
    if ((1 << logn) != n || logn < 9 || logn > 12) return none;
    *logn_out = logn;
    static const int NLS[13][3] = { {0}, {0}, {0}, {0}, {0}, {0}, {0}, {0}, {0}, {3, 2, 0}, {3, 3, 0}, {3, 2, 2}, {3, 3, 2} };
    const int *nl = NLS[logn];
    const int G = n / 16;
    std::vector<std::vector<int>> lv(18);
    collect_blocks(lv, logn, 0);
    int words = LEAF_WORDS;
    for (int k = 0; k < 3; k++) words += pass_words(nl[k]);
    std::vector<uint32_t> plan((size_t)words * G, 0);
    auto W = [&](int w, int tg) -> uint32_t & { return plan[(size_t)w * G + tg]; };
    const std::vector<float> t8 = cos_tab(3), t16 = cos_tab(4);
    for (int tg = 0; tg < G; tg++) {                               // leaf pass: thread tg owns z[16 tg .. 16 tg + 15]
        for (int i = 0; i < 16; i++) {
            const uint32_t o = (uint32_t)gather[16 * tg + i] * 8u;          // byte offset of the source sample (FFT) / of in1[2m] (MDCT)
            W(i >> 1, tg) |= (i & 1) ? (o << 16) : o;
        }
        const bool full = has(lv[4], 16 * tg);
        if (!full && !(has(lv[3], 16 * tg) && has(lv[3], 16 * tg + 8))) return none;
        W(8, tg) = full;
        W(9, tg) = fbits(t8[1]); W(10, tg) = fbits(t16[1]); W(11, tg) = fbits(t16[2]); W(12, tg) = fbits(t16[3]);
    }
    int a = 4, w0 = LEAF_WORDS;
    for (int k = 0; k < 3 && nl[k]; k++) {
        const int NL = nl[k], b = a + NL, q = 1 << (a - 1), C = 1 << b, E = 2 << NL;
        const bool last = (k == 2) || nl[k + 1] == 0;
        std::vector<std::vector<float>> tabs;
        for (int l = 1; l <= NL; l++) tabs.push_back(cos_tab(a + l));
        for (int tg = 0; tg < G; tg++)
            for (int s = 0; s < items(NL); s++) {
                const int I = tg + s * G;                          // item number, n / E of them
                int m, j;
                if (last) {                                        // one chunk; columns paired so that j and q-1-j sit in lanes l and 31-l
                    const int vw = I / 32, l = I % 32;
                    if (q < 32) return none;
                    m = 0;
                    j = l < 16 ? 16 * vw + l : q - 1 - (16 * vw + 31 - l);
                } else {
                    m = I / q; j = I % q;
                }
                const int o = m * C;
                const bool full = has(lv[b], o);
                if (!full && !(has(lv[b - 1], o) && has(lv[b - 1], o + C / 2))) return none;
                const int wb = w0 + s * (3 + 2 * ntw(NL));
                W(wb + 0, tg) = (uint32_t)((o + j) + ((o + j) >> 4));
                W(wb + 1, tg) = full;
                W(wb + 2, tg) = (uint32_t)(o + j);
                int k2 = 0;
                for (int l = 1; l <= NL; l++) {                   // level a+l: 2^(l-1) butterflies of this thread, columns j + u q
                    const int q4 = 1 << (a + l - 2);
                    for (int u = 0; u < (1 << (l - 1)); u++, k2++) {
                        const int jj = j + u * q;
                        W(wb + 3 + 2 * k2, tg) = fbits(tabs[l - 1][jj]);
                        W(wb + 4 + 2 * k2, tg) = fbits(tabs[l - 1][q4 - jj]);
                    }
                }
                (void)E;
            }
        a = b; w0 += pass_words(NL);
    }
    if (a != logn) return none;
    return plan;
}

TxR16 *tx_r16_create(int mode, int n, const int *gather, const float2 *exp_nat, int sm_count)
{
    if (mode != 0 && mode != 1) return nullptr;
    int logn = 0;
    const std::vector<uint32_t> plan = r16_plan(n, gather, &logn);
    if (plan.empty()) return nullptr;
    const int G = n / 16;
    TxR16 *p = new TxR16();
    p->mode = mode; p->n = n; p->logn = logn; p->G = G; p->groups = 256 / G;
    // the conflict-free leaf assignment pays where shared memory bounds the transform (2048 and 512 points), but the 1024-point FFT,
    // which it does not bound, runs slower with it
    p->leaf_perm = !(logn == 10 && mode == 0);
    const size_t zs = (size_t)n + n / 16;
    p->smem = (size_t)p->groups * 2 * zs * 8 + (mode == 1 ? (size_t)n * 8 : 0) + (size_t)p->groups * 2 * 8;
    int rc = -1;
    switch (logn * 2 + mode) {
    case 18: rc = r16_bind<9, 0, 3, 2, 0>(p, sm_count); break;
    case 19: rc = r16_bind<9, 1, 3, 2, 0>(p, sm_count); break;
    case 20: rc = r16_bind<10, 0, 3, 3, 0>(p, sm_count); break;
    case 21: rc = r16_bind<10, 1, 3, 3, 0>(p, sm_count); break;
    case 22: rc = r16_bind<11, 0, 3, 2, 2>(p, sm_count); break;
    case 23: rc = r16_bind<11, 1, 3, 2, 2>(p, sm_count); break;
    case 24: rc = r16_bind<12, 0, 3, 3, 2>(p, sm_count); break;
    case 25: rc = r16_bind<12, 1, 3, 3, 2>(p, sm_count); break;
    }
    if (rc < 0 || cudaMalloc(&p->plan, plan.size() * 4) != cudaSuccess) { delete p; return nullptr; }
    cudaMemcpy(p->plan, plan.data(), plan.size() * 4, cudaMemcpyHostToDevice);
    if (mode == 1) {
        if (!exp_nat || cudaMalloc(&p->exp_nat, (size_t)n * 8) != cudaSuccess) { cudaFree(p->plan); delete p; return nullptr; }
        cudaMemcpy(p->exp_nat, exp_nat, (size_t)n * 8, cudaMemcpyHostToDevice);
    }
    return p;
}

void tx_r16_destroy(TxR16 *p)
{
    if (!p) return;
    if (p->plan) cudaFree(p->plan);
    if (p->exp_nat) cudaFree(p->exp_nat);
    delete p;
}

bool tx_r16_accepts(const TxR16 *p, const void *out, const void *in, long long out_step, long long in_step)
{
    return p && !((uintptr_t)in & 15) && !(in_step & 15) && !((uintptr_t)out & 7) && !(out_step & 7);
}

int tx_r16_launch(TxR16 *p, cudaStream_t st, void *out, const void *in, long long out_step, long long in_step, long long count)
{
    if (count <= 0) return 0;
    long long blocks = (count + p->groups - 1) / p->groups;
    if (blocks > p->grid_cap) blocks = p->grid_cap;               // persistent CTAs: every group strides over the batch
    p->kernel<<<(unsigned)blocks, 256, p->smem, st>>>(p->plan, p->exp_nat, (char *)out, (const char *)in, out_step, in_step, count, p->leaf_perm);
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

// host-only (CPU test tier): the plan words of an n-point transform whose input permutation is ff_tx_gen_ptwo_revtab's for `inv`
static int r16_sr_perm(int i, int len, int inv)                   // split_radix_permutation, libavutil/tx.c:125-134
{
    len >>= 1;
    if (len <= 1) return i & 1;
    if (!(i & len)) return r16_sr_perm(i, len, inv) * 2;
    len >>= 1;
    return r16_sr_perm(i, len, inv) * 4 + 1 - 2 * (!(i & len) ^ inv);
}

B200_API int b200_tx_r16_plan(int n, int inv, uint32_t *words, int cap)
{
    if (n < 2 || (n & (n - 1))) return B200_EINVAL;
    std::vector<int> gather(n);
    for (int i = 0; i < n; i++) gather[i] = (-r16_sr_perm(i, n, inv)) & (n - 1);
    int logn = 0;
    const std::vector<uint32_t> plan = r16_plan(n, gather.data(), &logn);
    if (plan.empty()) return B200_ENOSYS;
    if (words) {
        if ((int)plan.size() > cap) return B200_EINVAL;
        memcpy(words, plan.data(), plan.size() * 4);
    }
    return (int)plan.size();
}

