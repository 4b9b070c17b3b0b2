// tx_dct.cu — libavutil/tx AV_TX_FLOAT_DCT on sm_90a: DCT-II (forward) and DCT-III (inverse).
//
// Reference semantics reproduced bit for bit (checker: the DCT part of oracle/tx_oracle.c), libavutil/tx_template.c:
//   :1832-1872 ff_tx_dct_init   (the inverse is set up on twice the length it is asked for; scale halved; factor table)
//   :1874-1925 ff_tx_dctII      pre-butterflies, real-to-complex DFT of len points, then a rotation whose odd outputs are a running sum
//   :1927-1968 ff_tx_dctIII     rotation, complex-to-real DFT, post-butterflies
// The DFT in the middle is the real transform of tx.cu (b200_tx_batch_device on a child context); the stages around it are the
// kernels below.  The DCT-II post stage accumulates `next += tmp` over len/2 steps in the reference's order, so it is one thread
// per transform (a parallel scan would round differently); the other three stages are one thread per butterfly.
// Unlike the reference the caller's input is not overwritten: the stages work in a scratch area.
#include "tx_dct.h"
#include <vector>
#include <cmath>

namespace {

// [device-code tx_dct] (tests/cuda_emu runs this block on the CPU against the checker; comment markers only)
// forward, before the DFT: S[i], S[len-1-i] from src[i], src[len-1-i]  (tx_template.c:1889-1909)
__global__ void __launch_bounds__(256)
tx_dct2_pre_kernel(const float *exp, int len, const float *in, long long in_step, float *S, long long s_step, long long count)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const long long tr = blockIdx.y;
    if (i >= (len >> 1) || tr >= count) return;
    const float *src = reinterpret_cast<const float *>(reinterpret_cast<const char *>(in) + tr * in_step);
    float *s = S + tr * s_step;
    const float in1 = src[i], in2 = src[len - i - 1], k = exp[len + i];
    const float tmp1 = (in1 + in2) * 0.5f, tmp2 = (in1 - in2) * k;
    s[i] = tmp1 + tmp2;
    s[len - i - 1] = tmp1 - tmp2;
}

// forward, after the DFT (D holds len + 2 floats per transform): tx_template.c:1913-1924, sequential in i like the reference
__global__ void __launch_bounds__(64)
tx_dct2_post_kernel(const float *exp, int len, const float *D, long long d_step, float *out, long long out_step, long long count)
{
    const long long tr = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (tr >= count) return;
    const float *d = D + tr * d_step;
    float *dst = reinterpret_cast<float *>(reinterpret_cast<char *>(out) + tr * out_step);
    float next = d[len];
    for (int i = len - 2; i > 0; i -= 2) {
        const float are = exp[len - i], aim = exp[i], bre = d[i + 0], bim = d[i + 1];
        const float tmp = are * bre - aim * bim;
        dst[i] = are * bim + aim * bre;
        dst[i + 1] = next;
        next += tmp;
    }
    dst[0] = exp[0] * d[0];
    dst[1] = next;
}

// inverse, before the DFT: S gets len + 2 floats per transform (tx_template.c:1936-1951)
__global__ void __launch_bounds__(256)
tx_dct3_pre_kernel(const float *exp, int len, const float *in, long long in_step, float *S, long long s_step, long long count)
{
    const int p = blockIdx.x * blockDim.x + threadIdx.x;               // pair index: i = 2 * p
    const long long tr = blockIdx.y;
    if (p >= (len >> 1) || tr >= count) return;
    const float *src = reinterpret_cast<const float *>(reinterpret_cast<const char *>(in) + tr * in_step);
    float *s = S + tr * s_step;
    const int i = 2 * p;
    if (i == 0) {
        s[0] = src[0]; s[1] = src[1];
        s[len] = 2 * src[len - 1]; s[len + 1] = 0.0f;
        return;
    }
    const float val1 = src[i], val2 = src[i - 1] - src[i + 1];
    const float are = exp[len - i], aim = exp[i];
    s[i + 1] = are * val1 - aim * val2;
    s[i] = are * val2 + aim * val1;
}

// inverse, after the DFT, in place on the output (tx_template.c:1955-1967)
__global__ void __launch_bounds__(256)
tx_dct3_post_kernel(const float *exp, int len, float *out, long long out_step, long long count)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const long long tr = blockIdx.y;
    if (i >= (len >> 1) || tr >= count) return;
    float *dst = reinterpret_cast<float *>(reinterpret_cast<char *>(out) + tr * out_step);
    const float in1 = dst[i], in2 = dst[len - i - 1], c = exp[len + i];
    const float tmp1 = in1 + in2;
    float tmp2 = in1 - in2;
    tmp2 *= c;
    dst[i] = tmp1 + tmp2;
    dst[len - i - 1] = tmp1 - tmp2;
}
// [/device-code tx_dct]

} // namespace

struct TxDct {
    B200Device *dev = nullptr;
    int inv = 0, n = 0;                        // n: points (len forward, 2 * len inverse)
    B200TXContext *sub = nullptr;              // r2c (forward) / c2r (inverse) of n points
    float *exp = nullptr;                      // device: n rotation factors + n/2 butterfly factors
    void *scratch = nullptr; size_t scratch_bytes = 0;
};

bool tx_dct_length_ok(int inv, int len)
{
    const long long n = inv ? 2LL * len : len;
    return len > 0 && n >= 4 && n <= 32768 && !(n & (n - 1));
}
int tx_dct_points(const TxDct *p) { return p->n; }

// the factor table of ff_tx_dct_init, host side (also handed to the CPU test tier)
static void dct_host_table(std::vector<float> &tab, int inv, int n)
{
    tab.assign((size_t)(n / 2) * 3, 0.f);
    const double freq = M_PI / (n * 2);
    for (int i = 0; i < n; i++) tab[i] = (float)(cos(i * freq) * (!inv + 1));
    for (int i = 0; i < n / 2; i++) tab[n + i] = inv ? (float)(0.5 / sin((2 * i + 1) * freq)) : (float)cos((n - 2 * i - 1) * freq);
}
B200_API int b200_tx_dct_table(int inv, int len, float *tab, int cap)
{
    if (!tx_dct_length_ok(inv, len)) return B200_ENOSYS;
    const int n = inv ? 2 * len : len;
    std::vector<float> t;
    dct_host_table(t, inv, n);
    if (tab && cap >= (int)t.size()) memcpy(tab, t.data(), t.size() * sizeof(float));
    return (int)t.size();
}

TxDct *tx_dct_create(B200Device *dev, int inv, int len, float scale)
{
    if (!tx_dct_length_ok(inv, len)) return nullptr;
    TxDct *p = new (std::nothrow) TxDct();
    if (!p) return nullptr;
    p->dev = dev; p->inv = inv; p->n = inv ? 2 * len : len;
    float rsc = scale;
    if (inv) rsc *= 0.5f;
    if (b200_tx_init_device(dev, &p->sub, nullptr, B200_TX_FLOAT_RDFT, inv, p->n, &rsc, 0) < 0) { delete p; return nullptr; }
    std::vector<float> tab;
    dct_host_table(tab, inv, p->n);
    if (cudaMalloc(&p->exp, tab.size() * sizeof(float)) != cudaSuccess ||
        cudaMemcpy(p->exp, tab.data(), tab.size() * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) {
        b200_set_error("tx_dct_create: device table");
        tx_dct_free(p);
        return nullptr;
    }
    return p;
}

void tx_dct_free(TxDct *p)
{
    if (!p) return;
    if (p->sub) b200_tx_uninit(&p->sub);
    if (p->exp) cudaFree(p->exp);
    if (p->scratch) cudaFree(p->scratch);
    delete p;
}

int tx_dct_launch(TxDct *p, cudaStream_t st, void *out, const void *in, int64_t count, ptrdiff_t out_step, ptrdiff_t in_step)
{
    if (count <= 0) return 0;
    // the stages around the DFT move single floats; the inverse's c2r writes the caller's output as float2 words
    if (((uintptr_t)in | (uintptr_t)in_step) & 3) {
        b200_set_error("b200_tx_batch_device: DCT input pointer and in_step must be multiples of 4 bytes");
        return B200_EINVAL;
    }
    if (((uintptr_t)out | (uintptr_t)out_step) & (p->inv ? 7 : 3)) {
        b200_set_error("b200_tx_batch_device: DCT output pointer and out_step must be multiples of %d bytes", p->inv ? 8 : 4);
        return B200_EINVAL;
    }
    const int n = p->n;
    const size_t line = (size_t)n + 2;                                  // floats per transform in each scratch area
    const int64_t chunk_max = (int64_t)((size_t)(256u << 20) / (2 * line * sizeof(float)));
    int64_t chunk = count < chunk_max ? count : chunk_max;
    if (chunk > 65535) chunk = 65535;                                   // grid.y
    const size_t need = 2 * line * sizeof(float) * (size_t)chunk;
    if (p->scratch_bytes < need) {
        if (p->scratch) { cudaStreamSynchronize(st); cudaFree(p->scratch); p->scratch = nullptr; p->scratch_bytes = 0; }
        B200_CUDA_OK(cudaMalloc(&p->scratch, need));
        p->scratch_bytes = need;
    }
    float *S = (float *)p->scratch, *D = S + line * (size_t)chunk;
    const long long ls = (long long)line;
    for (int64_t c0 = 0; c0 < count; c0 += chunk) {
        const long long cnt = count - c0 < chunk ? count - c0 : chunk;
        char *o = (char *)out + c0 * out_step;
        const char *i = (const char *)in + c0 * in_step;
        const dim3 gb(b200_ceil_div(n >> 1, 256), (unsigned)cnt), tb(256);
        if (!p->inv) {
            tx_dct2_pre_kernel<<<gb, tb, 0, st>>>(p->exp, n, (const float *)i, (long long)in_step, S, ls, cnt);
            B200_LAUNCHED();
            int ret = b200_tx_batch_device(p->sub, D, S, 4, cnt, (ptrdiff_t)(line * sizeof(float)), (ptrdiff_t)(line * sizeof(float)));
            if (ret < 0) return ret;
            tx_dct2_post_kernel<<<(unsigned)b200_ceil_div(cnt, 64), 64, 0, st>>>(p->exp, n, D, ls, (float *)o, (long long)out_step, cnt);
            B200_LAUNCHED();
        } else {
            tx_dct3_pre_kernel<<<gb, tb, 0, st>>>(p->exp, n, (const float *)i, (long long)in_step, S, ls, cnt);
            B200_LAUNCHED();
            int ret = b200_tx_batch_device(p->sub, o, S, 4, cnt, out_step, (ptrdiff_t)(line * sizeof(float)));
            if (ret < 0) return ret;
            tx_dct3_post_kernel<<<gb, tb, 0, st>>>(p->exp, n, (float *)o, (long long)out_step, cnt);
            B200_LAUNCHED();
        }
    }
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}
