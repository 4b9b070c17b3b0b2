// fdsp.cu — libavutil's AVFloatDSPContext on sm_90a (C ABI: "float_dsp").
//
// Reference semantics reproduced bit-for-bit (checker: oracle/fdsp_oracle.c): libavutil/float_dsp.c:27-141 and
// libavutil/float_scalarproduct.c:25-33, the C functions avpriv_float_dsp_alloc() installs.  Every product and every sum is
// rounded on its own (the library is built with --fmad=false, and the kernels spell the operations with __fmul_rn / __fadd_rn
// so no later flag change can fuse them); the scalar products accumulate left to right in the element type like the C loops,
// one thread per vector — they are exact, not fast: a tree reduction would change the rounding.
//
// Batched kernels: grid.x over the elements of a vector, grid.y over vectors; vector v of operand k starts at base_k + v*stride_k
// (stride 0 = shared by all vectors: the window of vector_fmul_window, a common gain table, ...).  Streaming, HBM-bound:
// 8-16 B per element.
#include "common.h"
#include <cstring>

namespace {

// [device-code fdsp] (tests/cuda_emu runs this block on the CPU against the checker; comment markers only)
template <typename T> __device__ __forceinline__ T mul_rn(T a, T b);
template <> __device__ __forceinline__ float  mul_rn(float a, float b)   { return __fmul_rn(a, b); }
template <> __device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
template <typename T> __device__ __forceinline__ T add_rn(T a, T b);
template <> __device__ __forceinline__ float  add_rn(float a, float b)   { return __fadd_rn(a, b); }
template <> __device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
template <typename T> __device__ __forceinline__ T sub_rn(T a, T b) { return add_rn(a, -b); }

struct Operands {
    void *dst; const void *src0, *src1, *src2;
    long long dstS, src0S, src1S, src2S;     // strides between vectors, in elements
};

template <typename T, int OP>
__global__ void __launch_bounds__(256)
fdsp_kernel(Operands o, long long v0, int len, T mul)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= len) return;
    const long long v = v0 + blockIdx.y;
    T *dst = static_cast<T *>(o.dst) + v * o.dstS;
    const T *src0 = static_cast<const T *>(o.src0) + v * o.src0S;
    const T *src1 = static_cast<const T *>(o.src1) + v * o.src1S;
    const T *src2 = static_cast<const T *>(o.src2) + v * o.src2S;
    if (OP == B200_FDSP_VECTOR_FMUL || OP == B200_FDSP_VECTOR_DMUL) dst[i] = mul_rn(src0[i], src1[i]);
    else if (OP == B200_FDSP_VECTOR_FMAC_SCALAR || OP == B200_FDSP_VECTOR_DMAC_SCALAR) dst[i] = add_rn(dst[i], mul_rn(src0[i], mul));
    else if (OP == B200_FDSP_VECTOR_FMUL_SCALAR || OP == B200_FDSP_VECTOR_DMUL_SCALAR) dst[i] = mul_rn(src0[i], mul);
    else if (OP == B200_FDSP_VECTOR_FMUL_WINDOW) {
        const int j = 2 * len - 1 - i;                                   // i in [0, len): the pair (i, j) of float_dsp.c:85-92
        const T s0 = src0[i], s1 = src1[j - len], wi = src2[i], wj = src2[j];
        dst[i] = sub_rn(mul_rn(s0, wj), mul_rn(s1, wi));
        dst[j] = add_rn(mul_rn(s0, wi), mul_rn(s1, wj));
    }
    else if (OP == B200_FDSP_VECTOR_FMUL_ADD) dst[i] = add_rn(mul_rn(src0[i], src1[i]), src2[i]);
    else if (OP == B200_FDSP_VECTOR_FMUL_REVERSE) dst[i] = mul_rn(src0[i], src1[len - 1 - i]);
    else if (OP == B200_FDSP_BUTTERFLIES_FLOAT) {
        T *v2 = const_cast<T *>(src0);
        const T a = dst[i], b = v2[i];
        dst[i] = add_rn(a, b);
        v2[i] = sub_rn(a, b);
    }
}

// scalarproduct_float / _double: one thread per vector, sum in the C loop's order
template <typename T>
__global__ void __launch_bounds__(128)
fdsp_dot_kernel(Operands o, long long nvec, int len)
{
    const long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nvec) return;
    const T *a = static_cast<const T *>(o.src0) + v * o.src0S, *b = static_cast<const T *>(o.src1) + v * o.src1S;
    T p = 0;
    for (int i = 0; i < len; i++) p = add_rn(p, mul_rn(a[i], b[i]));
    static_cast<T *>(o.dst)[v * o.dstS] = p;
}

// [/device-code fdsp]
template <typename T, int OP>
int launch_op(cudaStream_t st, const Operands &o, long long nvec, int len, double mul)
{
    dim3 t(256);
    for (long long v0 = 0; v0 < nvec; v0 += 65535) {
        const long long nv = nvec - v0 < 65535 ? nvec - v0 : 65535;
        dim3 g((unsigned)b200_ceil_div(len, 256), (unsigned)nv);
        fdsp_kernel<T, OP><<<g, t, 0, st>>>(o, v0, len, (T)mul);
        B200_LAUNCHED();
    }
    return 0;
}

int run(B200Device *dev, cudaStream_t st, int op, long long nvec, int len, const Operands &o, double mul)
{
    (void)dev;
    switch (op) {
#define EL(OPC, T) case OPC: return launch_op<T, OPC>(st, o, nvec, len, mul);
    EL(B200_FDSP_VECTOR_FMUL, float) EL(B200_FDSP_VECTOR_FMAC_SCALAR, float) EL(B200_FDSP_VECTOR_DMAC_SCALAR, double)
    EL(B200_FDSP_VECTOR_FMUL_SCALAR, float) EL(B200_FDSP_VECTOR_DMUL_SCALAR, double) EL(B200_FDSP_VECTOR_FMUL_WINDOW, float)
    EL(B200_FDSP_VECTOR_FMUL_ADD, float) EL(B200_FDSP_VECTOR_FMUL_REVERSE, float) EL(B200_FDSP_BUTTERFLIES_FLOAT, float)
    EL(B200_FDSP_VECTOR_DMUL, double)
#undef EL
    case B200_FDSP_SCALARPRODUCT_FLOAT:
        fdsp_dot_kernel<float><<<(unsigned)b200_ceil_div(nvec, 128), 128, 0, st>>>(o, nvec, len); B200_LAUNCHED(); return 0;
    case B200_FDSP_SCALARPRODUCT_DOUBLE:
        fdsp_dot_kernel<double><<<(unsigned)b200_ceil_div(nvec, 128), 128, 0, st>>>(o, nvec, len); B200_LAUNCHED(); return 0;
    }
    return B200_EINVAL;
}

bool is_double(int op)
{
    return op == B200_FDSP_VECTOR_DMAC_SCALAR || op == B200_FDSP_VECTOR_DMUL_SCALAR || op == B200_FDSP_VECTOR_DMUL ||
           op == B200_FDSP_SCALARPRODUCT_DOUBLE;
}
bool uses_src1(int op)
{
    return op == B200_FDSP_VECTOR_FMUL || op == B200_FDSP_VECTOR_DMUL || op == B200_FDSP_VECTOR_FMUL_WINDOW || op == B200_FDSP_VECTOR_FMUL_ADD ||
           op == B200_FDSP_VECTOR_FMUL_REVERSE || op == B200_FDSP_SCALARPRODUCT_FLOAT || op == B200_FDSP_SCALARPRODUCT_DOUBLE;
}
bool uses_src2(int op) { return op == B200_FDSP_VECTOR_FMUL_WINDOW || op == B200_FDSP_VECTOR_FMUL_ADD; }

constexpr const char *kFeature = "float_dsp";

// drop-in: one call through the device (host pointers); returns the scalar product for the two reducing ops
double host_op(int op, void *dst, const void *src0, const void *src1, const void *src2, double mul, int len)
{
    if (len < 0) B200HostCall::fail(kFeature, "negative length");
    if (len == 0) return 0.0;
    const size_t es = is_double(op) ? 8 : 4;
    const bool dot = op == B200_FDSP_SCALARPRODUCT_FLOAT || op == B200_FDSP_SCALARPRODUCT_DOUBLE;
    const size_t nd = dot ? 1 : op == B200_FDSP_VECTOR_FMUL_WINDOW ? 2 * (size_t)len : (size_t)len;
    const size_t n2 = op == B200_FDSP_VECTOR_FMUL_WINDOW ? 2 * (size_t)len : (size_t)len;
    const size_t seg = ((n2 * es) + 255) & ~(size_t)255;
    B200HostCall call(kFeature, nullptr, 4 * seg);
    uint8_t *scr = call.scratch;
    cudaStream_t st = call.stream;
    Operands o = { scr, scr + seg, scr + 2 * seg, scr + 3 * seg, 0, 0, 0, 0 };
    const bool dst_in = op == B200_FDSP_VECTOR_FMAC_SCALAR || op == B200_FDSP_VECTOR_DMAC_SCALAR || op == B200_FDSP_BUTTERFLIES_FLOAT;
    if (dst_in) call.check(cudaMemcpyAsync(scr, dst, nd * es, cudaMemcpyHostToDevice, st), "h2d dst");
    call.check(cudaMemcpyAsync(scr + seg, src0, (size_t)len * es, cudaMemcpyHostToDevice, st), "h2d src0");
    if (uses_src1(op)) call.check(cudaMemcpyAsync(scr + 2 * seg, src1, (size_t)len * es, cudaMemcpyHostToDevice, st), "h2d src1");
    if (uses_src2(op)) call.check(cudaMemcpyAsync(scr + 3 * seg, src2, n2 * es, cudaMemcpyHostToDevice, st), "h2d src2");
    call.launched(run(call.dev, st, op, 1, len, o, mul));
    double ret = 0.0;
    if (dot) {
        union { float f; double d; } r;
        call.check(cudaMemcpyAsync(&r, scr, es, cudaMemcpyDeviceToHost, st), "d2h");
        call.sync();
        return es == 4 ? (double)r.f : r.d;
    }
    call.check(cudaMemcpyAsync(dst, scr, nd * es, cudaMemcpyDeviceToHost, st), "d2h dst");
    if (op == B200_FDSP_BUTTERFLIES_FLOAT) call.check(cudaMemcpyAsync(const_cast<void *>(src0), scr + seg, (size_t)len * es, cudaMemcpyDeviceToHost, st), "d2h v2");
    call.sync();
    return ret;
}

void t_vector_fmul(float *d, const float *a, const float *b, int n) { host_op(B200_FDSP_VECTOR_FMUL, d, a, b, nullptr, 0, n); }
void t_vector_fmac_scalar(float *d, const float *a, float m, int n) { host_op(B200_FDSP_VECTOR_FMAC_SCALAR, d, a, nullptr, nullptr, m, n); }
void t_vector_dmac_scalar(double *d, const double *a, double m, int n) { host_op(B200_FDSP_VECTOR_DMAC_SCALAR, d, a, nullptr, nullptr, m, n); }
void t_vector_fmul_scalar(float *d, const float *a, float m, int n) { host_op(B200_FDSP_VECTOR_FMUL_SCALAR, d, a, nullptr, nullptr, m, n); }
void t_vector_dmul_scalar(double *d, const double *a, double m, int n) { host_op(B200_FDSP_VECTOR_DMUL_SCALAR, d, a, nullptr, nullptr, m, n); }
void t_vector_fmul_window(float *d, const float *a, const float *b, const float *w, int n) { host_op(B200_FDSP_VECTOR_FMUL_WINDOW, d, a, b, w, 0, n); }
void t_vector_fmul_add(float *d, const float *a, const float *b, const float *c, int n) { host_op(B200_FDSP_VECTOR_FMUL_ADD, d, a, b, c, 0, n); }
void t_vector_fmul_reverse(float *d, const float *a, const float *b, int n) { host_op(B200_FDSP_VECTOR_FMUL_REVERSE, d, a, b, nullptr, 0, n); }
void t_butterflies_float(float *v1, float *v2, int n) { host_op(B200_FDSP_BUTTERFLIES_FLOAT, v1, v2, nullptr, nullptr, 0, n); }
float t_scalarproduct_float(const float *a, const float *b, int n) { return (float)host_op(B200_FDSP_SCALARPRODUCT_FLOAT, nullptr, a, b, nullptr, 0, n); }
void t_vector_dmul(double *d, const double *a, const double *b, int n) { host_op(B200_FDSP_VECTOR_DMUL, d, a, b, nullptr, 0, n); }
double t_scalarproduct_double(const double *a, const double *b, size_t n)
{
    if (n > 0x7fffffff) B200HostCall::fail(kFeature, "length");
    return host_op(B200_FDSP_SCALARPRODUCT_DOUBLE, nullptr, a, b, nullptr, 0, (int)n);
}

} // namespace

B200_API int b200_float_dsp_init(B200FloatDSPContext *c)
{
    if (!c) return B200_EINVAL;
    if (!b200_default_device()) return B200_ENODEV;
    c->vector_fmul = t_vector_fmul; c->vector_fmac_scalar = t_vector_fmac_scalar; c->vector_dmac_scalar = t_vector_dmac_scalar;
    c->vector_fmul_scalar = t_vector_fmul_scalar; c->vector_dmul_scalar = t_vector_dmul_scalar;
    c->vector_fmul_window = t_vector_fmul_window; c->vector_fmul_add = t_vector_fmul_add; c->vector_fmul_reverse = t_vector_fmul_reverse;
    c->butterflies_float = t_butterflies_float; c->scalarproduct_float = t_scalarproduct_float;
    c->vector_dmul = t_vector_dmul; c->scalarproduct_double = t_scalarproduct_double;
    return 0;
}

B200_API int b200_float_dsp_batch_device(B200Device *dev, int op, int64_t nvec, int len, void *dst, int64_t dst_stride,
                                         const void *src0, int64_t src0_stride, const void *src1, int64_t src1_stride,
                                         const void *src2, int64_t src2_stride, double mul)
{
    if (int r = b200_use_device(dev)) return r;
    if (op < 0 || op > B200_FDSP_SCALARPRODUCT_DOUBLE || nvec < 0 || len < 0) return B200_EINVAL;
    if (nvec == 0 || len == 0) return 0;
    if (!dst || !src0 || (uses_src1(op) && !src1) || (uses_src2(op) && !src2)) return B200_EINVAL;
    const uintptr_t am = is_double(op) ? 7 : 3;
    if ((reinterpret_cast<uintptr_t>(dst) | reinterpret_cast<uintptr_t>(src0) | reinterpret_cast<uintptr_t>(src1) |
         reinterpret_cast<uintptr_t>(src2)) & am) return B200_EINVAL;
    Operands o = { dst, src0, src1 ? src1 : src0, src2 ? src2 : src0, dst_stride, src0_stride, src1_stride, src2_stride };
    const int ret = run(dev, dev->stream, op, nvec, len, o, mul);
    if (ret < 0) return ret;
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}
