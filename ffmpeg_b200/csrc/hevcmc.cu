// hevcmc.cu — HEVC inter prediction on sm_90a: the six motion-compensation tables of HEVCDSPContext (libavcodec/hevc/dsp.h:47-125)
// as ff_hevc_dsp_init fills them for 8, 9, 10 and 12 bit samples (hevc/dsp.c:140-196, :230-235), and a batched device entry that
// runs the decoder's per-prediction-unit sequence (hevcdec.c:1722-2040) with edge emulation fused into the sample reads.
//
// Reference semantics reproduced bit for bit (checker: oracle/hevcmc_oracle.c), h26x/h2656_inter_template.c and hevc/dsp_template.c:
//   pixels:  v = src << (14 - depth)
//   h / v:   v = FILTER(src) >> (depth - 8)                     (8 taps at -3..+4 for qpel, 4 taps at -1..+2 for epel)
//   hv:      tmp = FILTER_h(src) >> (depth - 8) stored as int16, v = FILTER_v(tmp) >> 6
//   plain:   dst16 = (int16) v;  uni: clip((v + o) >> (14 - depth));  uni_w: clip(((v wx + o) >> (denom + 14 - depth)) + ox << (depth - 8))
//   bi:      clip((v + src2 + o) >> (15 - depth));  bi_w: clip((v wx1 + src2 wx0 + ((ox << (depth - 8)) + 1) << log2Wd) >> (log2Wd + 1))
// A member filters in the directions its table position names ([!!my][!!mx]), with the phase it is given: phase 0 in a filtered
// direction selects the reference's all-zero dummy row of ff_hevc_?pel_filters.
//
// Kernel: a CTA of 8 warps takes a run of ops (1 to 32, chosen from the batch size so the grid covers the GPU), counts their 16 x 16
// output tiles and deals the (op, tile) list out to its warps, so a 64 x 64 unit is spread over the warps while a run of small chroma
// units shares one CTA.  A warp stages one reference's window for its tile in shared memory through clamped coordinates (edge
// replication), runs the horizontal pass into an int16 shared array (the reference's tmp), the vertical pass in registers; for a
// bi op it keeps reference 0's int16 result in registers while it does the same for reference 1, then clips and stores each output
// sample once.  Lane layout of the vertical pass: a column per lane, the tile's rows split between the lanes of a column.
#include "common.h"
#include <cstring>

namespace {

constexpr int kTile = 16;
constexpr int kWarps = 8;
constexpr int kMaxOpsPerCta = 32;
constexpr int kPitch = 24;                               // int16 per row of the window and of tmp: 16 + 7 samples
constexpr int kRows = kTile + 7;
constexpr int kWarpSmem = 2 * kRows * kPitch;            // int16: window, then horizontal pass
constexpr int kHead = kMaxOpsPerCta + 2;                 // ints in front: each op's first work item, and the total
constexpr size_t kSmem = kHead * sizeof(int) + (size_t)kWarps * kWarpSmem * sizeof(int16_t);
constexpr int kPlain = 4;                                // drop-in put_hevc_?pel: int16 dst, stride in bytes (128 for MAX_PB_SIZE)
constexpr int kMaxPb = 64;

// ff_hevc_qpel_filters / ff_hevc_epel_filters (hevc/dsp.c:83-105; the coefficients of H.265 8.5.3.3.3.1 / .2), plus a last all-zero
// row: the phase a drop-in member is handed for a direction it filters when its caller passes 0
__constant__ int8_t c_qpel[5][8] = { { 0 }, { -1, 4, -10, 58, 17, -5, 1, 0 }, { -1, 4, -11, 40, 40, -11, 4, -1 }, { 0, 1, -5, 17, 58, -10, 4, -1 }, { 0 } };
__constant__ int8_t c_epel[9][4] = { { 0 }, { -2, 58, 10, -2 }, { -4, 54, 16, -2 }, { -6, 46, 28, -4 }, { -4, 36, 36, -4 },
                                     { -4, 28, 46, -6 }, { -2, 16, 54, -4 }, { -2, 10, 58, -2 }, { 0 } };

struct McArgs {
    const B200HevcMcOp *ops;
    long long nops;
    uint8_t *dst;
    long long dst_stride;
    const uint8_t *ref;
    long long ref_stride;
    int pic_w, pic_h, depth, ops_per_cta;
    int max_phase, max_kind;             // batch: 3 / 7 and BI_W; drop-in members: the zero-row phase and kPlain
    const int16_t *src2;                 // drop-in _bi members: the caller's src2 (MAX_PB_SIZE stride) in place of reference 0
};

__host__ __device__ __forceinline__ bool is_bi(int kind) { return kind == B200_HEVC_MC_BI || kind == B200_HEVC_MC_BI_W; }

// the device-side guard: an op it refuses writes nothing
template <typename P>
__device__ __forceinline__ bool op_ok(const B200HevcMcOp &op, const McArgs &a)
{
    const int kind = op.kind;
    if (kind > a.max_kind || op.w < 1 || op.w > kMaxPb || op.h < 1 || op.h > kMaxPb || op.denom > 7) return false;
    if (op.mx[0] > a.max_phase || op.my[0] > a.max_phase) return false;
    if (is_bi(kind) && (op.mx[1] > a.max_phase || op.my[1] > a.max_phase)) return false;
    if (sizeof(P) == 2 && ((op.dst_off | op.ref_off[0] | (is_bi(kind) ? op.ref_off[1] : 0)) & 1)) return false;
    return true;
}

template <typename P, int T>
__global__ void __launch_bounds__(256) hevc_mc_kernel(McArgs a)
{
    extern __shared__ int16_t hevc_smem[];
    int *first = reinterpret_cast<int *>(hevc_smem);                    // [i] = first work item of op i of this CTA, [n] = total
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int16_t *win = hevc_smem + 2 * kHead + warp * kWarpSmem, *tmp = win + kRows * kPitch;
    const long long o0 = (long long)blockIdx.x * a.ops_per_cta;
    const int n = (int)(a.nops - o0 < a.ops_per_cta ? a.nops - o0 : a.ops_per_cta);
    if ((int)threadIdx.x < n) {
        const B200HevcMcOp &op = a.ops[o0 + threadIdx.x];
        first[threadIdx.x + 1] = op_ok<P>(op, a) ? ((op.w + kTile - 1) / kTile) * ((op.h + kTile - 1) / kTile) : 0;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        first[0] = 0;
        for (int i = 1; i <= n; i++) first[i] += first[i - 1];
    }
    __syncthreads();
    const int total = first[n], sh8 = a.depth - 8, maxv = (1 << a.depth) - 1;
    constexpr int B = T == 8 ? 3 : 1;                                   // taps before the sample
    for (int item = warp; item < total; item += kWarps) {
        int i = 0;
        while (first[i + 1] <= item) i++;
        const B200HevcMcOp &op = a.ops[o0 + i];
        const int kind = op.kind, ntx = (op.w + kTile - 1) / kTile, t = item - first[i];
        const int tx = (t % ntx) * kTile, ty = (t / ntx) * kTile;
        const int tw = min(kTile, op.w - tx), th = min(kTile, op.h - ty);
        const int lpc = tw >= 32 ? 1 : 32 / tw, R = (th + lpc - 1) / lpc;   // lanes per column, rows per lane
        const int c = lane % tw, g = lane / tw;
        const int r0 = g < lpc ? g * R : th, r1 = min(th, r0 + R);
        int v0[8];                                                       // reference 0's int16 result of a bi op (R <= 8)
        const int rb = is_bi(kind) && a.src2 ? 1 : 0, re = is_bi(kind) ? 2 : 1;
        for (int r = rb; r < re; r++) {
            const int mx = op.mx[r], my = op.my[r];
            const bool hf = mx != 0, vf = my != 0;
            const int wc = tw + (hf ? T - 1 : 0), wr = th + (vf ? T - 1 : 0);
            const uint8_t *base = a.ref + op.ref_off[r];
            const long long X = (long long)op.x[r] + tx - (hf ? B : 0), Y = (long long)op.y[r] + ty - (vf ? B : 0);
            __syncwarp();                                                // the previous tile's readers are done with win / tmp
            for (int e = lane; e < wc * wr; e += 32) {
                const int wi = e / wc, wj = e - wi * wc;
                long long yy = Y + wi, xx = X + wj;
                yy = yy < 0 ? 0 : yy >= a.pic_h ? a.pic_h - 1 : yy;
                xx = xx < 0 ? 0 : xx >= a.pic_w ? a.pic_w - 1 : xx;
                win[wi * kPitch + wj] = (int16_t)reinterpret_cast<const P *>(base + yy * a.ref_stride)[xx];
            }
            __syncwarp();
            if (hf) {
                int f[T];
#pragma unroll
                for (int k = 0; k < T; k++) f[k] = T == 8 ? c_qpel[mx][k] : c_epel[mx][k];
                for (int e = lane; e < tw * wr; e += 32) {
                    const int wi = e / tw, wj = e - wi * tw;
                    const int16_t *s = win + wi * kPitch + wj;
                    int acc = 0;
#pragma unroll
                    for (int k = 0; k < T; k++) acc += f[k] * s[k];
                    tmp[wi * kPitch + wj] = (int16_t)(acc >> sh8);
                }
                __syncwarp();
            }
            const int16_t *src = hf ? tmp : win;
            int fv[T];
#pragma unroll
            for (int k = 0; k < T; k++) fv[k] = T == 8 ? c_qpel[my][k] : c_epel[my][k];
#pragma unroll
            for (int k8 = 0; k8 < 8; k8++) {                             // static index: v0 stays in registers
                const int y = r0 + k8;
                if (y >= r1) break;
                int v;
                if (vf) {
                    const int16_t *s = src + y * kPitch + c;
                    int acc = 0;
#pragma unroll
                    for (int k = 0; k < T; k++) acc += fv[k] * s[k * kPitch];
                    v = acc >> (hf ? 6 : sh8);
                } else {
                    v = hf ? src[y * kPitch + c] : src[y * kPitch + c] << (14 - a.depth);
                }
                if (r == 0 && re == 2) {                                 // bi: reference 0 is put_hevc_?pel into the int16 tmp
                    v0[k8] = (int16_t)v;
                    continue;
                }
                uint8_t *drow = a.dst + op.dst_off + (long long)(ty + y) * a.dst_stride;
                if (kind == kPlain) {
                    reinterpret_cast<int16_t *>(drow)[tx + c] = (int16_t)v;
                    continue;
                }
                int out;
                if (kind == B200_HEVC_MC_UNI) {
                    out = (v + (1 << (13 - a.depth))) >> (14 - a.depth);
                } else if (kind == B200_HEVC_MC_UNI_W) {
                    const int shift = op.denom + 14 - a.depth;
                    out = ((v * op.wx0 + (1 << (shift - 1))) >> shift) + op.ox * (1 << sh8);
                } else {
                    const int s2 = a.src2 ? a.src2[(ty + y) * kMaxPb + tx + c] : v0[k8];
                    if (kind == B200_HEVC_MC_BI) {
                        out = (v + s2 + (1 << (14 - a.depth))) >> (15 - a.depth);
                    } else {
                        const int log2wd = op.denom + 14 - a.depth;
                        out = (v * op.wx1 + s2 * op.wx0 + (op.ox * (1 << sh8) + 1) * (1 << log2wd)) >> (log2wd + 1);
                    }
                }
                reinterpret_cast<P *>(drow)[tx + c] = (P)min(max(out, 0), maxv);
            }
        }
    }
}

constexpr long long kChunkOps = 1LL << 20;                               // ops per launch

bool depth_ok(int d) { return d == 8 || d == 9 || d == 10 || d == 12; }

cudaError_t launch(McArgs a, int epel, cudaStream_t st)
{
    const long long nops = a.nops;
    long long per = nops / 4096;                                         // ops per CTA: 1 for a CTU row, 32 for a frame of small units
    a.ops_per_cta = (int)(per < 1 ? 1 : per > kMaxOpsPerCta ? kMaxOpsPerCta : per);
    const B200HevcMcOp *ops = a.ops;
    for (long long b = 0; b < nops; b += kChunkOps) {
        a.ops = ops + b;
        a.nops = nops - b < kChunkOps ? nops - b : kChunkOps;
        const unsigned grid = (unsigned)((a.nops + a.ops_per_cta - 1) / a.ops_per_cta);
        if (a.depth == 8) {
            if (epel) hevc_mc_kernel<uint8_t, 4><<<grid, 32 * kWarps, kSmem, st>>>(a);
            else hevc_mc_kernel<uint8_t, 8><<<grid, 32 * kWarps, kSmem, st>>>(a);
        } else {
            if (epel) hevc_mc_kernel<uint16_t, 4><<<grid, 32 * kWarps, kSmem, st>>>(a);
            else hevc_mc_kernel<uint16_t, 8><<<grid, 32 * kWarps, kSmem, st>>>(a);
        }
        B200_LAUNCHED();
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// ---- drop-in members (host pointers).  The samples the reference function reads are copied into a dense device window that is the
// op's whole "picture" (so the clamped reads never clamp), src2 next to it, one op, and the block back.
enum { F_PLAIN, F_UNI, F_UNI_W, F_BI, F_BI_W };

void member_host(int depth, int epel, int form, int vdir, int hdir, uint8_t *dst, ptrdiff_t dststride, const uint8_t *src, ptrdiff_t srcstride,
                 const int16_t *src2, int height, int denom, int wx0, int wx1, int ox, intptr_t mx, intptr_t my, int width)
{
    const int maxp = epel ? 7 : 3, zero = maxp + 1, B = epel ? 1 : 3, A = epel ? 2 : 4, bps = depth > 8 ? 2 : 1;
    const char *feature = "hevc motion compensation";
    if (width < 1 || width > kMaxPb || height < 1 || height > kMaxPb) B200HostCall::fail(feature, "width / height outside 1..64");
    if ((hdir && (mx < 0 || mx > maxp)) || (vdir && (my < 0 || my > maxp))) B200HostCall::fail(feature, "phase outside the filter table");
    if ((form == F_UNI_W || form == F_BI_W) && (denom < 0 || denom > 7)) B200HostCall::fail(feature, "denom outside 0..7");
    const int x0 = hdir ? B : 0, y0 = vdir ? B : 0, wc = width + (hdir ? B + A : 0), wr = height + (vdir ? B + A : 0);
    const size_t wpitch = ((size_t)wc * bps + 15) & ~(size_t)15, wbytes = (wpitch * wr + 255) & ~(size_t)255;
    const size_t s2bytes = (size_t)kMaxPb * kMaxPb * sizeof(int16_t), dpitch = form == F_PLAIN ? kMaxPb * sizeof(int16_t) : wpitch;
    B200HostCall call(feature, nullptr, wbytes + s2bytes + 256 + dpitch * kMaxPb);
    uint8_t *scr = call.scratch;
    cudaStream_t st = call.stream;
    uint8_t *dwin = scr, *ds2 = scr + wbytes, *dop = ds2 + s2bytes, *ddst = dop + 256;
    call.check(b200_h2d_rows(dwin, wpitch, src - y0 * srcstride - x0 * bps, srcstride, (size_t)wc * bps, (size_t)wr, st), "h2d window");
    const bool bi = form == F_BI || form == F_BI_W;
    if (bi)
        call.check(b200_h2d_rows(ds2, kMaxPb * sizeof(int16_t), src2, kMaxPb * sizeof(int16_t), (size_t)width * sizeof(int16_t), (size_t)height, st),
                   "h2d src2");
    B200HevcMcOp op;
    memset(&op, 0, sizeof(op));
    const int r = bi ? 1 : 0;
    op.x[r] = x0;
    op.y[r] = y0;
    op.mx[r] = (uint8_t)(hdir ? (mx ? mx : zero) : 0);
    op.my[r] = (uint8_t)(vdir ? (my ? my : zero) : 0);
    op.w = (uint8_t)width;
    op.h = (uint8_t)height;
    op.kind = (uint8_t)(form == F_PLAIN ? kPlain : form - 1);
    op.denom = (uint8_t)denom;
    op.wx0 = wx0;
    op.wx1 = wx1;
    op.ox = ox;
    call.check(cudaMemcpyAsync(dop, &op, sizeof(op), cudaMemcpyHostToDevice, st), "h2d op");
    McArgs a = { (const B200HevcMcOp *)dop, 1, ddst, (long long)dpitch, dwin, (long long)wpitch, wc, wr, depth, 1, zero, kPlain,
                 bi ? (const int16_t *)ds2 : nullptr };
    call.check(launch(a, epel, st), "launch");
    if (form == F_PLAIN) call.check(b200_d2h_rows(dst, kMaxPb * sizeof(int16_t), ddst, dpitch, (size_t)width * sizeof(int16_t), (size_t)height, st), "d2h");
    else call.check(b200_d2h_rows(dst, dststride, ddst, dpitch, (size_t)width * bps, (size_t)height, st), "d2h");
    call.sync();
}

template <int D, int E, int V, int H>
void m_plain(int16_t *dst, const uint8_t *src, ptrdiff_t srcstride, int height, intptr_t mx, intptr_t my, int width)
{
    member_host(D, E, F_PLAIN, V, H, (uint8_t *)dst, 0, src, srcstride, nullptr, height, 0, 0, 0, 0, mx, my, width);
}
template <int D, int E, int V, int H>
void m_uni(uint8_t *dst, ptrdiff_t dststride, const uint8_t *src, ptrdiff_t srcstride, int height, intptr_t mx, intptr_t my, int width)
{
    member_host(D, E, F_UNI, V, H, dst, dststride, src, srcstride, nullptr, height, 0, 0, 0, 0, mx, my, width);
}
template <int D, int E, int V, int H>
void m_uni_w(uint8_t *dst, ptrdiff_t dststride, const uint8_t *src, ptrdiff_t srcstride, int height, int denom, int wx, int ox, intptr_t mx,
             intptr_t my, int width)
{
    member_host(D, E, F_UNI_W, V, H, dst, dststride, src, srcstride, nullptr, height, denom, wx, 0, ox, mx, my, width);
}
template <int D, int E, int V, int H>
void m_bi(uint8_t *dst, ptrdiff_t dststride, const uint8_t *src, ptrdiff_t srcstride, const int16_t *src2, int height, intptr_t mx, intptr_t my,
          int width)
{
    member_host(D, E, F_BI, V, H, dst, dststride, src, srcstride, src2, height, 0, 0, 0, 0, mx, my, width);
}
template <int D, int E, int V, int H>
void m_bi_w(uint8_t *dst, ptrdiff_t dststride, const uint8_t *src, ptrdiff_t srcstride, const int16_t *src2, int height, int denom, int wx0,
            int wx1, int ox, intptr_t mx, intptr_t my, int width)
{
    member_host(D, E, F_BI_W, V, H, dst, dststride, src, srcstride, src2, height, denom, wx0, wx1, ox, mx, my, width);
}

// hevc/dsp.c:140-196: every width index gets the same function; [idx][!!my][!!mx]
template <int D, int E, int V, int H>
void fill_dir(B200HEVCDSPContext *c)
{
    for (int i = 0; i < 10; i++) {
        (E ? c->put_hevc_epel : c->put_hevc_qpel)[i][V][H] = m_plain<D, E, V, H>;
        (E ? c->put_hevc_epel_uni : c->put_hevc_qpel_uni)[i][V][H] = m_uni<D, E, V, H>;
        (E ? c->put_hevc_epel_uni_w : c->put_hevc_qpel_uni_w)[i][V][H] = m_uni_w<D, E, V, H>;
        (E ? c->put_hevc_epel_bi : c->put_hevc_qpel_bi)[i][V][H] = m_bi<D, E, V, H>;
        (E ? c->put_hevc_epel_bi_w : c->put_hevc_qpel_bi_w)[i][V][H] = m_bi_w<D, E, V, H>;
    }
}
template <int D, int E>
void fill_pel(B200HEVCDSPContext *c)
{
    fill_dir<D, E, 0, 0>(c);
    fill_dir<D, E, 0, 1>(c);
    fill_dir<D, E, 1, 0>(c);
    fill_dir<D, E, 1, 1>(c);
}
template <int D>
void fill(B200HEVCDSPContext *c)
{
    fill_pel<D, 0>(c);
    fill_pel<D, 1>(c);
}

} // namespace

B200_API int b200_hevc_dsp_init(B200HEVCDSPContext *c, int bit_depth)
{
    if (!c) return B200_EINVAL;
    if (!depth_ok(bit_depth)) return B200_ENOSYS;
    if (!b200_default_device()) return B200_ENODEV;
    memset(c, 0, sizeof(*c));                                            // transforms, SAO, deblocking, put_pcm: not built, NULL
    switch (bit_depth) {
    case 8:  fill<8>(c); break;
    case 9:  fill<9>(c); break;
    case 10: fill<10>(c); break;
    default: fill<12>(c); break;
    }
    return 0;
}

B200_API int b200_hevc_mc_batch_device(B200Device *dev, int bit_depth, int epel, int64_t nops, const B200HevcMcOp *ops, uint8_t *dst,
                                       ptrdiff_t dst_stride, const uint8_t *ref, ptrdiff_t ref_stride, int pic_w, int pic_h)
{
    if (nops < 0 || (epel != 0 && epel != 1) || pic_w < 1 || pic_h < 1) {
        b200_set_error("hevc mc batch: negative nops, epel not 0 / 1, or an empty picture");
        return B200_EINVAL;
    }
    if (!depth_ok(bit_depth)) { b200_set_error("hevc mc batch: bit depth %d is not 8, 9, 10 or 12", bit_depth); return B200_EINVAL; }
    const int bps = bit_depth > 8 ? 2 : 1;
    if (dst_stride % bps || ref_stride % bps) { b200_set_error("hevc mc batch: stride not a multiple of the sample size"); return B200_EINVAL; }
    if (nops == 0) return 0;
    if (!ops || !dst || !ref || ((uintptr_t)ops & 7) || ((uintptr_t)dst % bps) || ((uintptr_t)ref % bps)) {
        b200_set_error("hevc mc batch: NULL or misaligned pointer");
        return B200_EINVAL;
    }
    if (int r = b200_use_device(dev)) return r;
    McArgs a = { ops, (long long)nops, dst, (long long)dst_stride, ref, (long long)ref_stride, pic_w, pic_h, bit_depth, 1,
                 epel ? 7 : 3, B200_HEVC_MC_BI_W, nullptr };
    B200_CUDA_OK(launch(a, epel, dev->stream));
    return 0;
}
