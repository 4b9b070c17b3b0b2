// vp9mc.cu — VP9 inter prediction on sm_90a: the mc[5][4][2][2][2] and smc[5][4][2] tables of VP9DSPContext (libavcodec/vp9dsp.h:40-122)
// as ff_vp9dsp_init fills them for 8, 10 and 12 bit samples (vp9dsp_template.c:2302-2361, :2540-2569), and a batched device entry that
// runs the decoder's per-block sequence (vp9_mc_template.c, vp9recon.c:299-551) with edge emulation fused into the sample reads.
//
// Reference semantics reproduced bit for bit (checker: oracle/vp9mc_oracle.c), vp9dsp_template.c:1971-2569:
//   8-tap:    v = clip((sum F[k] * src[-3 + k] + 64) >> 7); in two dimensions the horizontal pass is clipped to samples before the
//             vertical pass filters it (pixel-domain intermediates)
//   bilinear: v = src[0] + ((m * (src[1] - src[0]) + 8) >> 4), which equals ((16 - m) * src[0] + m * src[1] + 8) >> 4 and so the 8-tap
//             form with the row { 0, 0, 0, 128 - 8 m, 8 m, 0, 0, 0 } (the result lies between the two samples: the clip changes nothing).
//             The kernel keeps bilinear as a fourth bank of such rows; the checker keeps the reference's formula, so each checks the other.
//   scaled:   source column of output column x = (mx + x * dx) >> 4, phase (mx + x * dx) & 15 — the closed form of the reference's
//             running imx / ioff loop, which the checker keeps — likewise rows; x counts from the block's origin, not the tile's
//   put: dst = v;  avg: dst = (dst + v + 1) >> 1;  compound = put from slot 0, then avg from slot 1
// Phase 0 is the identity row, so a pass whose phases are all 0 (step 16, start phase 0) is skipped: the 1-D and full-pel entries.
//
// Kernel: the work distribution of hevcmc.cu.  A CTA of 8 warps takes a run of ops (1 to 32, chosen from the batch size so the grid
// covers the GPU), counts their output tiles and deals the (op, tile) list out to its warps.  A warp stages one reference's window for
// its tile in shared memory through clamped coordinates (edge replication), runs the horizontal pass into a second shared array of
// clipped samples (uint8 at 8 bit: half the size of HEVC's int16 intermediates), the vertical pass in registers; for a compound op it
// keeps slot 0's samples in registers while it does the same for slot 1, then stores each output sample once.
// Tile size: 16 output samples per direction, 8 in a direction where a reference of the op steps by more than 16.  The window is then
// at most ((15 * 16 + 15) >> 4) + 8 = ((7 * 32 + 15) >> 4) + 8 + 1 = 23 samples wide and high for every step, so scaled ops need no
// more shared memory than unscaled ones (8.8 KB per CTA at 8 bit, 17.4 KB at 16 bit) instead of the 38 x 38 window a 16 x 16 tile has
// at step 32 (17 / 34 KB per CTA).  ptxas gives both instances 78 registers and no spills, so the register file binds first, at 3 CTAs
// per SM, and either sizing would have the same occupancy; the smaller tiles were chosen because they leave up to 50 KB more of the
// SM's shared-memory / L1 array to the L1 that serves the clamped window gathers, and keep one window size for every op.
// Lane layout: a column per lane in both passes (tile widths 4, 8, 16 divide 32, so a lane's column, and with it its horizontal
// filter row, is fixed for the tile), the tile's rows split between the lanes of a column.
#include "common.h"
#include <cstring>

namespace {

constexpr int kWarps = 8;
constexpr int kMaxOpsPerCta = 32;
constexpr int kWin = 23;                                 // window rows / columns: the tile's source span + 7
constexpr int kPitch = 24;                               // samples per row of the window and of the horizontal pass
constexpr int kWarpSmem = 2 * kWin * kPitch;             // samples: window, then horizontal pass
constexpr int kHead = kMaxOpsPerCta + 2;                 // ints in front: each op's first work item, and the total
constexpr int kMaxRefs = 8;
constexpr int kAvgMember = 2;                            // drop-in avg members: slot 0 is the caller's dst block (McArgs::prev)

template <typename P> constexpr size_t smem_bytes() { return kHead * sizeof(int) + (size_t)kWarps * kWarpSmem * sizeof(P); }

// [bank][phase][tap]: smooth, regular, sharp = ff_vp9_subpel_filters in FilterMode order (vp9dsp.c:32-85; the subpel_filters of the VP9
// bitstream specification), then bilinear as 8-tap rows
__constant__ int16_t c_filters[4][16][8] = {
    {   // smooth
      { 0, 0, 0, 128, 0, 0, 0, 0 }, { -3, -1, 32, 64, 38, 1, -3, 0 }, { -2, -2, 29, 63, 41, 2, -3, 0 }, { -2, -2, 26, 63, 43, 4, -4, 0 },
      { -2, -3, 24, 62, 46, 5, -4, 0 }, { -2, -3, 21, 60, 49, 7, -4, 0 }, { -1, -4, 18, 59, 51, 9, -4, 0 }, { -1, -4, 16, 57, 53, 12, -4, -1 },
      { -1, -4, 14, 55, 55, 14, -4, -1 }, { -1, -4, 12, 53, 57, 16, -4, -1 }, { 0, -4, 9, 51, 59, 18, -4, -1 }, { 0, -4, 7, 49, 60, 21, -3, -2 },
      { 0, -4, 5, 46, 62, 24, -3, -2 }, { 0, -4, 4, 43, 63, 26, -2, -2 }, { 0, -3, 2, 41, 63, 29, -2, -2 }, { 0, -3, 1, 38, 64, 32, -1, -3 },
    },
    {   // regular
      { 0, 0, 0, 128, 0, 0, 0, 0 }, { 0, 1, -5, 126, 8, -3, 1, 0 }, { -1, 3, -10, 122, 18, -6, 2, 0 }, { -1, 4, -13, 118, 27, -9, 3, -1 },
      { -1, 4, -16, 112, 37, -11, 4, -1 }, { -1, 5, -18, 105, 48, -14, 4, -1 }, { -1, 5, -19, 97, 58, -16, 5, -1 }, { -1, 6, -19, 88, 68, -18, 5, -1 },
      { -1, 6, -19, 78, 78, -19, 6, -1 }, { -1, 5, -18, 68, 88, -19, 6, -1 }, { -1, 5, -16, 58, 97, -19, 5, -1 }, { -1, 4, -14, 48, 105, -18, 5, -1 },
      { -1, 4, -11, 37, 112, -16, 4, -1 }, { -1, 3, -9, 27, 118, -13, 4, -1 }, { 0, 2, -6, 18, 122, -10, 3, -1 }, { 0, 1, -3, 8, 126, -5, 1, 0 },
    },
    {   // sharp
      { 0, 0, 0, 128, 0, 0, 0, 0 }, { -1, 3, -7, 127, 8, -3, 1, 0 }, { -2, 5, -13, 125, 17, -6, 3, -1 }, { -3, 7, -17, 121, 27, -10, 5, -2 },
      { -4, 9, -20, 115, 37, -13, 6, -2 }, { -4, 10, -23, 108, 48, -16, 8, -3 }, { -4, 10, -24, 100, 59, -19, 9, -3 }, { -4, 11, -24, 90, 70, -21, 10, -4 },
      { -4, 11, -23, 80, 80, -23, 11, -4 }, { -4, 10, -21, 70, 90, -24, 11, -4 }, { -3, 9, -19, 59, 100, -24, 10, -4 }, { -3, 8, -16, 48, 108, -23, 10, -4 },
      { -2, 6, -13, 37, 115, -20, 9, -4 }, { -2, 5, -10, 27, 121, -17, 7, -3 }, { -1, 3, -6, 17, 125, -13, 5, -2 }, { 0, 1, -3, 8, 127, -7, 3, -1 },
    },
    {   // bilinear
      { 0, 0, 0, 128, 0, 0, 0, 0 }, { 0, 0, 0, 120, 8, 0, 0, 0 }, { 0, 0, 0, 112, 16, 0, 0, 0 }, { 0, 0, 0, 104, 24, 0, 0, 0 },
      { 0, 0, 0, 96, 32, 0, 0, 0 }, { 0, 0, 0, 88, 40, 0, 0, 0 }, { 0, 0, 0, 80, 48, 0, 0, 0 }, { 0, 0, 0, 72, 56, 0, 0, 0 },
      { 0, 0, 0, 64, 64, 0, 0, 0 }, { 0, 0, 0, 56, 72, 0, 0, 0 }, { 0, 0, 0, 48, 80, 0, 0, 0 }, { 0, 0, 0, 40, 88, 0, 0, 0 },
      { 0, 0, 0, 32, 96, 0, 0, 0 }, { 0, 0, 0, 24, 104, 0, 0, 0 }, { 0, 0, 0, 16, 112, 0, 0, 0 }, { 0, 0, 0, 8, 120, 0, 0, 0 },
    },
};

struct McArgs {
    const B200Vp9McOp *ops;
    long long nops;
    uint8_t *dst;
    long long dst_stride;
    int nrefs, depth, ops_per_cta, max_kind;     // max_kind: COMPOUND for the batch entry, kAvgMember for the drop-in members
    const uint8_t *prev;                         // drop-in avg members: the caller's dst block, dense at dst_stride, in place of slot 0
    B200Vp9McRef refs[kMaxRefs];
};

__host__ __device__ __forceinline__ int first_slot(int kind) { return kind == kAvgMember ? 1 : 0; }
__host__ __device__ __forceinline__ int end_slot(int kind) { return kind == B200_VP9_MC_SINGLE ? 1 : 2; }

// the device-side guard: an op it refuses writes nothing
template <typename P>
__device__ __forceinline__ bool op_ok(const B200Vp9McOp &op, const McArgs &a)
{
    const int w = op.w;
    if (op.kind > a.max_kind || op.filter > 3 || (w != 4 && w != 8 && w != 16 && w != 32 && w != 64) || op.h < 1 || op.h > 64) return false;
    for (int r = first_slot(op.kind); r < end_slot(op.kind); r++)
        if (op.ref[r] >= a.nrefs || op.mx[r] > 15 || op.my[r] > 15) return false;
    if (sizeof(P) == 2 && (op.dst_off & 1)) return false;
    return true;
}

// tile size of an op in each direction: 8 where one of its references steps by more than 16 (see the file header), else 16
__device__ __forceinline__ void tile_size(const B200Vp9McOp &op, const McArgs &a, int &tsx, int &tsy)
{
    tsx = tsy = 16;
    for (int r = first_slot(op.kind); r < end_slot(op.kind); r++) {
        if (a.refs[op.ref[r]].dx > 16) tsx = 8;
        if (a.refs[op.ref[r]].dy > 16) tsy = 8;
    }
}

template <typename P>
__global__ void __launch_bounds__(256) vp9_mc_kernel(McArgs a)
{
    extern __shared__ int16_t vp9_smem[];
    int *first = reinterpret_cast<int *>(vp9_smem);                     // [i] = first work item of op i of this CTA, [n] = total
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    P *win = reinterpret_cast<P *>(first + kHead) + warp * kWarpSmem, *tmp = win + kWin * kPitch;
    const long long o0 = (long long)blockIdx.x * a.ops_per_cta;
    const int n = (int)(a.nops - o0 < a.ops_per_cta ? a.nops - o0 : a.ops_per_cta);
    if ((int)threadIdx.x < n) {
        const B200Vp9McOp &op = a.ops[o0 + threadIdx.x];
        int cnt = 0;
        if (op_ok<P>(op, a)) {
            int tsx, tsy;
            tile_size(op, a, tsx, tsy);
            cnt = ((op.w + tsx - 1) / tsx) * ((op.h + tsy - 1) / tsy);
        }
        first[threadIdx.x + 1] = cnt;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        first[0] = 0;
        for (int i = 1; i <= n; i++) first[i] += first[i - 1];
    }
    __syncthreads();
    const int total = first[n], maxv = (1 << a.depth) - 1;
    for (int item = warp; item < total; item += kWarps) {
        int i = 0;
        while (first[i + 1] <= item) i++;
        const B200Vp9McOp &op = a.ops[o0 + i];
        const int kind = op.kind, t = item - first[i];
        int tsx, tsy;
        tile_size(op, a, tsx, tsy);
        const int ntx = (op.w + tsx - 1) / tsx;
        const int tx = (t % ntx) * tsx, ty = (t / ntx) * tsy;
        const int tw = min(tsx, op.w - tx), th = min(tsy, op.h - ty);
        const int lpc = 32 / tw, R = (th + lpc - 1) / lpc;                // lanes per column, rows per lane (<= 8)
        const int c = lane % tw, g = lane / tw;
        const int r0 = g * R < th ? g * R : th, r1 = min(th, r0 + R);
        const int16_t (*bank)[8] = c_filters[op.filter];
        int v0[8];                                                       // slot 0's samples of a compound op
        for (int r = first_slot(kind); r < end_slot(kind); r++) {
            const B200Vp9McRef &ref = a.refs[op.ref[r]];
            const int mx = op.mx[r], my = op.my[r], dx = ref.dx, dy = ref.dy;
            const bool hf = mx != 0 || dx != 16, vf = my != 0 || dy != 16;
            // positions in sixteenths from the block's origin: the tile's first column / row, this lane's column
            const int px0 = mx + tx * dx, py0 = my + ty * dy, pxc = mx + (tx + c) * dx;
            const int cx = (pxc >> 4) - (px0 >> 4);                       // this lane's source column in the window
            const int wc = hf ? ((mx + (tx + tw - 1) * dx) >> 4) - (px0 >> 4) + 8 : tw;
            const int wr = vf ? ((my + (ty + th - 1) * dy) >> 4) - (py0 >> 4) + 8 : th;
            const long long X = (long long)op.x[r] + (px0 >> 4) - (hf ? 3 : 0), Y = (long long)op.y[r] + (py0 >> 4) - (vf ? 3 : 0);
            __syncwarp();                                                // the previous tile's readers are done with win / tmp
            for (int e = lane; e < wc * wr; e += 32) {
                const int wi = e / wc, wj = e - wi * wc;
                long long yy = Y + wi, xx = X + wj;
                yy = yy < 0 ? 0 : yy >= ref.h ? ref.h - 1 : yy;
                xx = xx < 0 ? 0 : xx >= ref.w ? ref.w - 1 : xx;
                win[wi * kPitch + wj] = reinterpret_cast<const P *>(ref.data + yy * (long long)ref.stride)[xx];
            }
            __syncwarp();
            if (hf) {
                int f[8];
#pragma unroll
                for (int k = 0; k < 8; k++) f[k] = bank[pxc & 15][k];
                for (int wi = g; wi < wr; wi += lpc) {
                    const P *s = win + wi * kPitch + cx;
                    int acc = 64;
#pragma unroll
                    for (int k = 0; k < 8; k++) acc += f[k] * s[k];
                    tmp[wi * kPitch + c] = (P)min(max(acc >> 7, 0), maxv);
                }
                __syncwarp();
            }
            const P *src = hf ? tmp + c : win + cx;
#pragma unroll
            for (int k8 = 0; k8 < 8; k8++) {                             // static index: v0 stays in registers
                const int y = r0 + k8;
                if (y >= r1) break;
                int v;
                if (vf) {
                    const int py = my + (ty + y) * dy;
                    const int16_t *fv = bank[py & 15];
                    const P *s = src + ((py >> 4) - (py0 >> 4)) * kPitch;
                    int acc = 64;
#pragma unroll
                    for (int k = 0; k < 8; k++) acc += fv[k] * s[k * kPitch];
                    v = min(max(acc >> 7, 0), maxv);
                } else {
                    v = src[y * kPitch];
                }
                if (r == 0 && kind == B200_VP9_MC_COMPOUND) {
                    v0[k8] = v;
                    continue;
                }
                const long long row = op.dst_off + (long long)(ty + y) * a.dst_stride;
                if (kind == B200_VP9_MC_COMPOUND) v = (v0[k8] + v + 1) >> 1;
                else if (kind == kAvgMember) v = (reinterpret_cast<const P *>(a.prev + row)[tx + c] + v + 1) >> 1;
                reinterpret_cast<P *>(a.dst + row)[tx + c] = (P)v;
            }
        }
    }
}

constexpr long long kChunkOps = 1LL << 20;                               // ops per launch

bool depth_ok(int d) { return d == 8 || d == 10 || d == 12; }

cudaError_t launch(McArgs a, cudaStream_t st)
{
    const long long nops = a.nops;
    long long per = nops / 4096;                                         // ops per CTA: 1 for a superblock row, 32 for a frame of small blocks
    a.ops_per_cta = (int)(per < 1 ? 1 : per > kMaxOpsPerCta ? kMaxOpsPerCta : per);
    const B200Vp9McOp *ops = a.ops;
    for (long long b = 0; b < nops; b += kChunkOps) {
        a.ops = ops + b;
        a.nops = nops - b < kChunkOps ? nops - b : kChunkOps;
        const unsigned grid = (unsigned)((a.nops + a.ops_per_cta - 1) / a.ops_per_cta);
        if (a.depth == 8) vp9_mc_kernel<uint8_t><<<grid, 32 * kWarps, smem_bytes<uint8_t>(), st>>>(a);
        else vp9_mc_kernel<uint16_t><<<grid, 32 * kWarps, smem_bytes<uint16_t>(), st>>>(a);
        B200_LAUNCHED();
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// ---- drop-in members (host pointers).  The samples the reference function reads are copied into a dense device window that is the
// op's whole reference plane (for an 8-tap bank the clamped reads never clamp; for bilinear they clamp only under zero taps), the
// caller's dst block next to it for an avg member, one op, and the block back.
void member_host(int depth, int w, int bank, int avg, bool hdir, bool vdir, uint8_t *dst, ptrdiff_t dststride, const uint8_t *src,
                 ptrdiff_t srcstride, int h, int mx, int my, int dx, int dy)
{
    if (h < 1 || h > 64 || mx < 0 || mx > 15 || my < 0 || my > 15 || dx < 1 || dx > 32 || dy < 1 || dy > 32) {
        b200_set_error("vp9 mc member: h %d, phase (%d, %d) or step (%d, %d) outside 1..64, 0..15, 1..32", h, mx, my, dx, dy);
        return;
    }
    const int bps = depth > 8 ? 2 : 1, before = bank == 3 ? 0 : 3, span = bank == 3 ? 2 : 8;
    if (!hdir) mx = 0;
    if (!vdir) my = 0;
    const int x0 = hdir ? before : 0, y0 = vdir ? before : 0;
    const int wc = hdir ? (((w - 1) * dx + mx) >> 4) + span : w, wr = vdir ? (((h - 1) * dy + my) >> 4) + span : h;
    const size_t wpitch = ((size_t)wc * bps + 15) & ~(size_t)15, wbytes = (wpitch * wr + 255) & ~(size_t)255;
    const size_t dpitch = (size_t)64 * bps;
    B200HostCall call("vp9 motion compensation", nullptr, wbytes + 256 + dpitch * 64);
    uint8_t *scr = call.scratch;
    cudaStream_t st = call.stream;
    uint8_t *dwin = scr, *dop = scr + wbytes, *ddst = dop + 256;
    call.check(b200_h2d_rows(dwin, wpitch, src - y0 * srcstride - x0 * bps, srcstride, (size_t)wc * bps, (size_t)wr, st), "h2d window");
    if (avg) call.check(b200_h2d_rows(ddst, dpitch, dst, dststride, (size_t)w * bps, (size_t)h, st), "h2d dst");
    B200Vp9McOp op;
    memset(&op, 0, sizeof(op));
    const int r = avg ? 1 : 0;
    op.x[r] = x0;
    op.y[r] = y0;
    op.mx[r] = (uint8_t)mx;
    op.my[r] = (uint8_t)my;
    op.w = (uint8_t)w;
    op.h = (uint8_t)h;
    op.filter = (uint8_t)bank;
    op.kind = (uint8_t)(avg ? kAvgMember : B200_VP9_MC_SINGLE);
    call.check(cudaMemcpyAsync(dop, &op, sizeof(op), cudaMemcpyHostToDevice, st), "h2d op");
    McArgs a;
    memset(&a, 0, sizeof(a));
    a.ops = (const B200Vp9McOp *)dop;
    a.nops = 1;
    a.dst = ddst;
    a.dst_stride = (long long)dpitch;
    a.nrefs = 1;
    a.depth = depth;
    a.max_kind = kAvgMember;
    a.prev = ddst;
    a.refs[0].data = dwin;
    a.refs[0].stride = (ptrdiff_t)wpitch;
    a.refs[0].w = wc;
    a.refs[0].h = wr;
    a.refs[0].dx = dx;
    a.refs[0].dy = dy;
    call.check(launch(a, st), "launch");
    call.check(b200_d2h_rows(dst, dststride, ddst, dpitch, (size_t)w * bps, (size_t)h, st), "d2h");
    call.sync();
}

template <int D, int W, int F, int A, int H, int V>
void m_mc(uint8_t *dst, ptrdiff_t dst_stride, const uint8_t *ref, ptrdiff_t ref_stride, int h, int mx, int my)
{
    member_host(D, W, F, A, H, V, dst, dst_stride, ref, ref_stride, h, mx, my, 16, 16);
}
template <int D, int W, int F, int A>
void m_smc(uint8_t *dst, ptrdiff_t dst_stride, const uint8_t *ref, ptrdiff_t ref_stride, int h, int mx, int my, int dx, int dy)
{
    member_host(D, W, F, A, true, true, dst, dst_stride, ref, ref_stride, h, mx, my, dx, dy);
}

// vp9dsp_template.c:2308-2322: one full-pel function per size and put / avg, whatever the bank (installed as bank 0's)
template <int D, int I, int F, int A>
void fill_entry(B200VP9DSPContext *c)
{
    constexpr int W = 64 >> I;
    c->mc[I][F][A][0][0] = m_mc<D, W, 0, A, 0, 0>;
    c->mc[I][F][A][1][0] = m_mc<D, W, F, A, 1, 0>;
    c->mc[I][F][A][0][1] = m_mc<D, W, F, A, 0, 1>;
    c->mc[I][F][A][1][1] = m_mc<D, W, F, A, 1, 1>;
    c->smc[I][F][A] = m_smc<D, W, F, A>;
}
template <int D, int I>
void fill_size(B200VP9DSPContext *c)
{
    fill_entry<D, I, 0, 0>(c); fill_entry<D, I, 0, 1>(c);
    fill_entry<D, I, 1, 0>(c); fill_entry<D, I, 1, 1>(c);
    fill_entry<D, I, 2, 0>(c); fill_entry<D, I, 2, 1>(c);
    fill_entry<D, I, 3, 0>(c); fill_entry<D, I, 3, 1>(c);
}
template <int D>
void fill(B200VP9DSPContext *c)
{
    fill_size<D, 0>(c); fill_size<D, 1>(c); fill_size<D, 2>(c); fill_size<D, 3>(c); fill_size<D, 4>(c);
}

} // namespace

B200_API int b200_vp9_dsp_init(B200VP9DSPContext *c, int bit_depth)
{
    if (!c) return B200_EINVAL;
    if (!depth_ok(bit_depth)) return B200_ENOSYS;
    if (!b200_default_device()) return B200_ENODEV;
    memset(c, 0, sizeof(*c));                                            // intra_pred, itxfm_add, loop_filter_*: not built, NULL
    switch (bit_depth) {
    case 8:  fill<8>(c); break;
    case 10: fill<10>(c); break;
    default: fill<12>(c); break;
    }
    return 0;
}

B200_API int b200_vp9_mc_batch_device(B200Device *dev, int bit_depth, int nrefs, const B200Vp9McRef *refs, int64_t nops, const B200Vp9McOp *ops,
                                      uint8_t *dst, ptrdiff_t dst_stride)
{
    if (nops < 0 || nrefs < 1 || nrefs > kMaxRefs) { b200_set_error("vp9 mc batch: negative nops or nrefs outside 1..8"); return B200_EINVAL; }
    if (!depth_ok(bit_depth)) { b200_set_error("vp9 mc batch: bit depth %d is not 8, 10 or 12", bit_depth); return B200_EINVAL; }
    const int bps = bit_depth > 8 ? 2 : 1;
    if (dst_stride % bps) { b200_set_error("vp9 mc batch: stride not a multiple of the sample size"); return B200_EINVAL; }
    if (nops == 0) return 0;
    if (!refs || !ops || !dst || ((uintptr_t)ops & 7) || ((uintptr_t)dst % bps)) {
        b200_set_error("vp9 mc batch: NULL or misaligned pointer");
        return B200_EINVAL;
    }
    McArgs a;
    memset(&a, 0, sizeof(a));
    for (int r = 0; r < nrefs; r++) {
        const B200Vp9McRef &f = refs[r];
        if (!f.data || ((uintptr_t)f.data % bps) || f.stride % bps || f.w < 1 || f.h < 1 || f.dx < 1 || f.dx > 32 || f.dy < 1 || f.dy > 32) {
            b200_set_error("vp9 mc batch: reference %d has a NULL or misaligned plane, an empty size or a step outside 1..32", r);
            return B200_EINVAL;
        }
        a.refs[r] = f;
    }
    if (int r = b200_use_device(dev)) return r;
    a.ops = ops;
    a.nops = (long long)nops;
    a.dst = dst;
    a.dst_stride = (long long)dst_stride;
    a.nrefs = nrefs;
    a.depth = bit_depth;
    a.max_kind = B200_VP9_MC_COMPOUND;
    B200_CUDA_OK(launch(a, dev->stream));
    return 0;
}
