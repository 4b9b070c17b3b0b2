/* vp9intra_oracle.c — TEST INFRASTRUCTURE ONLY.  A plain-C checker for VP9 intra reconstruction: VP9DSPContext.intra_pred (the
 * predictors of libavcodec/vp9dsp_template.c:33-1106) and b200_vp9_intra_recon_frame_device (intra_recon, vp9recon.c:219-287).
 * It is written in a different form from ffmpeg_b200/csrc/vp9intra.cu: each predictor is its own function that builds the
 * reference's intermediate rows (v[], ve[] / vo[]) and copies them out, and check_intra_mode keeps the reference's table, flags and
 * if-chains (the direct-pointer path, the copy path with its replication) instead of closed forms.  The residual goes through
 * vp9itxfm_oracle.c. */
#include <stdlib.h>
#include <string.h>

#include "vp9intra_oracle.h"
#include "vp9itxfm_oracle.h"

enum { VERT, HOR, DC, DDL, DDR, VR, HD, VL, HU, TM, LDC, TDC, DC128, DC127, DC129, NMODES };

/* ---- the predictors: out[y * n + x], top[-1 ..] and left[] as ints, the reference's orders */
static void p_vert(int n, int *o, const int *l, const int *t, int bd)
{
    for (int y = 0; y < n; y++) for (int x = 0; x < n; x++) o[y * n + x] = t[x];
}
static void p_hor(int n, int *o, const int *l, const int *t, int bd)
{
    for (int y = 0; y < n; y++) for (int x = 0; x < n; x++) o[y * n + x] = l[n - 1 - y];
}
static void p_tm(int n, int *o, const int *l, const int *t, int bd)
{
    const int tl = t[-1], mx = (1 << bd) - 1;
    for (int y = 0; y < n; y++) {
        const int d = l[n - 1 - y] - tl;
        for (int x = 0; x < n; x++) {
            int v = t[x] + d;
            o[y * n + x] = v < 0 ? 0 : v > mx ? mx : v;
        }
    }
}
static void fill(int n, int *o, int v)
{
    for (int k = 0; k < n * n; k++) o[k] = v;
}
static int lg(int n) { return n == 4 ? 2 : n == 8 ? 3 : n == 16 ? 4 : 5; }
static void p_dc(int n, int *o, const int *l, const int *t, int bd)
{
    int s = n;
    for (int k = 0; k < n; k++) s += l[k] + t[k];
    fill(n, o, s >> (lg(n) + 1));
}
static void p_ldc(int n, int *o, const int *l, const int *t, int bd)
{
    int s = n / 2;
    for (int k = 0; k < n; k++) s += l[k];
    fill(n, o, s >> lg(n));
}
static void p_tdc(int n, int *o, const int *l, const int *t, int bd)
{
    int s = n / 2;
    for (int k = 0; k < n; k++) s += t[k];
    fill(n, o, s >> lg(n));
}
static void p_dc128(int n, int *o, const int *l, const int *t, int bd) { fill(n, o, 128 << (bd - 8)); }
static void p_dc127(int n, int *o, const int *l, const int *t, int bd) { fill(n, o, (128 << (bd - 8)) - 1); }
static void p_dc129(int n, int *o, const int *l, const int *t, int bd) { fill(n, o, (128 << (bd - 8)) + 1); }

#define F3(a, b, c) (((a) + (b) * 2 + (c) + 2) >> 2)
#define F2(a, b) (((a) + (b) + 1) >> 1)

static void p_ddl(int n, int *o, const int *l, const int *t, int bd)
{
    if (n == 4) {
        for (int y = 0; y < 4; y++)
            for (int x = 0; x < 4; x++) {
                const int s = x + y;
                o[y * 4 + x] = s == 6 ? t[7] : F3(t[s], t[s + 1], t[s + 2]);
            }
        return;
    }
    int v[31];
    for (int i = 0; i < n - 2; i++) v[i] = F3(t[i], t[i + 1], t[i + 2]);
    v[n - 2] = (t[n - 2] + t[n - 1] * 3 + 2) >> 2;
    for (int j = 0; j < n; j++) {
        for (int i = 0; i < n - 1 - j; i++) o[j * n + i] = v[i + j];
        for (int i = n - 1 - j; i < n; i++) o[j * n + i] = t[n - 1];
    }
}
static void p_ddr(int n, int *o, const int *l, const int *t, int bd)
{
    int v[63];
    for (int i = 0; i < n - 2; i++) {
        v[i] = F3(l[i], l[i + 1], l[i + 2]);
        v[n + 1 + i] = F3(t[i], t[i + 1], t[i + 2]);
    }
    v[n - 2] = F3(l[n - 2], l[n - 1], t[-1]);
    v[n - 1] = F3(l[n - 1], t[-1], t[0]);
    v[n] = F3(t[-1], t[0], t[1]);
    for (int j = 0; j < n; j++) for (int i = 0; i < n; i++) o[j * n + i] = v[n - 1 - j + i];
}
static void p_vr(int n, int *o, const int *l, const int *t, int bd)
{
    int ve[47], vo[47];
    if (n == 4) {                                       /* vert_right_4x4_c's terms, l0 = left[3], l1 = left[2], l2 = left[1] */
        vo[0] = F3(l[3], l[2], l[1]);
        ve[0] = F3(t[-1], l[3], l[2]);
    } else {
        for (int i = 0; i < n / 2 - 2; i++) {
            vo[i] = F3(l[i * 2 + 3], l[i * 2 + 2], l[i * 2 + 1]);
            ve[i] = F3(l[i * 2 + 4], l[i * 2 + 3], l[i * 2 + 2]);
        }
        vo[n / 2 - 2] = F3(l[n - 1], l[n - 2], l[n - 3]);
        ve[n / 2 - 2] = F3(t[-1], l[n - 1], l[n - 2]);
    }
    ve[n / 2 - 1] = F2(t[-1], t[0]);
    vo[n / 2 - 1] = F3(l[n - 1], t[-1], t[0]);
    for (int i = 0; i < n - 1; i++) {
        ve[n / 2 + i] = F2(t[i], t[i + 1]);
        vo[n / 2 + i] = F3(t[i - 1], t[i], t[i + 1]);
    }
    for (int j = 0; j < n / 2; j++)
        for (int i = 0; i < n; i++) {
            o[(2 * j) * n + i] = ve[n / 2 - 1 - j + i];
            o[(2 * j + 1) * n + i] = vo[n / 2 - 1 - j + i];
        }
}
static void p_hd(int n, int *o, const int *l, const int *t, int bd)
{
    int v[94];
    for (int i = 0; i < n - 2; i++) {
        v[i * 2] = F2(l[i + 1], l[i]);
        v[i * 2 + 1] = F3(l[i + 2], l[i + 1], l[i]);
        v[n * 2 + i] = F3(t[i - 1], t[i], t[i + 1]);
    }
    v[n * 2 - 2] = F2(t[-1], l[n - 1]);
    v[n * 2 - 4] = F2(l[n - 1], l[n - 2]);
    v[n * 2 - 1] = F3(t[0], t[-1], l[n - 1]);
    v[n * 2 - 3] = F3(t[-1], l[n - 1], l[n - 2]);
    for (int j = 0; j < n; j++) for (int i = 0; i < n; i++) o[j * n + i] = v[n * 2 - 2 - j * 2 + i];
}
static void p_vl(int n, int *o, const int *l, const int *t, int bd)
{
    if (n == 4) {
        for (int y = 0; y < 4; y++)
            for (int x = 0; x < 4; x++) {
                const int k = (y >> 1) + x;
                o[y * 4 + x] = (y & 1) ? F3(t[k], t[k + 1], t[k + 2]) : F2(t[k], t[k + 1]);
            }
        return;
    }
    int ve[31], vo[31];
    for (int i = 0; i < n - 2; i++) {
        ve[i] = F2(t[i], t[i + 1]);
        vo[i] = F3(t[i], t[i + 1], t[i + 2]);
    }
    ve[n - 2] = F2(t[n - 2], t[n - 1]);
    vo[n - 2] = (t[n - 2] + t[n - 1] * 3 + 2) >> 2;
    for (int j = 0; j < n / 2; j++)
        for (int i = 0; i < n; i++) {
            o[(2 * j) * n + i] = i < n - j - 1 ? ve[j + i] : t[n - 1];
            o[(2 * j + 1) * n + i] = i < n - j - 1 ? vo[j + i] : t[n - 1];
        }
}
static void p_hu(int n, int *o, const int *l, const int *t, int bd)
{
    int v[62];
    for (int i = 0; i < n - 2; i++) {
        v[i * 2] = F2(l[i], l[i + 1]);
        v[i * 2 + 1] = F3(l[i], l[i + 1], l[i + 2]);
    }
    v[n * 2 - 4] = F2(l[n - 2], l[n - 1]);
    v[n * 2 - 3] = (l[n - 2] + l[n - 1] * 3 + 2) >> 2;
    for (int j = 0; j < n; j++)
        for (int i = 0; i < n; i++) o[j * n + i] = j * 2 + i < n * 2 - 2 ? v[j * 2 + i] : l[n - 1];
}

typedef void (*pred_fn)(int n, int *o, const int *l, const int *t, int bd);
static const pred_fn preds[NMODES] = { p_vert, p_hor, p_dc, p_ddl, p_ddr, p_vr, p_hd, p_vl, p_hu, p_tm, p_ldc, p_tdc, p_dc128, p_dc127, p_dc129 };

static int get(const uint8_t *p, int bps) { return bps == 1 ? *p : *(const uint16_t *)p; }
static void put(uint8_t *p, int bps, int v)
{
    if (bps == 1) *p = (uint8_t)v;
    else *(uint16_t *)p = (uint16_t)v;
}

int orc_vp9_intra_pred(int depth, int tx, int mode, uint8_t *dst, ptrdiff_t stride, const uint8_t *left, const uint8_t *top)
{
    if ((depth != 8 && depth != 10 && depth != 12) || tx < 0 || tx > 3 || mode < 0 || mode >= NMODES) return -1;
    const int n = 4 << tx, bps = depth > 8 ? 2 : 1;
    /* only the samples this mode's reference function reads are looked at */
    int tb[41], lb[32], out[1024];
    static const signed char tlo[NMODES] = { 0, 0, 0, 0, -1, -1, -1, 0, 0, -1, 0, 0, 0, 0, 0 };
    int t1 = 0, l0 = 0, l1 = 0;
    memset(tb, 0, sizeof(tb));
    memset(lb, 0, sizeof(lb));
    if (mode == VERT || mode == DC || mode == TDC || mode == DDR || mode == VR || mode == TM) t1 = n;
    if (mode == DDL) t1 = n == 4 ? 8 : n;
    if (mode == VL) t1 = n == 4 ? 7 : n;
    if (mode == HD) t1 = n - 1;
    if (mode == HOR || mode == DC || mode == LDC || mode == DDR || mode == HD || mode == HU || mode == TM) l1 = n;
    if (mode == VR) l0 = 1, l1 = n;
    for (int k = t1 > 0 ? tlo[mode] : 0; k < t1; k++) tb[k + 1] = get(top + (ptrdiff_t)k * bps, bps);
    for (int k = l0; k < l1; k++) lb[k] = get(left + (ptrdiff_t)k * bps, bps);
    preds[mode](n, out, lb, tb + 1, depth);
    for (int y = 0; y < n; y++)
        for (int x = 0; x < n; x++) put(dst + (ptrdiff_t)y * stride + (ptrdiff_t)x * bps, bps, out[y * n + x]);
    return 0;
}

/* ---- check_intra_mode (vp9recon.c:33-217) on a plane read through `src`: the table, the flags and the two paths of the reference */
static const uint8_t mode_conv[10][2][2] = {
    [VERT] = { { DC127, VERT }, { DC127, VERT } },
    [HOR] = { { DC129, DC129 }, { HOR, HOR } },
    [DC] = { { DC128, TDC }, { LDC, DC } },
    [DDL] = { { DC127, DDL }, { DC127, DDL } },
    [DDR] = { { DDR, DDR }, { DDR, DDR } },
    [VR] = { { VR, VR }, { VR, VR } },
    [HD] = { { HD, HD }, { HD, HD } },
    [VL] = { { DC127, VL }, { DC127, VL } },
    [HU] = { { DC129, DC129 }, { HU, HU } },
    [TM] = { { DC129, VERT }, { HOR, TM } },
};
static const struct { uint8_t left, top, topleft, topright, invert; } edges[NMODES] = {
    [VERT] = { 0, 1, 0, 0, 0 }, [HOR] = { 1, 0, 0, 0, 0 }, [DC] = { 1, 1, 0, 0, 0 }, [DDL] = { 0, 1, 0, 1, 0 },
    [DDR] = { 1, 1, 1, 0, 0 }, [VR] = { 1, 1, 1, 0, 0 }, [HD] = { 1, 1, 1, 0, 0 }, [VL] = { 0, 1, 0, 1, 0 },
    [HU] = { 1, 0, 0, 0, 1 }, [TM] = { 1, 1, 1, 0, 0 }, [LDC] = { 1, 0, 0, 0, 0 }, [TDC] = { 0, 1, 0, 0, 0 },
};

typedef struct { const uint8_t *base; ptrdiff_t ls; int bps; } Plane;
static int px(const Plane *p, int y, int x) { return get(p->base + (ptrdiff_t)y * p->ls + (ptrdiff_t)x * p->bps, p->bps); }

/* a = top[-1 ..] (a[-1] valid), l = left[]; returns the converted mode */
static int check_intra_mode(const Plane *src, int mode, int *a, int *l, int x, int y, int W, int H, int have_left, int have_right, int tx,
                            int bpp)
{
    const int have_top = y > 0;
    mode = mode_conv[mode][have_left][have_top];
    if (edges[mode].top) {
        const int n_px_need = 4 << tx, n_px_have = W - x;
        int n_px_need_tr = 0;
        if (tx == 0 && edges[mode].topright && have_right) n_px_need_tr = 4;
        if (have_top && (!edges[mode].topleft || have_left) && (tx != 0 || !edges[mode].topright || have_right) &&
            n_px_need + n_px_need_tr <= n_px_have) {
            /* the reference points a at the row above: expose what the predictor can read there */
            for (int k = 0; k < n_px_need + n_px_need_tr; k++) a[k] = px(src, y - 1, x + k);
            if (edges[mode].topleft) a[-1] = px(src, y - 1, x - 1);
        } else {
            if (have_top) {
                if (n_px_need <= n_px_have) {
                    for (int k = 0; k < n_px_need; k++) a[k] = px(src, y - 1, x + k);
                } else {
                    for (int k = 0; k < n_px_have; k++) a[k] = px(src, y - 1, x + k);
                    for (int k = n_px_have; k < n_px_need; k++) a[k] = a[n_px_have - 1];
                }
            } else {
                for (int k = 0; k < n_px_need; k++) a[k] = (128 << (bpp - 8)) - 1;
            }
            if (edges[mode].topleft) {
                if (have_left && have_top) a[-1] = px(src, y - 1, x - 1);
                else a[-1] = (128 << (bpp - 8)) + (have_top ? +1 : -1);
            }
            if (tx == 0 && edges[mode].topright) {
                if (have_top && have_right && n_px_need + n_px_need_tr <= n_px_have) {
                    for (int k = 4; k < 8; k++) a[k] = px(src, y - 1, x + k);
                } else {
                    for (int k = 4; k < 8; k++) a[k] = a[3];
                }
            }
        }
    }
    if (edges[mode].left) {
        if (have_left) {
            const int n_px_need = 4 << tx, n_px_have = H - y;
            if (edges[mode].invert) {
                if (n_px_need <= n_px_have) {
                    for (int i = 0; i < n_px_need; i++) l[i] = px(src, y + i, x - 1);
                } else {
                    for (int i = 0; i < n_px_have; i++) l[i] = px(src, y + i, x - 1);
                    for (int i = n_px_have; i < n_px_need; i++) l[i] = l[n_px_have - 1];
                }
            } else {
                if (n_px_need <= n_px_have) {
                    for (int i = 0; i < n_px_need; i++) l[n_px_need - 1 - i] = px(src, y + i, x - 1);
                } else {
                    for (int i = 0; i < n_px_have; i++) l[n_px_need - 1 - i] = px(src, y + i, x - 1);
                    for (int i = 0; i < n_px_need - n_px_have; i++) l[i] = l[n_px_need - n_px_have];
                }
            }
        } else {
            for (int i = 0; i < 4 << tx; i++) l[i] = (128 << (bpp - 8)) + 1;
        }
    }
    return mode;
}

/* ff_vp9_intra_txfm_type (vp9data.c) for the ten coded modes */
static const uint8_t intra_txfm_type[10] = { 2, 1, 0, 0, 3, 2, 1, 2, 1, 3 };

int64_t orc_vp9_intra_frame(int depth, int ss_h, int ss_v, int width, int height, uint8_t *const planes[3], ptrdiff_t ls_y, ptrdiff_t ls_uv,
                            int64_t nops, const B200Vp9IntraOp *ops, const void *coef, int order)
{
    if ((depth != 8 && depth != 10 && depth != 12) || ss_h < 0 || ss_h > 1 || ss_v < 0 || ss_v > 1 || width < 1 || height < 1 || nops < 0 ||
        order < 0 || order > 1 || !planes)
        return -1;
    const int bps = depth > 8 ? 2 : 1, cols = (width + 7) >> 3, rows = (height + 7) >> 3;
    const int W[3] = { cols * 8, cols * 8 >> ss_h, cols * 8 >> ss_h }, H[3] = { rows * 8, rows * 8 >> ss_v, rows * 8 >> ss_v };
    const ptrdiff_t ls[3] = { ls_y, ls_uv, ls_uv };
    Plane live[3], before[3];
    uint8_t *copy[3] = { 0, 0, 0 };
    for (int p = 0; p < 3; p++) {
        live[p] = (Plane){ planes[p], ls[p], bps };
        before[p] = live[p];
        if (order == 1) {                                   /* every op reads the planes as they were before the call */
            copy[p] = malloc((size_t)H[p] * (size_t)ls[p]);
            memcpy(copy[p], planes[p], (size_t)(H[p] - 1) * (size_t)ls[p] + (size_t)W[p] * bps);
            before[p].base = copy[p];
        }
    }
    int64_t wrote = 0;
    for (int64_t k = 0; k < nops; k++) {
        const B200Vp9IntraOp *op = &ops[k];
        if (op->plane > 2 || op->tx > 3 || op->mode > 9 || op->x < 0 || op->y < 0 || (op->x & 3) || (op->y & 3) || op->coef_off < 0 ||
            (op->coef_off & 15) || ((op->flags & B200_VP9_INTRA_LOSSLESS) && op->tx != 0))
            continue;
        const int p = op->plane, n = 4 << op->tx;
        if (op->x >= W[p] || op->y >= H[p]) continue;
        int a_buf[1 + 40], l[32], out[1024];
        memset(a_buf, 0, sizeof(a_buf));
        memset(l, 0, sizeof(l));
        const int mode = check_intra_mode(&before[p], op->mode, a_buf + 1, l, op->x, op->y, W[p], H[p], !!(op->flags & B200_VP9_INTRA_HAVE_LEFT),
                                          !!(op->flags & B200_VP9_INTRA_HAVE_RIGHT), op->tx, depth);
        preds[mode](n, out, l, a_buf + 1, depth);
        /* the block in a buffer of its own (the decoder's emulated-edge buffer), the residual on it, and the part inside the plane back */
        uint8_t blk[32 * 32 * 2];
        for (int j = 0; j < n; j++) for (int i = 0; i < n; i++) put(blk + (ptrdiff_t)(j * n + i) * bps, bps, out[j * n + i]);
        if (op->eob) {
            const int lossless = !!(op->flags & B200_VP9_INTRA_LOSSLESS);
            const int txtp = p ? 0 : intra_txfm_type[op->mode];
            const size_t cs = depth > 8 ? 4 : 2;
            void *c = malloc((size_t)n * n * cs);
            memcpy(c, (const uint8_t *)coef + (size_t)op->coef_off * cs, (size_t)n * n * cs);
            orc_vp9_itxfm(depth, lossless ? 4 : op->tx, txtp, blk, (ptrdiff_t)n * bps, c, op->eob);
            free(c);
        }
        for (int j = 0; j < n && op->y + j < H[p]; j++)
            for (int i = 0; i < n && op->x + i < W[p]; i++)
                put(planes[p] + (ptrdiff_t)(op->y + j) * ls[p] + (ptrdiff_t)(op->x + i) * bps, bps, get(blk + (ptrdiff_t)(j * n + i) * bps, bps));
        wrote++;
    }
    for (int p = 0; p < 3; p++) free(copy[p]);
    return wrote;
}
