/*
 * h264pred_oracle.c — TEST INFRASTRUCTURE ONLY.  CPU restatement of libavcodec's H.264 intra prediction: the members of H264PredContext
 * (libavcodec/h264pred.h:94-114) as ff_h264_pred_init(h, AV_CODEC_ID_H264, depth, chroma_format_idc) installs them for depth 8, 9, 10,
 * 12 and 14 (libavcodec/h264pred.c:437-539).
 *
 * Follows (behaviour, not text) libavcodec/h264pred_template.c:
 *   :34-301    pred4x4: V, H, DC, the six diagonal modes (written here in the standard's closed forms, ITU-T H.264 8.3.1.2), LEFT_DC, TOP_DC,
 *              DC_128 = 1 << (depth - 1); DIAG_DOWN_LEFT and VERT_LEFT read four more top samples from `topright`
 *   :303-461   pred16x16: V, H, DC, PLANE (H, V = (5 x + 32) >> 6, clipped to the depth), LEFT_DC, TOP_DC, DC_128
 *   :463-744   pred8x8 / pred8x16 (chroma_format_idc <= 1 / above): the DC family per 4x4 quadrant, and the mad_cow compositions
 *              l0t, 0lt, l00, 0l0 (a DC form followed by a 4x4 DC form on one or two quadrants)
 *   :746-820   pred8x8 / pred8x16 PLANE
 *   :822-1101  pred8x8l: the [1 2 1] edge filter with has_topleft / has_topright substitution, then the 8x8 forms of the nine modes
 *   :1103-1330 the lossless add forms: running sums down a column / along a row in the sample type (wrapping modulo 2^8 or 2^16,
 *              no clip), coefficients cleared (int16 at 8 bit, int32 above); pred8x8_add / pred16x16_add apply the 4x4 form per
 *              block_offset entry in table order, the 8x16 forms take entries 0-3 and 8-11, coefficient sub-block i at 16 i.
 * table: 0 pred4x4, 1 pred8x8l, 2 pred8x8, 3 pred16x16, 4 pred4x4_add, 5 pred8x8l_add, 6 pred8x8l_filter_add, 7 pred8x8_add,
 * 8 pred16x16_add; mode = index into that table.  flags bit 0 = has_topleft, bit 1 = has_topright (pred8x8l, pred8x8l_filter_add).
 * stride in bytes.  Returns -1 where the reference leaves the member NULL.
 */
#include <string.h>
#include "oracle.h"

typedef struct { uint8_t *p; ptrdiff_t st; int hbd; } Pic;             /* st in samples */

static int px(const Pic *c, int x, int y) { return c->hbd ? ((uint16_t *)c->p)[x + y * c->st] : c->p[x + y * c->st]; }
static void put(const Pic *c, int x, int y, int v) { if (c->hbd) ((uint16_t *)c->p)[x + y * c->st] = (uint16_t)v; else c->p[x + y * c->st] = (uint8_t)v; }
static int a3(int a, int b, int c) { return (a + 2 * b + c + 2) >> 2; }
static int a2(int a, int b) { return (a + b + 1) >> 1; }

/* the nine directional modes on an N x N block from the edge e[]: e[N2 + i] = top sample i (i = -1 .. 2N-1), e[N2 - 2 - j] = left sample j
 * (j = 0 .. N-1), so that e[N2 - 1] is the corner and the edge runs from the bottom-left up and along the top */
#define N2 18
static int directional(int mode, int N, int x, int y, const int *e)
{
    const int *T = e + N2, *L0 = e + N2 - 2;                           /* T[i]; left j = L0[-j] */
#define LFT(j) ((j) < 0 ? T[-1] : L0[-(j)])
    switch (mode) {
    case 0: return T[x];
    case 1: return LFT(y);
    case 3: return x == N - 1 && y == N - 1 ? (T[2 * N - 2] + 3 * T[2 * N - 1] + 2) >> 2 : a3(T[x + y], T[x + y + 1], T[x + y + 2]);
    case 4:
        if (x > y) return a3(T[x - y - 2], T[x - y - 1], T[x - y]);
        if (x < y) return a3(LFT(y - x - 2), LFT(y - x - 1), LFT(y - x));
        return a3(T[0], T[-1], LFT(0));
    case 5: {
        const int z = 2 * x - y, i = x - (y >> 1);
        if (z >= 0 && !(z & 1)) return a2(T[i - 1], T[i]);
        if (z >= 0) return a3(T[i - 2], T[i - 1], T[i]);
        if (z == -1) return a3(LFT(0), T[-1], T[0]);
        return a3(LFT(y - 2 * x - 1), LFT(y - 2 * x - 2), LFT(y - 2 * x - 3));
    }
    case 6: {
        const int z = 2 * y - x, i = y - (x >> 1);
        if (z >= 0 && !(z & 1)) return a2(LFT(i - 1), LFT(i));
        if (z >= 0) return a3(LFT(i - 2), LFT(i - 1), LFT(i));
        if (z == -1) return a3(LFT(0), T[-1], T[0]);
        return a3(T[x - 2 * y - 1], T[x - 2 * y - 2], T[x - 2 * y - 3]);
    }
    case 7: {
        const int i = x + (y >> 1);
        return y & 1 ? a3(T[i], T[i + 1], T[i + 2]) : a2(T[i], T[i + 1]);
    }
    case 8: {
        const int z = x + 2 * y, i = y + (x >> 1);
        if (z > 2 * N - 3) return LFT(N - 1);
        if (z == 2 * N - 3) return (LFT(N - 2) + 3 * LFT(N - 1) + 2) >> 2;
        return z & 1 ? a3(LFT(i), LFT(i + 1), LFT(i + 2)) : a2(LFT(i), LFT(i + 1));
    }
    }
#undef LFT
    return 0;
}

static int dc_of(int mode, int N, const int *e, int mid)
{
    const int *T = e + N2, *L0 = e + N2 - 2;
    int st = 0, sl = 0, sh = N == 4 ? 2 : 3;
    for (int i = 0; i < N; i++) { st += T[i]; sl += L0[-i]; }
    if (mode == 2) return (st + sl + N) >> (sh + 1);
    if (mode == 9) return (sl + N / 2) >> sh;
    if (mode == 10) return (st + N / 2) >> sh;
    return mid;
}

/* pred4x4 (template :34-301) */
static void pred4x4(const Pic *c, int mode, const uint8_t *topright, int mid)
{
    int e[2 * N2 + 16] = { 0 };
    const int needs_tr = mode == 3 || mode == 7;
    const int needs_top = mode == 0 || mode == 2 || (mode >= 3 && mode <= 7) || mode == 10;
    const int needs_left = mode == 1 || mode == 2 || (mode >= 4 && mode <= 6) || mode == 8 || mode == 9;
    if (needs_top) for (int i = 0; i < 4; i++) e[N2 + i] = px(c, i, -1);
    if (needs_tr) for (int i = 0; i < 4; i++) e[N2 + 4 + i] = c->hbd ? ((const uint16_t *)topright)[i] : topright[i];
    if (needs_left) for (int j = 0; j < 4; j++) e[N2 - 2 - j] = px(c, -1, j);
    if (mode >= 4 && mode <= 6) e[N2 - 1] = px(c, -1, -1);
    for (int y = 0; y < 4; y++)
        for (int x = 0; x < 4; x++)
            put(c, x, y, (mode <= 8 && mode != 2) ? directional(mode, 4, x, y, e) : dc_of(mode, 4, e, mid));
}

/* PREDICT_8x8_LOAD_* (template :822-851): the filtered edge into e[] in directional()'s layout */
static void edge8x8(const Pic *c, int mode, int tl, int tr, int *e)
{
    const int top = mode == 0 || mode == 2 || (mode >= 3 && mode <= 7) || mode == 10;
    const int left = mode == 1 || mode == 2 || (mode >= 4 && mode <= 6) || mode == 8 || mode == 9;
    int *T = e + N2, *L0 = e + N2 - 2;
    if (top) {
        int r[17];
        for (int i = 0; i < 8; i++) r[i + 1] = px(c, i, -1);
        r[0] = tl ? px(c, -1, -1) : r[1];
        r[9] = tr ? px(c, 8, -1) : r[8];
        for (int i = 0; i < 8; i++) T[i] = a3(r[i], r[i + 1], r[i + 2]);
        if (mode == 3 || mode == 7) {                                   /* top-right: filtered, or eight copies of SRC(7, -1) */
            if (tr) {
                int q[9];
                for (int i = 0; i < 9; i++) q[i] = px(c, 7 + i, -1);
                for (int i = 8; i < 15; i++) T[i] = a3(q[i - 8], q[i - 7], q[i - 6]);
                T[15] = (q[7] + 3 * q[8] + 2) >> 2;
            } else
                for (int i = 8; i < 16; i++) T[i] = px(c, 7, -1);
        }
    }
    if (left) {
        int r[10];
        for (int j = 0; j < 8; j++) r[j + 1] = px(c, -1, j);
        r[0] = tl ? px(c, -1, -1) : r[1];
        r[9] = r[8];
        for (int j = 0; j < 8; j++) L0[-j] = a3(r[j], r[j + 1], r[j + 2]);
    }
    if (mode >= 4 && mode <= 6) T[-1] = a3(px(c, -1, 0), px(c, -1, -1), px(c, 0, -1));
}

static void pred8x8l(const Pic *c, int mode, int tl, int tr, int mid)
{
    int e[2 * N2 + 16] = { 0 };
    edge8x8(c, mode, tl, tr, e);
    for (int y = 0; y < 8; y++)
        for (int x = 0; x < 8; x++)
            put(c, x, y, (mode <= 8 && mode != 2) ? directional(mode, 8, x, y, e) : dc_of(mode, 8, e, mid));
}

static int clipd(int v, int maxv) { return v < 0 ? 0 : v > maxv ? maxv : v; }

/* pred8x8 (rows = 8) / pred8x16 (rows = 16) and pred16x16 (w = 16): template :303-820 */
static void pred_block(const Pic *c, int w, int rows, int mode, int mid, int maxv)
{
    int T[17], L[17];                                                    /* T[0] / L[0] = corner, T[1 + i], L[1 + j] */
    const int top = mode == 0 || mode == 2 || mode == 3 || mode == 5 || mode == 7 || mode == 8;
    const int left = mode == 0 || mode == 1 || mode == 3 || mode == 4 || mode >= 7;
    for (int i = 0; i < w; i++) T[1 + i] = top ? px(c, i, -1) : 0;
    for (int j = 0; j < rows; j++) L[1 + j] = left ? px(c, -1, j) : 0;
    T[0] = L[0] = mode == 3 ? px(c, -1, -1) : 0;
    if (mode == 3) {
        int H = 0, V = 0, a;
        const int hw = w / 2, hr = rows / 2;
        for (int k = 1; k <= hw; k++) H += k * (T[hw + k] - T[hw - k]);
        for (int k = 1; k <= hr; k++) V += k * (L[hr + k] - L[hr - k]);
        H = w == 16 ? (5 * H + 32) >> 6 : (17 * H + 16) >> 5;
        V = rows == 16 ? (5 * V + 32) >> 6 : (17 * V + 16) >> 5;
        a = 16 * (L[rows] + T[w] + 1) - (hr - 1) * V - (hw - 1) * H;
        for (int y = 0; y < rows; y++)
            for (int x = 0; x < w; x++) put(c, x, y, clipd((a + y * V + x * H) >> 5, maxv));
        return;
    }
    if (w == 16) {
        int st = 0, sl = 0;
        for (int i = 1; i <= 16; i++) { st += T[i]; sl += L[i]; }
        for (int y = 0; y < 16; y++)
            for (int x = 0; x < 16; x++)
                put(c, x, y, mode == 0 ? (st + sl + 16) >> 5 : mode == 1 ? L[1 + y] : mode == 2 ? T[1 + x] : mode == 4 ? (sl + 8) >> 4
                           : mode == 5 ? (st + 8) >> 4 : mid);
        return;
    }
    const int s0 = T[1] + T[2] + T[3] + T[4], s1 = T[5] + T[6] + T[7] + T[8];
    for (int y = 0; y < rows; y++) {
        const int q = y / 4, sq = L[1 + 4 * q] + L[2 + 4 * q] + L[3 + 4 * q] + L[4 + 4 * q];
        for (int x = 0; x < 8; x++) {
            int v;
            switch (mode) {
            case 1: v = L[1 + y]; break;
            case 2: v = T[1 + x]; break;
            case 4: case 9: case 10: v = (sq + 2) >> 2; break;
            case 5: case 7: v = x < 4 ? (s0 + 2) >> 2 : (s1 + 2) >> 2; break;
            case 6: v = mid; break;
            default:                                                     /* 0 and 8: pred8x8_dc / pred8x16_dc */
                if (q == 0) v = x < 4 ? (s0 + sq + 4) >> 3 : (s1 + 2) >> 2;
                else v = x < 4 ? (sq + 2) >> 2 : (s1 + sq + 4) >> 3;
            }
            if (mode == 7 && x < 4 && y < 4) v = (s0 + L[1] + L[2] + L[3] + L[4] + 4) >> 3;   /* l0t: then pred4x4_dc */
            if (mode == 8 && x < 4 && y < 4) v = (s0 + 2) >> 2;                                /* 0lt: then pred4x4_top_dc */
            if (mode == 9 && y >= 4 && y < 8) v = mid;                                          /* l00: then DC_128 on rows 4-7 */
            if (mode == 10 && y < 4) v = mid;                                                   /* 0l0: then DC_128 on rows 0-3 */
            put(c, x, y, v);
        }
    }
}

static int coef_get(const void *b, int hbd, int i) { return hbd ? ((const int32_t *)b)[i] : ((const int16_t *)b)[i]; }
static void coef_clear(void *b, int hbd, int n) { memset(b, 0, (size_t)n * (hbd ? 4 : 2)); }

/* the running sums of the lossless forms on an N x N block at (0, 0) of c with coefficients b (row-major N x N); start[] = the value
 * each column (vertical) / row (horizontal) starts from */
static void add_runs(const Pic *c, int N, int vert, const int *start, const void *b, int hbd)
{
    const unsigned mask = hbd ? 0xFFFFu : 0xFFu;
    for (int i = 0; i < N; i++) {
        unsigned v = (unsigned)start[i];
        for (int k = 0; k < N; k++) {
            const int x = vert ? i : k, y = vert ? k : i;
            v = (v + (unsigned)coef_get(b, hbd, y * N + x)) & mask;
            put(c, x, y, (int)v);
        }
    }
}

static void add4x4(const Pic *c, int vert, void *b, int hbd)
{
    int s[4];
    for (int i = 0; i < 4; i++) s[i] = vert ? px(c, i, -1) : px(c, -1, i);
    add_runs(c, 4, vert, s, b, hbd);
    coef_clear(b, hbd, 16);
}

int orc_h264_pred(int depth, int idc, int table, int mode, uint8_t *pix, const uint8_t *topright, int flags, void *block,
                  const int *block_offset, ptrdiff_t stride)
{
    if (depth != 8 && depth != 9 && depth != 10 && depth != 12 && depth != 14) return -1;
    const int hbd = depth > 8, mid = 1 << (depth - 1), maxv = (1 << depth) - 1, tl = flags & 1, tr = (flags >> 1) & 1;
    const Pic c = { pix, stride >> hbd, hbd };
    switch (table) {
    case 0: if (mode > 11) return -1; pred4x4(&c, mode, topright, mid); return 0;
    case 1: if (mode > 11) return -1; pred8x8l(&c, mode, tl, tr, mid); return 0;
    case 2: if (mode > 10) return -1; pred_block(&c, 8, idc <= 1 ? 8 : 16, mode, mid, maxv); return 0;
    case 3: if (mode > 6) return -1; pred_block(&c, 16, 16, mode, mid, maxv); return 0;
    case 4: if (mode > 1) return -1; add4x4(&c, mode == 0, block, hbd); return 0;
    case 5: case 6: {
        if (mode > 1) return -1;
        int s[8], e[2 * N2 + 16] = { 0 };
        const int vert = mode == 0;
        if (table == 6) {                                                /* pred8x8l_*_filter_add: from the filtered edge */
            edge8x8(&c, vert ? 0 : 1, tl, tr, e);
            for (int i = 0; i < 8; i++) s[i] = vert ? e[N2 + i] : e[N2 - 2 - i];
        } else
            for (int i = 0; i < 8; i++) s[i] = vert ? px(&c, i, -1) : px(&c, -1, i);
        add_runs(&c, 8, vert, s, block, hbd);
        coef_clear(block, hbd, 64);
        return 0;
    }
    case 7: case 8: {
        if (mode != 1 && mode != 2) return -1;
        const int n = table == 8 ? 16 : idc <= 1 ? 4 : 8;
        for (int i = 0; i < n; i++) {
            const Pic s = { pix + block_offset[table == 7 && i >= 4 ? i + 4 : i], c.st, hbd };
            add4x4(&s, mode == 2, (uint8_t *)block + (size_t)i * 16 * (hbd ? 4 : 2), hbd);
        }
        return 0;
    }
    }
    return -1;
}
