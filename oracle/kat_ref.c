/*
 * kat_ref.c — TEST INFRASTRUCTURE: pins oracle/hevc_oracle.c against the UNMODIFIED reference.
 *
 * Links oracle/_ref/libohevc_ref.so (the reference's own C tables, built by build_ref.sh from
 * /root/reference) and calls every HEVCDSPContext / HEVCPredContext slot of SURVEY.md §8(a)
 * on seeded random inputs, comparing with the restatement bit for bit.
 * Compiled against the reference headers where they lie (-I/root/reference); never shipped.
 *
 * usage: kat_ref [trials]     exit code 0 = every comparison identical
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <stdint.h>
#include "libavcodec/hevc.h"
#include "libavcodec/hevcdsp.h"
#include "libavcodec/hevcpred.h"
#include "libavcodec/videodsp.h"
#include "../include/b200hevc_worklist.h"

/* oracle entry points */
void orc_idct(int16_t *c, int log2, int col_limit, int bd);
void orc_idct_dc(int16_t *c, int log2, int bd);
void orc_dst4(int16_t *c, int bd);
void orc_transform_skip(int16_t *c, int log2, int bd);
void orc_rdpcm(int16_t *c, int log2, int vertical);
void orc_add_residual(uint16_t *dst, int stride, const int16_t *r, int n, int bd);
void orc_mc_rec(const B200McRec *m, uint16_t *dst, int dst_stride, const uint16_t *ref0, const uint16_t *ref1, int pw, int ph, int bd);
void orc_intra_rec(const B200IntraRec *r, uint16_t *plane, int stride, int bd);
void orc_deblock_luma_seg(uint16_t *pix, int xs, int ys, int beta8, int tc8, int no_p, int no_q, int bd);
void orc_deblock_chroma_seg(uint16_t *pix, int xs, int ys, int tc8, int no_p, int no_q, int bd);
void orc_sao_ctb(const B200SaoRec *s, uint16_t *dst, const uint16_t *src, int stride, int x0, int y0, int w, int h, int bd);

extern const uint8_t ff_hevc_pel_weight[65];

static uint64_t g_seed = 0xB2000001ULL;
static uint64_t rnd64(void) { uint64_t z = (g_seed += 0x9E3779B97F4A7C15ULL); z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL; z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL; return z ^ (z >> 31); }
static int rnd(int n) { return (int)(rnd64() % (uint64_t)n); }
static int rndr(int lo, int hi) { return lo + rnd(hi - lo + 1); }

static int g_fail, g_checks, g_wraps, g_strong, g_strong_edge[2], g_bclip[2];
#define CHECK(cond, ...) do { g_checks++; if (!(cond)) { if (g_fail < 20) { fprintf(stderr, "MISMATCH: " __VA_ARGS__); fprintf(stderr, "\n"); } g_fail++; } } while (0)

/* native-format plane (uint8 for 8 bit, uint16 above) <-> oracle uint16 plane */
typedef struct { uint8_t *base; uint8_t *data; int stride; int w, h, pad, bd; } Plane;
static Plane plane_alloc(int w, int h, int pad, int bd)
{
    Plane p; int B = bd > 8 ? 2 : 1;
    p.w = w; p.h = h; p.pad = pad; p.bd = bd; p.stride = (w + 2 * pad) * B;
    p.base = calloc((size_t)p.stride * (h + 2 * pad), 1);
    p.data = p.base + pad * p.stride + pad * B;
    return p;
}
static void plane_free(Plane *p) { free(p->base); }
static void plane_put(Plane *p, int x, int y, int v) { if (p->bd > 8) ((uint16_t *)(p->data + y * p->stride))[x] = (uint16_t)v; else p->data[y * p->stride + x] = (uint8_t)v; }
static int plane_get(const Plane *p, int x, int y) { return p->bd > 8 ? ((uint16_t *)(p->data + y * p->stride))[x] : p->data[y * p->stride + x]; }
/* luma fraction 2 (hevcdsp.c:1028-1042): the 2-D filter of fraction (2, 2) has every tap product nonzero */
static const int k_qpel2[8] = { -1, 4, -11, 40, 40, -11, 4, -1 };

/* smooth-ish random content so that deblock / SAO / intra-strong decisions hit every branch; mode 2 (3): the sign pattern, the
 * maximum where the tap product of fraction (2, 2) at (x mod 8, y mod 8) is positive (negative), else 0 -- the content that takes
 * the 2-D intermediate to its maximum (minimum), beyond int16 for the maximum */
static void plane_fill(Plane *p, int mode)
{
    if (mode >= 2) {
        const int maxv = (1 << p->bd) - 1;
        for (int y = -p->pad; y < p->h + p->pad; y++)
            for (int x = -p->pad; x < p->w + p->pad; x++) {
                const int prod = k_qpel2[x & 7] * k_qpel2[y & 7];
                plane_put(p, x, y, (mode == 2 ? prod > 0 : prod < 0) ? maxv : 0);
            }
        return;
    }
    int maxv = (1 << p->bd) - 1, base = rnd(maxv + 1), gx = rndr(-3, 3), gy = rndr(-3, 3), noise = mode == 0 ? maxv : (1 << rnd(4)) << (p->bd - 8);
    for (int y = -p->pad; y < p->h + p->pad; y++)
        for (int x = -p->pad; x < p->w + p->pad; x++) {
            int v = mode == 0 ? rnd(maxv + 1) : base + ((gx * x + gy * y) << (p->bd - 8)) / 2 + rnd(noise + 1) - noise / 2 + ((x / 8 + y / 8) & 1) * rnd(3) * (4 << (p->bd - 8));
            plane_put(p, x, y, v < 0 ? 0 : v > maxv ? maxv : v);
        }
}
static uint16_t *plane_to_u16(const Plane *p)
{
    uint16_t *o = malloc(sizeof(uint16_t) * p->w * p->h);
    for (int y = 0; y < p->h; y++) for (int x = 0; x < p->w; x++) o[y * p->w + x] = (uint16_t)plane_get(p, x, y);
    return o;
}
static int plane_cmp(const Plane *p, const uint16_t *o)
{
    int bad = 0;
    for (int y = 0; y < p->h; y++) for (int x = 0; x < p->w; x++) bad += plane_get(p, x, y) != o[y * p->w + x];
    return bad;
}

/* ---------------------------------------------------------------- transforms */
/* sign of T[j][r], weight of input j in output r of the N-point inverse DCT (HEVC core transform), or of the inverse DST-VII */
static int basis_sign(int dst, int n, int j, int r)
{
    static const int8_t D[4][4] = { { 29, 55, 74, 84 }, { 74, 74, 0, -74 }, { 84, -29, -74, 55 }, { 55, -84, 74, -29 } };
    if (dst) return D[j][r] >= 0 ? 1 : -1;
    const int m = ((2 * r + 1) * j * (32 / n)) & 127;           /* T32[j * 32 / n][r] = +-|cos(m * pi / 64)| */
    return (m <= 32 || m >= 96) ? 1 : -1;
}
static void test_transforms(HEVCDSPContext *d, int bd, int trials)
{
    for (int t = 0; t < trials; t++) {
        int log2 = rndr(2, 5), n = 1 << log2, n2 = n * n;
        DECLARE_ALIGNED(32, int16_t, a[1024]); DECLARE_ALIGNED(32, int16_t, b[1024]);
        int style = rnd(5), which = rnd(8);
        memset(a, 0, sizeof(a));
        if (style == 4) {   /* basis sign pattern: the sign of coefficient (j, i) is that of basis entry j of output row r times entry i of
                             * output column c, so every first-stage sum of row r is as large as int32 input allows (far beyond int16) */
            const int m = which == 5 ? 4 : n, r = rnd(m), c = rnd(m), big = rnd(2) ? 32767 : -32768;
            for (int j = 0; j < m; j++)
                for (int i = 0; i < m; i++)
                    a[j * m + i] = (int16_t)((basis_sign(which == 5, m, j, r) * basis_sign(which == 5, m, i, c) > 0) ? big : (big < 0 ? 32767 : -32768));
        }
        for (int i = 0; i < n2 && style != 4; i++) {
            int v = 0;
            if (style == 0) v = rndr(-32768, 32767);                         /* dense, full range */
            else if (style == 1) v = rnd(4) ? 0 : rndr(-2000, 2000);         /* sparse moderate */
            else if (style == 2) { int x = i % n, y = i / n; v = (x + y < rndr(1, n)) ? rndr(-600, 600) : 0; } /* low-frequency triangle */
            else v = rndr(-64, 64);
            a[i] = (int16_t)v;
        }
        memcpy(b, a, sizeof(a));
        if (which <= 3) {
            int col_limit = rnd(3) ? rndr(1, 2 * n + 4) : n;
            d->idct[log2 - 2](a, col_limit); orc_idct(b, log2, col_limit, bd);
            CHECK(!memcmp(a, b, n2 * 2), "idct bd%d n%d col_limit %d style %d", bd, n, col_limit, style);
        } else if (which == 4) {
            d->idct_dc[log2 - 2](a); orc_idct_dc(b, log2, bd);
            CHECK(!memcmp(a, b, n2 * 2), "idct_dc bd%d n%d", bd, n);
        } else if (which == 5) {
            d->idct_4x4_luma(a); orc_dst4(b, bd);
            CHECK(!memcmp(a, b, 32), "dst4 bd%d", bd);
        } else if (which == 6) {
            d->transform_skip(a, log2); orc_transform_skip(b, log2, bd);
            CHECK(!memcmp(a, b, n2 * 2), "transform_skip bd%d n%d", bd, n);
            int mode = rnd(2);
            d->transform_rdpcm(a, log2, mode); orc_rdpcm(b, log2, mode);
            CHECK(!memcmp(a, b, n2 * 2), "rdpcm bd%d n%d mode %d", bd, n, mode);
        } else {
            Plane p = plane_alloc(64, 64, 0, bd); plane_fill(&p, rnd(2));
            uint16_t *o = plane_to_u16(&p);
            int x = rnd(64 / n) * n, y = rnd(64 / n) * n;
            d->transform_add[log2 - 2](p.data + y * p.stride + x * (bd > 8 ? 2 : 1), a, p.stride);
            orc_add_residual(o + y * 64 + x, 64, b, n, bd);
            CHECK(!plane_cmp(&p, o), "transform_add bd%d n%d", bd, n);
            free(o); plane_free(&p);
        }
    }
}

/* ---------------------------------------------------------------- inter prediction */
/* does the 2-D intermediate of luma fraction (2, 2) exceed int16 anywhere in the w x h block at (sx, sy)?  List 0 of a bi-predicted
 * block travels through the int16 tmp[] of hevc.c:1761 and wraps there; the oracle must wrap it the same way */
static int qpel22_exceeds_int16(const Plane *r, int sx, int sy, int w, int h, int bd)
{
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            int acc2 = 0;
            for (int j = 0; j < 8; j++) {
                const int yy = FFMIN(FFMAX(sy + y + j - 3, 0), r->h - 1);
                int acc = 0;
                for (int i = 0; i < 8; i++) acc += k_qpel2[i] * plane_get(r, FFMIN(FFMAX(sx + x + i - 3, 0), r->w - 1), yy);
                acc2 += k_qpel2[j] * (acc >> (bd - 8));
            }
            if ((acc2 >> 6) > 32767) return 1;
        }
    return 0;
}

static void test_mc(HEVCDSPContext *d, VideoDSPContext *vd, int bd, int trials)
{
    static const int widths[10] = { 2, 4, 6, 8, 12, 16, 24, 32, 48, 64 };
    const int B = bd > 8 ? 2 : 1;
    for (int t = 0; t < trials; t++) {
        const int PW = 160, PH = 128;
        Plane r0 = plane_alloc(PW, PH, 0, bd), r1 = plane_alloc(PW, PH, 0, bd), dst = plane_alloc(PW, PH, 0, bd);
        const int sign = rnd(4) == 0;              /* the sign pattern in list 0, its complement in list 1 */
        plane_fill(&r0, sign ? 2 : rnd(3) == 0); plane_fill(&r1, sign ? 3 : rnd(3) == 0); plane_fill(&dst, 1);
        int chroma = rnd(2), widx = chroma ? rnd(9) : rndr(1, 9); if (!chroma && widths[widx] == 6) widx = 3;
        int w = widths[widx], h = chroma ? (1 + rnd(32)) * 2 : (1 + rnd(16)) * 4; if (h > 64) h = 64;
        int bi = rnd(2), weighted = rnd(2);
        int fmax = chroma ? 8 : 4, before = chroma ? 1 : 3, extra = chroma ? 3 : 7;
        int mx0 = rnd(fmax), my0 = rnd(fmax), mx1 = rnd(fmax), my1 = rnd(fmax);
        if (sign && !chroma && bi) mx0 = my0 = 2;
        int dx = rnd(PW - w + 1), dy = rnd(PH - h + 1);
        int edge = rnd(sign ? 8 : 4) == 0;   /* let the source window hang over the picture: emulated_edge_mc path */
        int sx[2], sy[2];
        for (int l = 0; l < 2; l++) {
            if (edge) { sx[l] = rndr(-w - 12, PW + 12); sy[l] = rndr(-h - 12, PH + 12); }
            else { sx[l] = rndr(before, PW - w - extra + before - 1); sy[l] = rndr(before, PH - h - extra + before - 1); }
        }
        /* explicit weights: luma_weight = 2^denom + delta, delta and the offsets in [-128, 127] (hevc.c:251); the limits a quarter of the time */
        int denom = rnd(8), w0 = (1 << denom) + (rnd(4) ? rndr(-128, 127) : rnd(2) ? -128 : 127), w1 = (1 << denom) + (rnd(4) ? rndr(-128, 127) : rnd(2) ? -128 : 127);
        int o0 = rnd(4) ? rndr(-128, 127) : rnd(2) ? -128 : 127, o1 = rnd(4) ? rndr(-128, 127) : rnd(2) ? -128 : 127;
        uint16_t *od = plane_to_u16(&dst), *or0 = plane_to_u16(&r0), *or1 = plane_to_u16(&r1);

        /* reference: mimic hevc.c:1641-1790 (pointer + optional edge emulation + table call) */
        DECLARE_ALIGNED(16, int16_t, tmp[64 * 64]);
        uint8_t *emu[2]; emu[0] = malloc(80 * 2 * 80); emu[1] = malloc(80 * 2 * 80);
        uint8_t *src[2]; ptrdiff_t sstride[2];
        Plane *rp[2] = { &r0, &r1 };
        for (int l = 0; l < 2; l++) {
            src[l] = rp[l]->data + sy[l] * rp[l]->stride + sx[l] * B; sstride[l] = rp[l]->stride;
            if (sx[l] < before || sy[l] < before || sx[l] >= PW - w - (extra - before) || sy[l] >= PH - h - (extra - before)) {
                int es = 80 * B;
                vd->emulated_edge_mc(emu[l], src[l] - before * sstride[l] - before * B, es, sstride[l], w + extra, h + extra,
                                     sx[l] - before, sy[l] - before, PW, PH);
                src[l] = emu[l] + before * es + before * B; sstride[l] = es;
            }
        }
        uint8_t *dp = dst.data + dy * dst.stride + dx * B;
        int idx = ff_hevc_pel_weight[w];
        if (!chroma) {
            if (!bi) {
                if (!weighted) d->put_hevc_qpel_uni[idx][!!my0][!!mx0](dp, dst.stride, src[0], sstride[0], h, mx0, my0, w);
                else d->put_hevc_qpel_uni_w[idx][!!my0][!!mx0](dp, dst.stride, src[0], sstride[0], h, denom, w0, o0, mx0, my0, w);
            } else {
                d->put_hevc_qpel[idx][!!my0][!!mx0](tmp, 64, src[0], sstride[0], h, mx0, my0, w);
                if (!weighted) d->put_hevc_qpel_bi[idx][!!my1][!!mx1](dp, dst.stride, src[1], sstride[1], tmp, 64, h, mx1, my1, w);
                else d->put_hevc_qpel_bi_w[idx][!!my1][!!mx1](dp, dst.stride, src[1], sstride[1], tmp, 64, h, denom, w0, w1, o0, o1, mx1, my1, w);
            }
        } else {
            if (!bi) {
                if (!weighted) d->put_hevc_epel_uni[idx][!!my0][!!mx0](dp, dst.stride, src[0], sstride[0], h, mx0, my0, w);
                else d->put_hevc_epel_uni_w[idx][!!my0][!!mx0](dp, dst.stride, src[0], sstride[0], h, denom, w0, o0, mx0, my0, w);
            } else {
                d->put_hevc_epel[idx][!!my0][!!mx0](tmp, 64, src[0], sstride[0], h, mx0, my0, w);
                if (!weighted) d->put_hevc_epel_bi[idx][!!my1][!!mx1](dp, dst.stride, src[1], sstride[1], tmp, 64, h, mx1, my1, w);
                else d->put_hevc_epel_bi_w[idx][!!my1][!!mx1](dp, dst.stride, src[1], sstride[1], tmp, 64, h, denom, w0, w1, o0, o1, mx1, my1, w);
            }
        }
        B200McRec m; memset(&m, 0, sizeof(m));
        m.x = dx; m.y = dy; m.w = w; m.h = h; m.plane = chroma; m.flags = (bi ? B200_MCF_BI : 0) | (weighted ? B200_MCF_WEIGHTED : 0) | (chroma ? B200_MCF_CHROMA : 0);
        m.sx0 = sx[0]; m.sy0 = sy[0]; m.sx1 = sx[1]; m.sy1 = sy[1]; m.frac0 = mx0 | my0 << 4; m.frac1 = mx1 | my1 << 4;
        m.w0 = w0; m.w1 = w1; m.o0 = o0; m.o1 = o1; m.denom = denom;
        orc_mc_rec(&m, od, PW, or0, or1, PW, PH, bd);
        if (bi && !chroma && mx0 == 2 && my0 == 2) g_wraps += qpel22_exceeds_int16(&r0, sx[0], sy[0], w, h, bd);
        CHECK(!plane_cmp(&dst, od), "mc bd%d chroma%d %dx%d bi%d w%d frac %d,%d %d,%d edge%d src %d,%d", bd, chroma, w, h, bi, weighted, mx0, my0, mx1, my1, edge, sx[0], sy[0]);
        free(od); free(or0); free(or1); free(emu[0]); free(emu[1]);
        plane_free(&r0); plane_free(&r1); plane_free(&dst);
    }
}

/* ---------------------------------------------------------------- intra prediction */
/* the top row (from the corner to index 2n - 1) and the left column of an n x n block at (x, y) of plane p, where they exist */
static void fill_neighbours(Plane *p, int x, int y, int n, int content)
{
    const int maxv = (1 << p->bd) - 1, thr = 1 << (p->bd - 5);
    int top[65], left[65];                                   /* [k] = index k - 1 */
    if (content == 1) {
        const int st = rnd(maxv / 70 + 1), sl = rnd(maxv / 70 + 1), base = rndr(thr + 1, maxv - 65 * FFMAX(st, sl) - thr - 1);
        for (int k = 0; k <= 2 * n; k++) { top[k] = base + st * k; left[k] = base + sl * k; }
        const int d = (int[3]){ 0, thr - 1, thr }[rnd(3)];
        int *side = rnd(2) ? top : left;
        side[2 * n] += side[2 * n] + d <= maxv ? d : -d;
    } else if (content == 2) {
        const int kind = rnd(3);
        for (int k = 0; k <= 2 * n; k++) top[k] = left[k] = kind == 0 ? 0 : kind == 1 ? maxv : (k & 1) * maxv;
    } else {
        const int hi = rnd(2);
        for (int k = 0; k <= 2 * n; k++) top[k] = left[k] = (k == 0) == hi ? 0 : maxv;
    }
    if (y > 0) for (int k = 0; k <= 2 * n && x - 1 + k < p->w; k++) if (x - 1 + k >= 0) plane_put(p, x - 1 + k, y - 1, top[k]);
    if (x > 0) for (int k = 0; k <= 2 * n && y - 1 + k < p->h; k++) if (y - 1 + k >= 0) plane_put(p, x - 1, y - 1 + k, left[k]);
}

/* what the block's prediction must go through, restated where the up-left, up and left neighbours exist (the reference
 * arrays are then the picture's samples, with the unavailable or out-of-picture part of the up-right / bottom-left halves
 * replaced by the last sample before it): strong smoothing decisions (and blocks one step either side of the threshold),
 * and the mode-26 / mode-10 boundary filters clipped at 0 and at max */
static void count_intra_limits(const B200IntraRec *r, const uint16_t *o, int pw, int ph, int bd)
{
    const int need = B200_INF_UP_LEFT | B200_INF_UP | B200_INF_LEFT;
    if ((r->flags & need) != need) return;
    const int n = 1 << r->log2, x = r->x, y = r->y, maxv = (1 << bd) - 1, thr = 1 << (bd - 5);
    int tb[65], lb[65], *top = tb + 1, *left = lb + 1;
    top[-1] = left[-1] = o[(y - 1) * pw + x - 1];
    for (int i = 0; i < n; i++) { top[i] = o[(y - 1) * pw + x + i]; left[i] = o[(y + i) * pw + x - 1]; }
    for (int i = 0; i < n; i++) {
        top[n + i] = (r->flags & B200_INF_UP_RIGHT) ? o[(y - 1) * pw + x + n + FFMIN(i, r->top_right_size - 1)] : top[n - 1];
        left[n + i] = (r->flags & B200_INF_BOTTOM_LEFT) ? o[(y + n + FFMIN(i, r->bottom_left_size - 1)) * pw + x - 1] : left[n - 1];
    }
    (void)ph;
    const int mode = r->mode;
    if (r->plane == 0 && n < 32 && (mode == 10 || mode == 26))
        for (int i = 0; i < n; i++) {
            const int v = mode == 26 ? top[0] + ((left[i] - left[-1]) >> 1) : left[0] + ((top[i] - top[-1]) >> 1);
            if (v < 0) { g_bclip[0]++; break; }
            if (v > maxv) { g_bclip[1]++; break; }
        }
    if (r->plane == 0 && r->log2 == 5 && (r->flags & B200_INF_FILTER) && (r->flags & B200_INF_STRONG) && mode != 1 && mode != 10 && mode != 26) {
        const int d = FFMAX(abs(top[-1] + top[63] - 2 * top[31]), abs(left[-1] + left[63] - 2 * left[31]));
        g_strong += d < thr;
        g_strong_edge[0] += d == thr - 1;
        g_strong_edge[1] += d == thr;
    }
}
static void test_intra(int bd, int trials, int cfi)
{
    /* a genuine (minimal) decoder context: intra_pred reads sps/pps/frame/HEVClc, hevcpred_template.c:30-110 */
    HEVCContext *s = calloc(1, sizeof(*s));
    HEVCSPS *sps = calloc(1, sizeof(*sps));
    HEVCPPS *pps = calloc(1, sizeof(*pps));
    HEVCLocalContext *lc = calloc(1, sizeof(*lc));
    AVFrame *fr = calloc(1, sizeof(*fr));
    const int W = 192, H = 128, B = bd > 8 ? 2 : 1;
    s->sps = sps; s->pps = pps; s->HEVClc = lc; s->frame = fr;
    ff_hevc_pred_init(&s->hpc, bd);
    sps->width = W; sps->height = H; sps->log2_ctb_size = 6; sps->log2_min_tb_size = 2; sps->log2_min_pu_size = 2;
    sps->tb_mask = 15; sps->min_pu_width = W / 4; sps->min_pu_height = H / 4; sps->chroma_array_type = cfi; sps->pixel_shift = bd > 8;
    sps->hshift[0] = sps->vshift[0] = 0;
    sps->hshift[1] = sps->hshift[2] = cfi != 3; sps->vshift[1] = sps->vshift[2] = cfi == 1;
    sps->ctb_width = W / 64; sps->ctb_height = H / 64;
    int *zs = malloc(sizeof(int) * 17 * 17);
    pps->min_tb_addr_zs_tab = zs; pps->min_tb_addr_zs = zs + 17 + 1;
    for (int y = 0; y < 17; y++) { zs[y * 17] = -1; zs[y] = -1; }
    for (int y = 0; y < 16; y++) for (int x = 0; x < 16; x++) { int v = 0; for (int i = 0; i < 4; i++) { int m = 1 << i; v += (m & x ? m * m : 0) + (m & y ? 2 * m * m : 0); } pps->min_tb_addr_zs[y * 17 + x] = v; }

    for (int t = 0; t < trials; t++) {
        Plane pl[3]; uint16_t *op[3];
        for (int c = 0; c < 3; c++) { pl[c] = plane_alloc(W >> sps->hshift[c], H >> sps->vshift[c], 0, bd); plane_fill(&pl[c], rnd(3) == 0); fr->data[c] = pl[c].data; fr->linesize[c] = pl[c].stride; }
        sps->sps_strong_intra_smoothing_enable_flag = rnd(2);
        sps->spsRext.intra_smoothing_disabled_flag = rnd(8) == 0;
        int c_idx = rnd(3), log2 = rndr(2, 5), n = 1 << log2;
        /* neighbour content at the limits: 1 linear ramps, with the second difference at index 31 of one side 0, thr - 1 or
         * thr (the strong-smoothing test, hevcpred_template.c:296-300); 2 all 0, all max or 0 / max alternating; 3 corner
         * and top / left at opposite ends (the mode-10 / mode-26 boundary filters past 0 or max) */
        const int content = rnd(3) ? 0 : 1 + rnd(3);
        if (content == 1 && rnd(2)) c_idx = 0, log2 = 5, n = 32;
        if (content == 3 && rnd(2)) c_idx = 0, log2 = rndr(2, 4), n = 1 << log2;
        if (c_idx && cfi != 3 && log2 == 5 && rnd(2)) log2 = 4, n = 16;
        int hs = sps->hshift[c_idx], vs = sps->vshift[c_idx];
        int nl_h = n << hs, nl_v = n << vs;               /* size in luma units */
        if (nl_h > 64 || nl_v > 64) { log2--; n >>= 1; nl_h >>= 1; nl_v >>= 1; }
        int x0 = rnd(W / nl_h) * nl_h, y0 = rnd(H / nl_v) * nl_v;
        if (rnd(3) == 0) x0 = rnd(2) ? 0 : W - nl_h;
        if (rnd(3) == 0) y0 = rnd(2) ? 0 : H - nl_v;
        int mode = rnd(4) == 0 ? rnd(2) : rndr(2, 34);
        if (rnd(6) == 0 || content == 3) mode = rnd(2) ? 10 : 26;
        if (content) fill_neighbours(&pl[c_idx], x0 >> hs, y0 >> vs, n, content);
        lc->tu.intra_pred_mode = lc->tu.intra_pred_mode_c = mode;
        /* CTB neighbourhood flags as hls_decode_neighbour would set them for a single slice / tile (hevc.c:2590-2660) */
        int xc = x0 >> 6, yc = y0 >> 6;
        lc->ctb_left_flag = xc > 0; lc->ctb_up_flag = yc > 0; lc->ctb_up_left_flag = xc > 0 && yc > 0;
        lc->ctb_up_right_flag = yc > 0 && xc + 1 < sps->ctb_width;
        lc->end_of_tiles_x = W; lc->end_of_tiles_y = FFMIN((yc + 1) * 64, H);
        if (rnd(8) == 0) { lc->ctb_left_flag = rnd(2) && xc > 0; lc->ctb_up_flag = rnd(2) && yc > 0; lc->ctb_up_left_flag &= rnd(2); lc->ctb_up_right_flag &= rnd(2); } /* slice / tile borders */
        ff_hevc_set_neighbour_available(s, x0, y0, nl_h, nl_v);
        for (int c = 0; c < 3; c++) op[c] = plane_to_u16(&pl[c]);

        s->hpc.intra_pred[log2 - 2](s, x0, y0, c_idx);

        /* record exactly what the B200 recorder derives (same logic as hevcpred_template.c:82-109) */
        B200IntraRec r; memset(&r, 0, sizeof(r));
        int tbs_h = nl_h >> 2, tbs_v = nl_v >> 2, x_tb = (x0 >> 2) & 15, y_tb = (y0 >> 2) & 15;
        int cur = pps->min_tb_addr_zs[y_tb * 17 + x_tb];
        int bl = lc->na.cand_bottom_left && cur > pps->min_tb_addr_zs[((y_tb + tbs_v) & 15) * 17 + x_tb - 1];
        int ur = lc->na.cand_up_right && cur > pps->min_tb_addr_zs[(y_tb - 1) * 17 + ((x_tb + tbs_h) & 15)];
        r.x = x0 >> hs; r.y = y0 >> vs; r.plane = c_idx; r.log2 = log2; r.mode = mode;
        r.flags = (lc->na.cand_up_left ? B200_INF_UP_LEFT : 0) | (lc->na.cand_up ? B200_INF_UP : 0) | (ur ? B200_INF_UP_RIGHT : 0) |
                  (lc->na.cand_left ? B200_INF_LEFT : 0) | (bl ? B200_INF_BOTTOM_LEFT : 0) |
                  ((!sps->spsRext.intra_smoothing_disabled_flag && (c_idx == 0 || cfi == 3)) ? B200_INF_FILTER : 0) |
                  (sps->sps_strong_intra_smoothing_enable_flag ? B200_INF_STRONG : 0);
        r.bottom_left_size = (FFMIN(y0 + 2 * nl_v, H) - (y0 + nl_v)) >> vs;
        r.top_right_size = (FFMIN(x0 + 2 * nl_h, W) - (x0 + nl_h)) >> hs;
        r.resid_off = B200_NO_RESID;
        count_intra_limits(&r, op[c_idx], pl[c_idx].w, pl[c_idx].h, bd);
        orc_intra_rec(&r, op[c_idx], pl[c_idx].w, bd);
        CHECK(!plane_cmp(&pl[c_idx], op[c_idx]), "intra bd%d cfi%d c%d n%d mode%d at %d,%d flags %x", bd, cfi, c_idx, n, mode, x0, y0, r.flags);
        for (int c = 0; c < 3; c++) { free(op[c]); plane_free(&pl[c]); }
    }
    free(zs); free(fr); free(lc); free(pps); free(sps); free(s);
    (void)B;
}

/* ---------------------------------------------------------------- deblocking */
static void test_deblock(HEVCDSPContext *d, int bd, int trials)
{
    const int B = bd > 8 ? 2 : 1;
    for (int t = 0; t < trials; t++) {
        Plane p = plane_alloc(32, 32, 0, bd); plane_fill(&p, rnd(5) == 0 ? 0 : 1);
        uint16_t *o = plane_to_u16(&p);
        int vert = rnd(2), chroma = rnd(2), c_variant = rnd(2);
        int beta = rnd(65), tc[2] = { rnd(4) ? rnd(25) : 0, rnd(4) ? rnd(25) : 0 };
        uint8_t no_p[2] = { rnd(4) == 0, rnd(4) == 0 }, no_q[2] = { rnd(4) == 0, rnd(4) == 0 };
        int x = vert ? 8 * rndr(1, 3) : 8 * rnd(4), y = vert ? 8 * rnd(4) : 8 * rndr(1, 3);
        uint8_t *pix = p.data + y * p.stride + x * B;
        if (!chroma) {
            if (vert) (c_variant ? d->hevc_v_loop_filter_luma_c : d->hevc_v_loop_filter_luma)(pix, p.stride, beta, tc, no_p, no_q);
            else      (c_variant ? d->hevc_h_loop_filter_luma_c : d->hevc_h_loop_filter_luma)(pix, p.stride, beta, tc, no_p, no_q);
        } else {
            if (vert) (c_variant ? d->hevc_v_loop_filter_chroma_c : d->hevc_v_loop_filter_chroma)(pix, p.stride, tc, no_p, no_q);
            else      (c_variant ? d->hevc_h_loop_filter_chroma_c : d->hevc_h_loop_filter_chroma)(pix, p.stride, tc, no_p, no_q);
        }
        for (int j = 0; j < 2; j++) {
            uint16_t *q = o + (vert ? (y + 4 * j) * 32 + x : y * 32 + x + 4 * j);
            if (!chroma) orc_deblock_luma_seg(q, vert ? 1 : 32, vert ? 32 : 1, beta, tc[j], no_p[j], no_q[j], bd);
            else         orc_deblock_chroma_seg(q, vert ? 1 : 32, vert ? 32 : 1, tc[j], no_p[j], no_q[j], bd);
        }
        CHECK(!plane_cmp(&p, o), "deblock bd%d vert%d chroma%d beta%d tc%d,%d", bd, vert, chroma, beta, tc[0], tc[1]);
        free(o); plane_free(&p);
    }
}

/* ---------------------------------------------------------------- SAO */
static void test_sao(HEVCDSPContext *d, int bd, int trials)
{
    const int B = bd > 8 ? 2 : 1;
    for (int t = 0; t < trials; t++) {
        int w = rnd(3) ? 64 >> rnd(2) : 8 * rndr(1, 8), h = rnd(3) ? 64 >> rnd(2) : 8 * rndr(1, 8);
        /* the reference filters frame <- sao_frame copy; both carry a 1-sample ring (hevc.c:369-385) */
        Plane src = plane_alloc(w, h, 1, bd), dst = plane_alloc(w, h, 1, bd);
        plane_fill(&src, rnd(4) == 0 ? 0 : 1);
        memcpy(dst.base, src.base, (size_t)src.stride * (h + 2));
        SAOParams sp; memset(&sp, 0, sizeof(sp));
        int c_idx = rnd(3), edge = rnd(2), variant = rnd(2);
        int maxo = (1 << (FFMIN(bd, 10) - 5)) - 1;
        sp.band_position[c_idx] = rnd(32); sp.eo_class[c_idx] = rnd(4);
        for (int k = 1; k < 5; k++) sp.offset_val[c_idx][k] = rndr(-maxo, maxo);
        int borders[4]; uint8_t ve[2], he[2], de[4];
        for (int k = 0; k < 4; k++) borders[k] = rnd(4) == 0;
        ve[0] = !borders[0] && rnd(3) == 0; ve[1] = !borders[2] && rnd(3) == 0; he[0] = !borders[1] && rnd(3) == 0; he[1] = !borders[3] && rnd(3) == 0;
        de[0] = !borders[0] && !borders[1] && rnd(3) == 0; de[1] = !borders[1] && !borders[2] && rnd(3) == 0;
        de[2] = !borders[2] && !borders[3] && rnd(3) == 0; de[3] = !borders[0] && !borders[3] && rnd(3) == 0;
        /* oracle works on a picture that contains the tile and its ring */
        int PW = w + 2;
        uint16_t *osrc = malloc(sizeof(uint16_t) * PW * (h + 2)), *odst = malloc(sizeof(uint16_t) * PW * (h + 2));
        for (int y = -1; y <= h; y++) for (int x = -1; x <= w; x++) osrc[(y + 1) * PW + x + 1] = odst[(y + 1) * PW + x + 1] = (uint16_t)plane_get(&src, x, y);
        if (!edge) d->sao_band_filter(dst.data, src.data, dst.stride, src.stride, &sp, borders, w, h, c_idx);
        else d->sao_edge_filter[variant](dst.data, src.data, dst.stride, src.stride, &sp, borders, w, h, c_idx, ve, he, de);
        B200SaoRec r; memset(&r, 0, sizeof(r));
        r.type = edge ? B200_SAO_EDGE : B200_SAO_BAND; r.param = edge ? sp.eo_class[c_idx] : sp.band_position[c_idx];
        r.borders = borders[0] | borders[1] << 1 | borders[2] << 2 | borders[3] << 3;
        r.edges = ve[0] | ve[1] << 1 | he[0] << 2 | he[1] << 3 | de[0] << 4 | de[1] << 5 | de[2] << 6 | de[3] << 7;
        r.variant = variant;
        for (int k = 0; k < 5; k++) r.offset_val[k] = sp.offset_val[c_idx][k];
        orc_sao_ctb(&r, odst, osrc, PW, 1, 1, w, h, bd);
        int bad = 0;
        for (int y = 0; y < h; y++) for (int x = 0; x < w; x++) bad += plane_get(&dst, x, y) != odst[(y + 1) * PW + x + 1];
        CHECK(!bad, "sao bd%d edge%d variant%d class%d %dx%d borders %x edges %x", bd, edge, variant, r.param, w, h, r.borders, r.edges);
        free(osrc); free(odst); plane_free(&src); plane_free(&dst);
    }
    (void)B;
}

int main(int argc, char **argv)
{
    int trials = argc > 1 ? atoi(argv[1]) : 2000;
    static const int depths[3] = { 8, 10, 12 };
    for (int k = 0; k < 3; k++) {
        int bd = depths[k];
        HEVCDSPContext d; VideoDSPContext vd;
        ff_hevc_dsp_init(&d, bd); ff_videodsp_init(&vd, bd);
        int f0 = g_fail;
        test_transforms(&d, bd, trials * 4);     printf("bd%-2d transforms  fails %d\n", bd, g_fail - f0); f0 = g_fail;
        const int w0 = g_wraps;
        test_mc(&d, &vd, bd, trials);             printf("bd%-2d mc          fails %d, blocks whose list 0 wrapped in int16 %d\n", bd, g_fail - f0, g_wraps - w0);
        CHECK(g_wraps > w0, "bd%d: no bi-predicted block took list 0 beyond int16", bd);
        f0 = g_fail;
        const int s0 = g_strong, e0 = g_strong_edge[0], e1 = g_strong_edge[1], c0 = g_bclip[0], c1 = g_bclip[1];
        for (int cfi = 1; cfi <= 3; cfi++) test_intra(bd, trials, cfi);
        printf("bd%-2d intra       fails %d, strong smoothing %d (at threshold - 1: %d, at threshold: %d), boundary filter clipped at 0: %d, at max: %d\n",
               bd, g_fail - f0, g_strong - s0, g_strong_edge[0] - e0, g_strong_edge[1] - e1, g_bclip[0] - c0, g_bclip[1] - c1);
        CHECK(g_strong > s0, "bd%d: no 32x32 luma block took strong smoothing", bd);
        CHECK(g_bclip[0] > c0 && g_bclip[1] > c1, "bd%d: the mode-10 / mode-26 boundary filters were not clipped at both ends", bd);
        f0 = g_fail;
        test_deblock(&d, bd, trials * 2);         printf("bd%-2d deblock     fails %d\n", bd, g_fail - f0); f0 = g_fail;
        test_sao(&d, bd, trials);                 printf("bd%-2d sao         fails %d\n", bd, g_fail - f0);
    }
    printf("kat_ref: %d checks, %d mismatches\n", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
