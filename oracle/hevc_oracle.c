/*
 * hevc_oracle.c — TEST INFRASTRUCTURE ONLY (never linked into, imported by or executed
 * from the product path; only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline
 * leg may use it).
 *
 * Plain-C restatement of openHEVC's per-CTU pixel-reconstruction path, i.e. of the
 * functions behind HEVCDSPContext / HEVCPredContext, operating on the packed work list
 * of include/b200hevc_worklist.h.  Each function cites the reference file:line it
 * follows.  It is *restated*, not copied: transforms are written as masked matrix
 * products, MC as one generic separable FIR with clamped addressing, deblocking / SAO
 * as whole-picture passes.
 *
 * Parity pinning: the reference ships no golden vectors (SURVEY.md §4), so this file is
 * pinned against the reference's own C tables compiled from /root/reference into
 * oracle/_ref/libohevc_ref.so (oracle/build_ref.sh) by oracle/kat_ref.c, function by
 * function, against committed fixtures in tests/golden/ produced by that harness, at picture
 * level by oracle/replay_ref.c (the reference's functions in the decoder's call order), and at
 * stream level: the real decoder parses the committed Annex-B streams with the recording tables
 * installed (B200_SHIM_DUMP), this file executes the recorded work lists, and the per-plane MD5s
 * must equal those of the unmodified decoder (tests/test_stream_oracle_cpu.py).
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "../include/b200hevc_worklist.h"

typedef uint16_t pix_t; /* the oracle stores every sample as uint16, whatever the bit depth */

static inline int clip3(int v, int lo, int hi) { return v < lo ? lo : v > hi ? hi : v; }
static inline int clip16(int v) { return clip3(v, -32768, 32767); }
static inline int clip_pix(int v, int bd) { return clip3(v, 0, (1 << bd) - 1); }
static inline int iabs(int v) { return v < 0 ? -v : v; }

/* ------------------------------------------------------------------------------------------
 * Inverse transforms.  Reference: libavcodec/hevcdsp_template.c:165-326, matrix
 * libavcodec/hevcdsp.c:879-944 (the standard HEVC core transform).
 * ---------------------------------------------------------------------------------------- */
static int8_t g_T[32][32];
static int g_T_ready;

/* |64*sqrt(2)*cos(j*pi/64)| as standardised (hand-tuned integers), j = 0..32; j=0 is the DC row gain 64 */
static const int8_t k_cos_tab[33] = { 64, 90, 90, 90, 89, 88, 87, 85, 83, 82, 80, 78, 75, 73, 70, 67, 64,
                                      61, 57, 54, 50, 46, 43, 38, 36, 31, 25, 22, 18, 13, 9, 4, 0 };

static void build_matrix(void)
{
    if (g_T_ready) return;
    for (int k = 0; k < 32; k++)
        for (int n = 0; n < 32; n++) {
            int m = ((2 * n + 1) * k) & 127, v;
            if (m <= 32)      v =  k_cos_tab[m];
            else if (m <= 64) v = -k_cos_tab[64 - m];
            else if (m < 96)  v = -k_cos_tab[m - 64];
            else              v =  k_cos_tab[128 - m];
            g_T[k][n] = (int8_t)v;
        }
    g_T_ready = 1;
}
const int8_t *orc_transform_matrix(void) { build_matrix(); return &g_T[0][0]; }

/* Which input index j of an N-point 1-D transform the reference's pruned butterflies really read
 * when called with `end` (TR_8/16/32 macros, hevcdsp_template.c:223-269): odd terms are cut at
 * `end` on each recursion level that receives it, the innermost levels always read everything. */
static int idct_keep(int n, int j, int end)
{
    if (n == 4) return 1;
    if (n == 8 || n == 16) return !(j & 1) || j < end;
    /* n == 32 */
    if (j & 1) return j < end;
    if ((j & 3) == 2) return (j >> 1) < end / 2;
    return 1;
}

/* hevcdsp.idct[log2-2](coeffs, col_limit), in place */
void orc_idct(int16_t *c, int log2, int col_limit, int bd)
{
    build_matrix();
    const int n = 1 << log2, step = 32 >> log2;
    int tmp[32 * 32];
    int limit  = col_limit < n ? col_limit : n;           /* IDCT_VAR8: limit  */
    int limit2 = col_limit + 4 < n ? col_limit + 4 : n;   /*            limit2 */
    for (int i = 0; i < n; i++) {                         /* first stage: columns, >>7 */
        for (int r = 0; r < n; r++) {
            int acc = 0;
            for (int j = 0; j < n; j++)
                if (idct_keep(n, j, limit2))
                    acc += g_T[j * step][r] * c[j * n + i];
            tmp[r * n + i] = clip16((acc + 64) >> 7);
        }
        if (limit2 < n && (i & 3) == 0 && i) limit2 -= 4; /* hevcdsp_template.c:288-292 */
    }
    const int shift = 20 - bd, add = 1 << (shift - 1);
    for (int r = 0; r < n; r++)                           /* second stage: rows */
        for (int x = 0; x < n; x++) {
            int acc = 0;
            for (int j = 0; j < n; j++)
                if (idct_keep(n, j, limit))
                    acc += g_T[j * step][x] * tmp[r * n + j];
            c[r * n + x] = (int16_t)clip16((acc + add) >> shift);
        }
}

/* hevcdsp.idct_dc[log2-2], hevcdsp_template.c:303-316 */
void orc_idct_dc(int16_t *c, int log2, int bd)
{
    const int shift = 14 - bd, add = 1 << (shift - 1);
    const int v = (((c[0] + 1) >> 1) + add) >> shift;
    for (int i = 0; i < (1 << (2 * log2)); i++) c[i] = (int16_t)v;
}

/* hevcdsp.idct_4x4_luma (inverse DST-VII), hevcdsp_template.c:170-203 */
void orc_dst4(int16_t *c, int bd)
{
    static const int8_t M[4][4] = { { 29, 55, 74, 84 }, { 74, 74, 0, -74 }, { 84, -29, -74, 55 }, { 55, -84, 74, -29 } };
    int tmp[16];
    for (int i = 0; i < 4; i++)
        for (int r = 0; r < 4; r++) {
            int acc = 0;
            for (int j = 0; j < 4; j++) acc += M[j][r] * c[j * 4 + i];
            tmp[r * 4 + i] = clip16((acc + 64) >> 7);
        }
    const int shift = 20 - bd, add = 1 << (shift - 1);
    for (int r = 0; r < 4; r++)
        for (int x = 0; x < 4; x++) {
            int acc = 0;
            for (int j = 0; j < 4; j++) acc += M[j][x] * tmp[r * 4 + j];
            c[r * 4 + x] = (int16_t)clip16((acc + add) >> shift);
        }
}

/* hevcdsp.transform_skip, hevcdsp_template.c:139-163 */
void orc_transform_skip(int16_t *c, int log2, int bd)
{
    const int shift = 15 - bd - log2, n2 = 1 << (2 * log2);
    if (shift > 0) { for (int i = 0; i < n2; i++) c[i] = (int16_t)((c[i] + (1 << (shift - 1))) >> shift); }
    else           { for (int i = 0; i < n2; i++) c[i] = (int16_t)(c[i] << -shift); }
}

/* hevcdsp.transform_rdpcm, hevcdsp_template.c:114-136: running sums kept in int16 (wraps) */
void orc_rdpcm(int16_t *c, int log2, int vertical)
{
    const int n = 1 << log2;
    if (vertical) { for (int y = 1; y < n; y++) for (int x = 0; x < n; x++) c[y * n + x] = (int16_t)(c[y * n + x] + c[(y - 1) * n + x]); }
    else          { for (int y = 0; y < n; y++) for (int x = 1; x < n; x++) c[y * n + x] = (int16_t)(c[y * n + x] + c[y * n + x - 1]); }
}

/* residual of one TU record, in place in the pool */
static void tu_residual(const B200TuRec *t, int16_t *c, int bd)
{
    switch (t->kind) {
    case B200_TU_IDCT:   orc_idct(c, t->log2, t->col_limit, bd); break;
    case B200_TU_DC:     orc_idct_dc(c, t->log2, bd); break;
    case B200_TU_DST:    orc_dst4(c, bd); break;
    case B200_TU_SKIP:   orc_transform_skip(c, t->log2, bd); break;
    default: break;
    }
    if (t->flags & B200_TUF_RDPCM) orc_rdpcm(c, t->log2, !!(t->flags & B200_TUF_RDPCM_VERT));
}

/* hevcdsp.transform_add[log2-2], hevcdsp_template.c:45-111 */
void orc_add_residual(pix_t *dst, int stride, const int16_t *r, int n, int bd)
{
    for (int y = 0; y < n; y++)
        for (int x = 0; x < n; x++)
            dst[y * stride + x] = (pix_t)clip_pix(dst[y * stride + x] + r[y * n + x], bd);
}

/* ------------------------------------------------------------------------------------------
 * Inter prediction.  Reference: hevcdsp_template.c:610-1609 (put_hevc_{qpel,epel}*),
 * filters hevcdsp.c:1028-1042, edge emulation videodsp_template.c:26-100 (== clamp).
 * ---------------------------------------------------------------------------------------- */
static const int8_t k_qpel[4][8] = { { 0, 0, 0, 64, 0, 0, 0, 0 }, { -1, 4, -10, 58, 17, -5, 1, 0 },
                                     { -1, 4, -11, 40, 40, -11, 4, -1 }, { 0, 1, -5, 17, 58, -10, 4, -1 } };
static const int8_t k_epel[8][4] = { { 0, 64, 0, 0 }, { -2, 58, 10, -2 }, { -4, 54, 16, -2 }, { -6, 46, 28, -4 },
                                     { -4, 36, 36, -4 }, { -4, 28, 46, -6 }, { -2, 16, 54, -4 }, { -2, 10, 58, -2 } };

static inline int ref_px(const pix_t *ref, int pw, int ph, int x, int y)
{
    return ref[clip3(y, 0, ph - 1) * pw + clip3(x, 0, pw - 1)];
}

/* 14-bit intermediate of one reference list at output sample (x,y): the value put_hevc_qpel /
 * put_hevc_epel would write into its int16 dst */
static int mc_intermediate(const pix_t *ref, int pw, int ph, int x, int y, int mx, int my, int chroma, int bd)
{
    const int taps = chroma ? 4 : 8, before = chroma ? 1 : 3;
    const int8_t *fx = chroma ? k_epel[mx] : k_qpel[mx];
    const int8_t *fy = chroma ? k_epel[my] : k_qpel[my];
    if (!mx && !my) return ref_px(ref, pw, ph, x, y) << (14 - bd);
    if (mx && !my) {
        int acc = 0;
        for (int k = 0; k < taps; k++) acc += fx[k] * ref_px(ref, pw, ph, x + k - before, y);
        return acc >> (bd - 8);
    }
    if (!mx && my) {
        int acc = 0;
        for (int k = 0; k < taps; k++) acc += fy[k] * ref_px(ref, pw, ph, x, y + k - before);
        return acc >> (bd - 8);
    }
    int acc2 = 0;
    for (int j = 0; j < taps; j++) {
        int acc = 0;
        for (int k = 0; k < taps; k++) acc += fx[k] * ref_px(ref, pw, ph, x + k - before, y + j - before);
        acc2 += fy[j] * (int16_t)(acc >> (bd - 8));   /* tmp[] is int16, hevcdsp_template.c:774 */
    }
    return acc2 >> 6;
}

void orc_mc_rec(const B200McRec *m, pix_t *dst, int dst_stride, const pix_t *ref0, const pix_t *ref1,
                int pw, int ph, int bd)
{
    const int chroma = !!(m->flags & B200_MCF_CHROMA);
    const int mx0 = m->frac0 & 15, my0 = m->frac0 >> 4, mx1 = m->frac1 & 15, my1 = m->frac1 >> 4;
    const int shift = 14 - bd;
    for (int y = 0; y < m->h; y++)
        for (int x = 0; x < m->w; x++) {
            pix_t *d = &dst[(m->y + y) * dst_stride + m->x + x];
            int v0 = mc_intermediate(ref0, pw, ph, m->sx0 + x, m->sy0 + y, mx0, my0, chroma, bd), out;
            if (!(m->flags & B200_MCF_BI)) {
                if (!(m->flags & B200_MCF_WEIGHTED)) {
                    /* put_hevc_*_uni_*: full-pel is a plain copy (:626-640), else (v + off) >> (14-BD) */
                    out = (!mx0 && !my0) ? (v0 >> shift) : clip_pix((v0 + (1 << (shift - 1))) >> shift, bd);
                } else {
                    /* put_hevc_*_uni_w_*  :668-690 */
                    const int s = m->denom + shift;
                    out = clip_pix(((v0 * m->w0 + (1 << (s - 1))) >> s) + m->o0 * (1 << (bd - 8)), bd);
                }
            } else {
                int v1 = mc_intermediate(ref1, pw, ph, m->sx1 + x, m->sy1 + y, mx1, my1, chroma, bd);
                v0 = (int16_t)v0;                       /* first list goes through the int16 tmp[] (hevc.c:1761) */
                if (!(m->flags & B200_MCF_WEIGHTED)) {
                    out = clip_pix((v1 + v0 + (1 << shift)) >> (shift + 1), bd);        /* :642-666 */
                } else {
                    const int log2wd = m->denom + shift;                                   /* :692-720 */
                    const int o = (m->o0 + m->o1) * (1 << (bd - 8)) + 1;
                    out = clip_pix((v1 * m->w1 + v0 * m->w0 + (o << log2wd)) >> (log2wd + 1), bd);
                }
            }
            *d = (pix_t)out;
        }
}

/* ------------------------------------------------------------------------------------------
 * Intra prediction.  Reference: hevcpred_template.c:30-344 (neighbour gathering, substitution,
 * smoothing), :359-384 planar, :388-417 DC, :419-538 angular.  constrained_intra_pred
 * (:116-163 candidate flags from the PU types, :185-249 substitution of the samples of inter
 * neighbours) is restated in orc_cip_flags() / orc_cip_substitute(); the record's flags are the
 * availability BEFORE those rules, the intra bitmap travels in the blob (B200BlobHeader.cip).
 * ---------------------------------------------------------------------------------------- */
typedef struct OrcCip {          /* NULL pointer = picture without constrained_intra_pred */
    int log2_min_pu, pu_w, pu_h;
    const uint32_t *bits;        /* one bit per min-PU, row-major: MvField.pred_flag == PF_INTRA */
    int hs, vs;                  /* chroma shifts of the plane the record is in */
    int pic_w, pic_h;            /* luma size (sps->width / height) */
} OrcCip;

static int cip_pu_intra(const OrcCip *c, int px, int py)                   /* MVF(x, y).pred_flag == PF_INTRA (:35-36) */
{
    const long i = (long)px + (long)py * c->pu_w;                          /* the reference indexes the array linearly */
    if (i < 0 || i >= (long)c->pu_w * c->pu_h) return 0;                   /* never reached by a legal stream (see DESIGN.md) */
    return (c->bits[i >> 5] >> (i & 31)) & 1;
}
/* IS_INTRA(x, y) (:37-40): x, y = sample offsets from the block origin, in samples of the block's plane */
static int cip_is_intra(const OrcCip *c, int x0, int y0, int x, int y)
{
    return cip_pu_intra(c, (x0 + x * (1 << c->hs)) >> c->log2_min_pu, (y0 + y * (1 << c->vs)) >> c->log2_min_pu);
}

/* :116-163 -- a neighbour stays a candidate only if one of its PUs (every second one is looked at) is intra */
static void orc_cip_flags(const B200IntraRec *r, const OrcCip *c, int *up_left, int *up, int *up_right, int *lft, int *bottom_left)
{
    const int n = 1 << r->log2, pu = c->log2_min_pu;
    const int x0 = r->x << c->hs, y0 = r->y << c->vs, sl_h = n << c->hs, sl_v = n << c->vs;
    const int pv = sl_v >> pu;
    int ph = sl_h >> pu;
    const int on_x = !(x0 & ((1 << pu) - 1)), on_y = !(y0 & ((1 << pu) - 1));
    if (!ph) ph++;                                                          /* only the horizontal count is bumped (:121-122) */
    if (*bottom_left && on_x) {
        const int xl = (x0 - 1) >> pu, yb = (y0 + sl_v) >> pu;
        int max = pv < c->pu_h - yb ? pv : c->pu_h - yb, any = 0;
        for (int i = 0; i < max; i += 2) any |= cip_pu_intra(c, xl, yb + i);
        *bottom_left = any;
    }
    if (*lft && on_x) {
        const int xl = (x0 - 1) >> pu, yl = y0 >> pu;
        int max = pv < c->pu_h - yl ? pv : c->pu_h - yl, any = 0;
        for (int i = 0; i < max; i += 2) any |= cip_pu_intra(c, xl, yl + i);
        *lft = any;
    }
    if (*up_left) *up_left = cip_pu_intra(c, (x0 - 1) >> pu, (y0 - 1) >> pu);
    if (*up && on_y) {
        const int xt = x0 >> pu, yt = (y0 - 1) >> pu;
        int max = ph < c->pu_w - xt ? ph : c->pu_w - xt, any = 0;
        for (int i = 0; i < max; i += 2) any |= cip_pu_intra(c, xt + i, yt);
        *up = any;
    }
    if (*up_right && on_y) {
        const int yt = (y0 - 1) >> pu, xr = (x0 + sl_h) >> pu;
        int max = ph < c->pu_w - xr ? ph : c->pu_w - xr, any = 0;
        for (int i = 0; i < max; i += 2) any |= cip_pu_intra(c, xr + i, yt);
        *up_right = any;
    }
}

static void put4(int *p, int v) { p[0] = p[1] = p[2] = p[3] = v; }         /* AV_WN4P of a splatted pixel */

/* :185-249 -- runs after the candidate samples were copied: samples of inter-coded neighbours are replaced by
 * propagating the nearest intra-coded ones, in groups of four like the reference's 4-pixel stores */
static void orc_cip_substitute(const B200IntraRec *r, const OrcCip *c, int *left, int *top,
                               int up_left, int up, int up_right, int lft, int bottom_left)
{
    if (!(bottom_left || lft || up_left || up || up_right)) return;
    const int n = 1 << r->log2;
    const int x0 = r->x << c->hs, y0 = r->y << c->vs;
#define ISI(x, y) cip_is_intra(c, x0, y0, (x), (y))
    int smx = x0 + ((2 * n) << c->hs) < c->pic_w ? 2 * n : (c->pic_w - x0) >> c->hs;
    int smy = y0 + ((2 * n) << c->vs) < c->pic_h ? 2 * n : (c->pic_h - y0) >> c->vs;
    int j = n + (bottom_left ? r->bottom_left_size : 0) - 1, i, a;
    if (!up_right)    smx = x0 + (n << c->hs) < c->pic_w ? n : (c->pic_w - x0) >> c->hs;
    if (!bottom_left) smy = y0 + (n << c->vs) < c->pic_h ? n : (c->pic_h - y0) >> c->vs;
    if (bottom_left || lft || up_left) {
        while (j > -1 && !ISI(-1, j)) j--;                                  /* lowest intra sample of the left column */
        if (!ISI(-1, j)) {                                                   /* none, not even the corner: take the first intra sample of the top row */
            j = 0;
            while (j < smx && !ISI(j, -1)) j++;
            for (i = j; i > -1; i--) if (!ISI(i - 1, -1)) top[i - 1] = top[i];      /* EXTEND_LEFT_CIP(top, j, j + 1) */
            left[-1] = top[-1];
        }
    } else {
        j = 0;
        while (j < smx && !ISI(j, -1)) j++;
        if (j > 0) {
            if (x0 > 0) { for (i = j; i > -1; i--) if (!ISI(i - 1, -1)) top[i - 1] = top[i]; }
            else { for (i = j; i > 0; i--) if (!ISI(i - 1, -1)) top[i - 1] = top[i]; top[-1] = top[0]; }
        }
        left[-1] = top[-1];
    }
    left[-1] = top[-1];
    if (bottom_left || lft) {                                                /* EXTEND_DOWN_CIP(left, 0, smy) */
        a = left[-1];
        for (i = 0; i < smy; i += 4) { if (!ISI(-1, i)) put4(left + i, a); else a = left[i + 3]; }
    }
    if (!lft) for (i = 0; i < n; i += 4) put4(left + i, left[-1]);
    if (!bottom_left) { const int v = left[n - 1]; for (i = 0; i < n; i += 4) put4(left + n + i, v); }
    if (x0 != 0 && y0 != 0) {
        a = left[smy - 1];
        for (i = smy - 1; i > -1; i -= 4) { if (!ISI(-1, i - 3)) put4(left + i - 3, a); else a = left[i - 3]; }   /* EXTEND_UP_CIP */
        if (!ISI(-1, -1)) left[-1] = left[0];
    } else if (x0 == 0) {
        for (i = 0; i < smy; i += 4) put4(left + i, 0);
    } else {
        a = left[smy - 1];
        for (i = smy - 1; i > -1; i -= 4) { if (!ISI(-1, i - 3)) put4(left + i - 3, a); else a = left[i - 3]; }
    }
    top[-1] = left[-1];
    if (y0 != 0) {                                                           /* EXTEND_RIGHT_CIP(top, 0, smx) */
        a = left[-1];
        for (i = 0; i < smx; i += 4) { if (!ISI(i, -1)) put4(top + i, a); else a = top[i + 3]; }
    }
#undef ISI
}

static const int8_t k_intra_angle[33] = { 32, 26, 21, 17, 13, 9, 5, 2, 0, -2, -5, -9, -13, -17, -21, -26, -32,
                                          -26, -21, -17, -13, -9, -5, -2, 0, 2, 5, 9, 13, 17, 21, 26, 32 };
static const int16_t k_inv_angle[15] = { -4096, -1638, -910, -630, -482, -390, -315, -256, -315, -390, -482, -630, -910, -1638, -4096 };

static void orc_intra_rec_cip(const B200IntraRec *r, pix_t *plane, int stride, int bd, const OrcCip *cip);
void orc_intra_rec(const B200IntraRec *r, pix_t *plane, int stride, int bd) { orc_intra_rec_cip(r, plane, stride, bd, NULL); }

static void orc_intra_rec_cip(const B200IntraRec *r, pix_t *plane, int stride, int bd, const OrcCip *cip)
{
    const int n = 1 << r->log2, n2 = 2 * n;
    pix_t *src = plane + r->y * stride + r->x;
    int lbuf[2][8 + 65 + 8], tbuf[2][8 + 65 + 8];          /* index 8 holds [-1]; slack for the 4-sample stores of the CIP rules */
    int *left = lbuf[0] + 9, *top = tbuf[0] + 9;
    int up_left = !!(r->flags & B200_INF_UP_LEFT), up = !!(r->flags & B200_INF_UP), up_right = !!(r->flags & B200_INF_UP_RIGHT);
    int lft = !!(r->flags & B200_INF_LEFT), bottom_left = !!(r->flags & B200_INF_BOTTOM_LEFT);
    int i;
    for (i = -1; i < n2; i++) left[i] = top[i] = 0;
    if (cip) {
        /* :116-163, then memset(left / top, 128, ...) of `pixel`s (:159-161): 0x80 or 0x8080 per sample, top[-1] = 128 */
        orc_cip_flags(r, cip, &up_left, &up, &up_right, &lft, &bottom_left);
        for (i = 0; i < 64; i++) left[i] = top[i] = bd > 8 ? 0x8080 : 0x80;
        left[-1] = top[-1] = 128;
    }

    /* gather what exists (:164-183) */
    if (up_left) left[-1] = top[-1] = src[-stride - 1];
    if (up) for (i = 0; i < n; i++) top[i] = src[-stride + i];
    if (up_right) {
        for (i = 0; i < r->top_right_size; i++) top[n + i] = src[-stride + n + i];
        for (; i < n; i++) top[n + i] = src[-stride + n + r->top_right_size - 1];
    }
    if (lft) for (i = 0; i < n; i++) left[i] = src[i * stride - 1];
    if (bottom_left) {
        for (i = 0; i < r->bottom_left_size; i++) left[n + i] = src[(n + i) * stride - 1];
        for (; i < n; i++) left[n + i] = src[(n + r->bottom_left_size - 1) * stride - 1];
    }
    if (cip) orc_cip_substitute(r, cip, left, top, up_left, up, up_right, lft, bottom_left);
    /* substitution chain (:250-286) */
    if (!bottom_left) {
        if (lft) { for (i = 0; i < n; i++) left[n + i] = left[n - 1]; }
        else if (up_left) { for (i = 0; i < n2; i++) left[i] = left[-1]; lft = 1; }
        else if (up) { left[-1] = top[0]; for (i = 0; i < n2; i++) left[i] = left[-1]; up_left = lft = 1; }
        else if (up_right) {
            for (i = 0; i < n; i++) top[i] = top[n];
            left[-1] = top[n];
            for (i = 0; i < n2; i++) left[i] = left[-1];
            up = up_left = lft = 1;
        } else {
            left[-1] = 1 << (bd - 1);
            for (i = 0; i < n2; i++) top[i] = left[i] = left[-1];
        }
    }
    if (!lft) for (i = 0; i < n; i++) left[i] = left[n];
    if (!up_left) left[-1] = left[0];
    if (!up) for (i = 0; i < n; i++) top[i] = left[-1];
    if (!up_right) for (i = 0; i < n; i++) top[n + i] = top[n - 1];
    top[-1] = left[-1];

    /* smoothing (:288-327) */
    const int mode = r->mode;
    if ((r->flags & B200_INF_FILTER) && mode != 1 && n != 4) {
        static const int thresh[3] = { 7, 1, 0 };
        int d26 = iabs(mode - 26), d10 = iabs(mode - 10), dist = d26 < d10 ? d26 : d10;
        if (dist > thresh[r->log2 - 3]) {
            int *fl = lbuf[1] + 9, *ft = tbuf[1] + 9;
            if ((r->flags & B200_INF_STRONG) && r->plane == 0 && r->log2 == 5 &&
                iabs(top[-1] + top[63] - 2 * top[31]) < (1 << (bd - 5)) &&
                iabs(left[-1] + left[63] - 2 * left[31]) < (1 << (bd - 5))) {
                ft[-1] = top[-1]; ft[63] = top[63]; fl[-1] = left[-1]; fl[63] = left[63];
                for (i = 0; i < 63; i++) {
                    ft[i] = ((63 - i) * top[-1] + (i + 1) * top[63] + 32) >> 6;
                    fl[i] = ((63 - i) * left[-1] + (i + 1) * left[63] + 32) >> 6;
                }
            } else {
                fl[n2 - 1] = left[n2 - 1]; ft[n2 - 1] = top[n2 - 1];
                for (i = n2 - 2; i >= 0; i--) {
                    fl[i] = (left[i + 1] + 2 * left[i] + left[i - 1] + 2) >> 2;
                    ft[i] = (top[i + 1] + 2 * top[i] + top[i - 1] + 2) >> 2;
                }
                ft[-1] = fl[-1] = (left[0] + 2 * left[-1] + top[0] + 2) >> 2;
            }
            left = fl; top = ft;
        }
    }

    if (mode == 0) {                                    /* planar :359-371 */
        for (int y = 0; y < n; y++)
            for (int x = 0; x < n; x++)
                src[y * stride + x] = (pix_t)(((n - 1 - x) * left[y] + (x + 1) * top[n] + (n - 1 - y) * top[x] + (y + 1) * left[n] + n) >> (r->log2 + 1));
    } else if (mode == 1) {                             /* DC :388-417 */
        int dc = n;
        for (i = 0; i < n; i++) dc += left[i] + top[i];
        dc >>= r->log2 + 1;
        for (int y = 0; y < n; y++) for (int x = 0; x < n; x++) src[y * stride + x] = (pix_t)dc;
        if (r->plane == 0 && n < 32) {
            src[0] = (pix_t)((left[0] + 2 * dc + top[0] + 2) >> 2);
            for (int x = 1; x < n; x++) src[x] = (pix_t)((top[x] + 3 * dc + 2) >> 2);
            for (int y = 1; y < n; y++) src[y * stride] = (pix_t)((left[y] + 3 * dc + 2) >> 2);
        }
    } else {                                            /* angular :419-510 */
        const int angle = k_intra_angle[mode - 2], last = (n * angle) >> 5;
        const int vertical = mode >= 18;
        const int *mainr = vertical ? top : left, *side = vertical ? left : top;
        int refbuf[3 * 32 + 4], *ref = refbuf + 32;     /* ref[k] == main[k-1] */
        for (i = 0; i <= n2; i++) ref[i] = mainr[i - 1];
        if (angle < 0 && last < -1)
            for (i = last; i <= -1; i++) ref[i] = side[-1 + ((i * k_inv_angle[mode - 11] + 128) >> 8)];
        for (int a = 0; a < n; a++) {                   /* a runs along the prediction direction */
            const int idx = ((a + 1) * angle) >> 5, fact = ((a + 1) * angle) & 31;
            for (int b = 0; b < n; b++) {
                int v = fact ? ((32 - fact) * ref[b + idx + 1] + fact * ref[b + idx + 2] + 16) >> 5 : ref[b + idx + 1];
                if (vertical) src[a * stride + b] = (pix_t)v; else src[b * stride + a] = (pix_t)v;
            }
        }
        if (r->plane == 0 && n < 32) {
            if (mode == 26) for (int y = 0; y < n; y++) src[y * stride] = (pix_t)clip_pix(top[0] + ((left[y] - left[-1]) >> 1), bd);
            if (mode == 10) for (int x = 0; x < n; x++) src[x] = (pix_t)clip_pix(left[0] + ((top[x] - top[-1]) >> 1), bd);
        }
    }
}

/* ------------------------------------------------------------------------------------------
 * Deblocking.  Reference: hevcdsp_template.c:1629-1723 (luma), :1725-1755 (chroma).
 * One call of the table function covers two 4-line segments; here one segment at a time.
 * xs = step across the edge, ys = step along it.
 * ---------------------------------------------------------------------------------------- */
void orc_deblock_luma_seg(pix_t *pix, int xs, int ys, int beta8, int tc8, int no_p, int no_q, int bd)
{
    const int beta = beta8 << (bd - 8), tc = tc8 << (bd - 8);
#define PX(i, l) ((int)pix[(i) * xs + (l) * ys])
    const int dp0 = iabs(PX(-3, 0) - 2 * PX(-2, 0) + PX(-1, 0)), dq0 = iabs(PX(2, 0) - 2 * PX(1, 0) + PX(0, 0));
    const int dp3 = iabs(PX(-3, 3) - 2 * PX(-2, 3) + PX(-1, 3)), dq3 = iabs(PX(2, 3) - 2 * PX(1, 3) + PX(0, 3));
    const int d0 = dp0 + dq0, d3 = dp3 + dq3;
    if (d0 + d3 >= beta) return;
    const int tc25 = (tc * 5 + 1) >> 1;
    const int strong = iabs(PX(-4, 0) - PX(-1, 0)) + iabs(PX(3, 0) - PX(0, 0)) < (beta >> 3) && iabs(PX(-1, 0) - PX(0, 0)) < tc25 &&
                       iabs(PX(-4, 3) - PX(-1, 3)) + iabs(PX(3, 3) - PX(0, 3)) < (beta >> 3) && iabs(PX(-1, 3) - PX(0, 3)) < tc25 &&
                       (d0 << 1) < (beta >> 2) && (d3 << 1) < (beta >> 2);
    const int nd_p = dp0 + dp3 < ((beta + (beta >> 1)) >> 3), nd_q = dq0 + dq3 < ((beta + (beta >> 1)) >> 3);
    for (int l = 0; l < 4; l++) {
        const int p3 = PX(-4, l), p2 = PX(-3, l), p1 = PX(-2, l), p0 = PX(-1, l);
        const int q0 = PX(0, l), q1 = PX(1, l), q2 = PX(2, l), q3 = PX(3, l);
        pix_t *p = pix + l * ys;
        if (strong) {
            const int t2 = tc << 1;
            if (!no_p) {
                p[-1 * xs] = (pix_t)(p0 + clip3(((p2 + 2 * p1 + 2 * p0 + 2 * q0 + q1 + 4) >> 3) - p0, -t2, t2));
                p[-2 * xs] = (pix_t)(p1 + clip3(((p2 + p1 + p0 + q0 + 2) >> 2) - p1, -t2, t2));
                p[-3 * xs] = (pix_t)(p2 + clip3(((2 * p3 + 3 * p2 + p1 + p0 + q0 + 4) >> 3) - p2, -t2, t2));
            }
            if (!no_q) {
                p[0]      = (pix_t)(q0 + clip3(((p1 + 2 * p0 + 2 * q0 + 2 * q1 + q2 + 4) >> 3) - q0, -t2, t2));
                p[xs]     = (pix_t)(q1 + clip3(((p0 + q0 + q1 + q2 + 2) >> 2) - q1, -t2, t2));
                p[2 * xs] = (pix_t)(q2 + clip3(((2 * q3 + 3 * q2 + q1 + q0 + p0 + 4) >> 3) - q2, -t2, t2));
            }
        } else {
            int delta = (9 * (q0 - p0) - 3 * (q1 - p1) + 8) >> 4;
            if (iabs(delta) < 10 * tc) {
                const int th = tc >> 1;
                delta = clip3(delta, -tc, tc);
                if (!no_p) p[-1 * xs] = (pix_t)clip_pix(p0 + delta, bd);
                if (!no_q) p[0]       = (pix_t)clip_pix(q0 - delta, bd);
                if (!no_p && nd_p) p[-2 * xs] = (pix_t)clip_pix(p1 + clip3((((p2 + p0 + 1) >> 1) - p1 + delta) >> 1, -th, th), bd);
                if (!no_q && nd_q) p[xs]      = (pix_t)clip_pix(q1 + clip3((((q2 + q0 + 1) >> 1) - q1 - delta) >> 1, -th, th), bd);
            }
        }
    }
#undef PX
}

void orc_deblock_chroma_seg(pix_t *pix, int xs, int ys, int tc8, int no_p, int no_q, int bd)
{
    const int tc = tc8 << (bd - 8);
    if (tc <= 0) return;
    for (int l = 0; l < 4; l++) {
        pix_t *p = pix + l * ys;
        const int p1 = p[-2 * xs], p0 = p[-xs], q0 = p[0], q1 = p[xs];
        const int delta = clip3((((q0 - p0) * 4) + p1 - q1 + 4) >> 3, -tc, tc);
        if (!no_p) p[-xs] = (pix_t)clip_pix(p0 + delta, bd);
        if (!no_q) p[0]   = (pix_t)clip_pix(q0 - delta, bd);
    }
}

/* whole-picture deblocking of one plane: every vertical edge, then every horizontal edge
 * (the semantic order; the reference's CTB-staggered schedule hevc_filter.c:1027-1064 is equivalent) */
static void deblock_plane(pix_t *pl, int pw, int ph, int plane, const uint16_t *grid, const B200DbkLayout *L, int bd)
{
    for (int dir = 0; dir < 2; dir++) {
        const uint16_t *g = grid + L->off[plane][dir];
        const int gs = (int)L->stride[plane][dir];
        if (dir == 0) {
            for (int y = 0; y + 4 <= ph; y += 4)
                for (int x = 8; x < pw; x += 8) {
                    uint16_t e = g[(y >> 2) * gs + (x >> 3)];
                    if (!(e & B200_DBK_PRESENT)) continue;
                    if (plane == 0) orc_deblock_luma_seg(pl + y * pw + x, 1, pw, B200_DBK_BETA(e), B200_DBK_TC(e), B200_DBK_NOP(e), B200_DBK_NOQ(e), bd);
                    else            orc_deblock_chroma_seg(pl + y * pw + x, 1, pw, B200_DBK_TC(e), B200_DBK_NOP(e), B200_DBK_NOQ(e), bd);
                }
        } else {
            for (int y = 8; y < ph; y += 8)
                for (int x = 0; x + 4 <= pw; x += 4) {
                    uint16_t e = g[(y >> 3) * gs + (x >> 2)];
                    if (!(e & B200_DBK_PRESENT)) continue;
                    if (plane == 0) orc_deblock_luma_seg(pl + y * pw + x, pw, 1, B200_DBK_BETA(e), B200_DBK_TC(e), B200_DBK_NOP(e), B200_DBK_NOQ(e), bd);
                    else            orc_deblock_chroma_seg(pl + y * pw + x, pw, 1, B200_DBK_TC(e), B200_DBK_NOP(e), B200_DBK_NOQ(e), bd);
                }
        }
    }
}

/* ------------------------------------------------------------------------------------------
 * Deblocking parameters derived from the picture's records (SURVEY.md 8f N2; product: openhevc_b200/csrc/k_dbd.cuh).
 * Restates, in the reference's own order, what the reference computes on the host:
 *   the motion field and cbf_luma as the parse leaves them        hevc.c:1568-1576 (cbf), hevc.c hls_prediction_unit (tab_mvf)
 *   ff_hevc_deblocking_boundary_strengths()                       hevc_filter.c:805-941, boundary_strength() :583-700
 *   deblocking_filter_CTB(), CTB by CTB, its filter calls written into the grids the way the recorder writes the
 *   reference's real calls (b200_rec_deblock)                     hevc_filter.c:345-581
 * ---------------------------------------------------------------------------------------- */
typedef struct OrcMvf { int16_t mx[2], my[2]; int ref[2]; int pred; } OrcMvf;     /* pred: 0 intra, 1 one motion vector (index 0), 3 two */
typedef struct OrcDbd {
    const B200BlobHeader *h; const B200DbdHeader *d; const uint8_t *sec;
    int uw, uh; OrcMvf *mvf; uint8_t *cbf, *vbs, *hbs;
    uint16_t *grid; B200DbkLayout L;
} OrcDbd;
static int orc_far(int ax, int ay, int bx, int by) { return abs(ax - bx) >= 4 || abs(ay - by) >= 4; }
static int orc_boundary_strength(const OrcMvf *c, const OrcMvf *n)
{
    if (c->pred == 3 && n->pred == 3) {
        if (c->ref[0] == n->ref[0] && c->ref[0] == c->ref[1] && n->ref[0] == n->ref[1])
            return (orc_far(n->mx[0], n->my[0], c->mx[0], c->my[0]) || orc_far(n->mx[1], n->my[1], c->mx[1], c->my[1])) &&
                   (orc_far(n->mx[1], n->my[1], c->mx[0], c->my[0]) || orc_far(n->mx[0], n->my[0], c->mx[1], c->my[1]));
        if (n->ref[0] == c->ref[0] && n->ref[1] == c->ref[1])
            return orc_far(n->mx[0], n->my[0], c->mx[0], c->my[0]) || orc_far(n->mx[1], n->my[1], c->mx[1], c->my[1]);
        if (n->ref[1] == c->ref[0] && n->ref[0] == c->ref[1])
            return orc_far(n->mx[1], n->my[1], c->mx[0], c->my[0]) || orc_far(n->mx[0], n->my[0], c->mx[1], c->my[1]);
        return 1;
    }
    if (c->pred != 3 && n->pred != 3) return c->ref[0] == n->ref[0] ? orc_far(c->mx[0], c->my[0], n->mx[0], n->my[0]) : 1;
    return 1;
}
static const OrcMvf *orc_mvf_at(const OrcDbd *o, int x, int y) { return &o->mvf[(y >> 2) * o->uw + (x >> 2)]; }
static int orc_bs_tu_edge(const OrcDbd *o, int xc, int yc, int xn, int yn)
{
    const OrcMvf *c = orc_mvf_at(o, xc, yc), *n = orc_mvf_at(o, xn, yn);
    if (!c->pred || !n->pred) return 2;
    if (o->cbf[(yc >> 2) * o->uw + (xc >> 2)] || o->cbf[(yn >> 2) * o->uw + (xn >> 2)]) return 1;
    return orc_boundary_strength(c, n);
}
static void orc_bs_leaf(OrcDbd *o, uint32_t leaf)
{
    const int x0 = (int)(leaf & 0xfff) << 2, y0 = (int)((leaf >> 12) & 0xfff) << 2, log2 = (int)((leaf >> 24) & 7) + 2, size = 1 << log2;
    const int W = o->h->width, H = o->h->height;
    if (x0 >= W || y0 >= H) return;
    if ((leaf >> 28) & 1)
        for (int i = 0; i < size && x0 + i < W; i += 4) o->hbs[(y0 >> 2) * o->uw + ((x0 + i) >> 2)] = (uint8_t)orc_bs_tu_edge(o, x0 + i, y0, x0 + i, y0 - 1);
    if ((leaf >> 29) & 1)
        for (int i = 0; i < size && y0 + i < H; i += 4) o->vbs[((y0 + i) >> 2) * o->uw + (x0 >> 2)] = (uint8_t)orc_bs_tu_edge(o, x0, y0 + i, x0 - 1, y0 + i);
    if (log2 > (int)o->d->log2_min_pu_size && orc_mvf_at(o, x0, y0)->pred) {
        for (int i = 0; i < size && x0 + i < W; i += 4) {             /* :906-922, the running `top` */
            const OrcMvf *top = orc_mvf_at(o, x0 + i, y0 + 8 - 1);
            for (int j = 8; j < size && y0 + j < H; j += 8) {
                const OrcMvf *curr = orc_mvf_at(o, x0 + i, y0 + j);
                o->hbs[((y0 + j) >> 2) * o->uw + ((x0 + i) >> 2)] = (uint8_t)((curr->pred && top->pred) ? orc_boundary_strength(curr, top) : 1);
                top = curr;
            }
        }
        for (int j = 0; j < size && y0 + j < H; j += 4) {             /* :924-940 */
            const OrcMvf *left = orc_mvf_at(o, x0 + 8 - 1, y0 + j);
            for (int i = 8; i < size && x0 + i < W; i += 8) {
                const OrcMvf *curr = orc_mvf_at(o, x0 + i, y0 + j);
                o->vbs[((y0 + j) >> 2) * o->uw + ((x0 + i) >> 2)] = (uint8_t)((curr->pred && left->pred) ? orc_boundary_strength(curr, left) : 1);
                left = curr;
            }
        }
    }
}
static const uint8_t orc_tctable[54] = { 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4,
                                         5, 5, 6, 6, 7, 8, 9, 10, 11, 13, 14, 16, 18, 20, 22, 24 };
static const uint8_t orc_betatable[52] = { 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 20, 22, 24, 26, 28, 30, 32, 34, 36,
                                           38, 40, 42, 44, 46, 48, 50, 52, 54, 56, 58, 60, 62, 64 };
static int orc_qpy(const OrcDbd *o, int x, int y)
{
    const int8_t *qp = (const int8_t *)(o->sec + o->d->off_qp);
    int xc = x >> o->d->log2_min_cb_size, yc = y >> o->d->log2_min_cb_size;
    if (yc >= (int)o->d->min_cb_height) yc = (int)o->d->min_cb_height - 1;      /* (the reference reads past the table there; the value is never used) */
    if (xc >= (int)o->d->min_cb_width) xc = (int)o->d->min_cb_width - 1;
    return qp[xc + yc * (int)o->d->min_cb_width];
}
static int orc_get_pcm(const OrcDbd *o, int x, int y)
{
    if (x < 0 || y < 0) return 2;
    const int xp = x >> o->d->log2_min_pu_size, yp = y >> o->d->log2_min_pu_size;
    if (xp >= (int)o->d->min_pu_width || yp >= (int)o->d->min_pu_height) return 2;
    return o->sec[o->d->off_pcm + yp * o->d->min_pu_width + xp];
}
static int orc_chroma_tc(const OrcDbd *o, int qp_y, int c_idx, int tc_offset)
{
    static const int qp_c[] = { 29, 30, 31, 32, 33, 33, 34, 34, 35, 35, 36, 36, 37, 37 };
    const int qp_i = clip3(qp_y + (c_idx == 1 ? o->d->cb_qp_offset : o->d->cr_qp_offset), 0, 57);
    int qp;
    if (o->h->chroma_format_idc == 1) qp = qp_i < 30 ? qp_i : qp_i > 43 ? qp_i - 6 : qp_c[qp_i - 30];
    else qp = clip3(qp_i, 0, 51);
    return orc_tctable[clip3(qp + 2 + tc_offset, 0, 53)];
}
#define ORC_TC_CALC(qp, bs) orc_tctable[clip3((qp) + 2 * ((bs) - 1) + (tc_offset >> 1 << 1), 0, 53)]
/* one filter call of the reference, as the recorder writes it (recorder.cpp b200_rec_deblock) */
static void orc_dbk_call(OrcDbd *o, int plane, int vertical, int x, int y, int beta, const int tc[2], const int no_p[2], const int no_q[2])
{
    int pw, ph;
    b200_plane_dims(o->h->width, o->h->height, o->h->chroma_format_idc, plane, &pw, &ph);
    uint16_t *g = o->grid + o->L.off[plane][vertical ? 0 : 1];
    const int gs = (int)o->L.stride[plane][vertical ? 0 : 1];
    for (int j = 0; j < 2; j++) {
        const int sx = vertical ? x : x + 4 * j, sy = vertical ? y + 4 * j : y;
        if (sx >= pw || sy >= ph) continue;
        g[vertical ? (sy >> 2) * gs + (sx >> 3) : (sy >> 3) * gs + (sx >> 2)] = B200_DBK_PACK(tc[j], plane ? 0 : beta, no_p[j] != 0, no_q[j] != 0);
    }
}
static void orc_deblocking_filter_ctb(OrcDbd *o, int x0, int y0)          /* hevc_filter.c:345-581 */
{
    const int W = o->h->width, H = o->h->height, log2_ctb = o->h->log2_ctb_size, ctb_size = 1 << log2_ctb;
    const int ctb_w = (W + ctb_size - 1) >> log2_ctb;
    const int ctb = (x0 >> log2_ctb) + (y0 >> log2_ctb) * ctb_w;
    const int8_t *off = (const int8_t *)(o->sec + o->d->off_ctb);
    const int cur_tc_offset = off[2 * ctb + 1], cur_beta_offset = off[2 * ctb];
    const int left_tc_offset = x0 ? off[2 * (ctb - 1) + 1] : 0, left_beta_offset = x0 ? off[2 * (ctb - 1)] : 0;
    const int pcmf = (o->d->flags & B200_DBDF_PCM) != 0;
    const int cfi = o->h->chroma_format_idc, hs = cfi != 3, vs = cfi == 1;
    int x_end = x0 + ctb_size > W ? W : x0 + ctb_size, y_end = y0 + ctb_size > H ? H : y0 + ctb_size;
    int tc_offset = cur_tc_offset, beta_offset = cur_beta_offset;
    int tc[2], c_tc[2], c_tc2[2], no_p[2] = { 0, 0 }, no_q[2] = { 0, 0 };
#define VBS(x, y) ((y) < H && (x) < W ? o->vbs[((y) >> 2) * o->uw + ((x) >> 2)] : 0)
#define HBS(x, y) ((y) < H && (x) < W ? o->hbs[((y) >> 2) * o->uw + ((x) >> 2)] : 0)
    for (int y = y0; y < y_end; y += 8)                                   /* vertical edges, luma */
        for (int x = x0 ? x0 : 8; x < x_end; x += 8) {
            const int bs0 = VBS(x, y), bs1 = VBS(x, y + 4);
            if (!bs0 && !bs1) continue;
            const int qp = (orc_qpy(o, x - 1, y) + orc_qpy(o, x, y) + 1) >> 1;
            const int beta = orc_betatable[clip3(qp + beta_offset, 0, 51)];
            tc[0] = bs0 ? ORC_TC_CALC(qp, bs0) : 0; tc[1] = bs1 ? ORC_TC_CALC(qp, bs1) : 0;
            if (pcmf) { no_p[0] = orc_get_pcm(o, x - 1, y); no_p[1] = orc_get_pcm(o, x - 1, y + 4); no_q[0] = orc_get_pcm(o, x, y); no_q[1] = orc_get_pcm(o, x, y + 4); }
            orc_dbk_call(o, 0, 1, x, y, beta, tc, no_p, no_q);
        }
    if (cfi) {                                                            /* vertical edges, chroma */
        const int h = 1 << hs, v = 1 << vs;
        for (int y = y0; y < y_end; y += 8 * v)
            for (int x = x0 ? x0 : 8 * h; x < x_end; x += 8 * h) {
                const int bs0 = VBS(x, y), bs1 = VBS(x, y + 4 * v);
                if (bs0 != 2 && bs1 != 2) continue;
                const int qp0 = (orc_qpy(o, x - 1, y) + orc_qpy(o, x, y) + 1) >> 1, qp1 = (orc_qpy(o, x - 1, y + 4 * v) + orc_qpy(o, x, y + 4 * v) + 1) >> 1;
                c_tc[0] = bs0 == 2 ? orc_chroma_tc(o, qp0, 1, tc_offset) : 0; c_tc[1] = bs1 == 2 ? orc_chroma_tc(o, qp1, 1, tc_offset) : 0;
                c_tc2[0] = bs0 == 2 ? orc_chroma_tc(o, qp0, 2, tc_offset) : 0; c_tc2[1] = bs1 == 2 ? orc_chroma_tc(o, qp1, 2, tc_offset) : 0;
                if (pcmf) { no_p[0] = orc_get_pcm(o, x - 1, y); no_p[1] = orc_get_pcm(o, x - 1, y + 4 * v); no_q[0] = orc_get_pcm(o, x, y); no_q[1] = orc_get_pcm(o, x, y + 4 * v); }
                orc_dbk_call(o, 1, 1, x >> hs, y >> vs, 0, c_tc, no_p, no_q);
                orc_dbk_call(o, 2, 1, x >> hs, y >> vs, 0, c_tc2, no_p, no_q);
            }
    }
    const int x_end2 = x_end;                                             /* horizontal edges, luma */
    if (x_end != W) x_end -= 8;
    for (int y = y0 ? y0 : 8; y < y_end; y += 8) {
        beta_offset = x0 ? left_beta_offset : cur_beta_offset;
        for (int x = x0 ? x0 - 8 : 0; x < x_end; x += 8) {
            const int bs0 = HBS(x, y), bs1 = HBS(x + 4, y);
            if (bs0 || bs1) {
                const int qp = (orc_qpy(o, x, y - 1) + orc_qpy(o, x, y) + 1) >> 1;
                const int beta = orc_betatable[clip3(qp + beta_offset, 0, 51)];
                tc[0] = bs0 ? ORC_TC_CALC(qp, bs0) : 0; tc[1] = bs1 ? ORC_TC_CALC(qp, bs1) : 0;
                if (pcmf) { no_p[0] = orc_get_pcm(o, x, y - 1); no_p[1] = orc_get_pcm(o, x + 4, y - 1); no_q[0] = orc_get_pcm(o, x, y); no_q[1] = orc_get_pcm(o, x + 4, y); }
                orc_dbk_call(o, 0, 0, x, y, beta, tc, no_p, no_q);
            }
            beta_offset = cur_beta_offset;
        }
    }
    if (cfi) {                                                            /* horizontal edges, chroma */
        const int h = 1 << hs, v = 1 << vs;
        if (x_end2 != W) x_end = x_end2 - 8 * h;
        for (int y = y0 ? y0 : 8 * v; y < y_end; y += 8 * v) {
            tc_offset = x0 ? left_tc_offset : cur_tc_offset;
            for (int x = x0 ? x0 - 8 * h : 0; x < x_end; x += 8 * h) {
                const int bs0 = HBS(x, y), bs1 = HBS(x + 4 * h, y);
                if (bs0 == 2 || bs1 == 2) {
                    const int qp0 = bs0 == 2 ? (orc_qpy(o, x, y - 1) + orc_qpy(o, x, y) + 1) >> 1 : 0;
                    const int qp1 = bs1 == 2 ? (orc_qpy(o, x + 4 * h, y - 1) + orc_qpy(o, x + 4 * h, y) + 1) >> 1 : 0;
                    c_tc[0] = bs0 == 2 ? orc_chroma_tc(o, qp0, 1, tc_offset) : 0; c_tc[1] = bs1 == 2 ? orc_chroma_tc(o, qp1, 1, cur_tc_offset) : 0;
                    c_tc2[0] = bs0 == 2 ? orc_chroma_tc(o, qp0, 2, tc_offset) : 0; c_tc2[1] = bs1 == 2 ? orc_chroma_tc(o, qp1, 2, cur_tc_offset) : 0;
                    if (pcmf) { no_p[0] = orc_get_pcm(o, x, y - 1); no_p[1] = orc_get_pcm(o, x + 4 * h, y - 1); no_q[0] = orc_get_pcm(o, x, y); no_q[1] = orc_get_pcm(o, x + 4 * h, y); }
                    orc_dbk_call(o, 1, 0, x >> hs, y >> vs, 0, c_tc, no_p, no_q);
                    orc_dbk_call(o, 2, 0, x >> hs, y >> vs, 0, c_tc2, no_p, no_q);
                }
                tc_offset = cur_tc_offset;
            }
        }
    }
#undef VBS
#undef HBS
}
/* grid (b200_dbk_layout, zero-filled by the caller) <- the picture's DBD section + MC / TU records */
int orc_dbd_derive(const uint8_t *blob, uint16_t *grid)
{
    const B200BlobHeader *h = (const B200BlobHeader *)blob;
    if (!h->dbd.count) return -1;
    OrcDbd o;
    memset(&o, 0, sizeof(o));
    o.h = h; o.sec = blob + h->dbd.off; o.d = (const B200DbdHeader *)o.sec; o.grid = grid;
    b200_dbk_layout(h->width, h->height, h->chroma_format_idc, &o.L);
    o.uw = h->width / 4; o.uh = h->height / 4;
    const size_t U = (size_t)o.uw * o.uh;
    o.mvf = (OrcMvf *)calloc(U, sizeof(OrcMvf)); o.cbf = (uint8_t *)calloc(U, 1); o.vbs = (uint8_t *)calloc(U, 1); o.hbs = (uint8_t *)calloc(U, 1);
    if (!o.mvf || !o.cbf || !o.vbs || !o.hbs) { free(o.mvf); free(o.cbf); free(o.vbs); free(o.hbs); return -3; }
    const B200McRec *mc = (const B200McRec *)(blob + h->sec[B200_SEC_MC].off);
    for (uint32_t i = 0; i < h->sec[B200_SEC_MC].count; i++) {           /* the motion field: what hls_prediction_unit left in tab_mvf */
        const B200McRec *m = &mc[i];
        if (m->plane) continue;
        OrcMvf v;
        memset(&v, 0, sizeof(v));
        v.pred = (m->flags & B200_MCF_BI) ? 3 : 1;
        v.mx[0] = (int16_t)(((m->sx0 - m->x) << 2) | (m->frac0 & 3)); v.my[0] = (int16_t)(((m->sy0 - m->y) << 2) | ((m->frac0 >> 4) & 3));
        v.ref[0] = h->ref_slot[m->ref0 & 15];
        if (v.pred == 3) {
            v.mx[1] = (int16_t)(((m->sx1 - m->x) << 2) | (m->frac1 & 3)); v.my[1] = (int16_t)(((m->sy1 - m->y) << 2) | ((m->frac1 >> 4) & 3));
            v.ref[1] = h->ref_slot[m->ref1 & 15];
        }
        for (int y = m->y; y < m->y + m->h && y < h->height; y += 4)
            for (int x = m->x; x < m->x + m->w && x < h->width; x += 4) o.mvf[(y >> 2) * o.uw + (x >> 2)] = v;
    }
    for (int s = B200_SEC_TU4; s <= B200_SEC_TU32; s++) {                /* cbf_luma, hevc.c:1568-1576 */
        const B200TuRec *tu = (const B200TuRec *)(blob + h->sec[s].off);
        const int n = 4 << (s - B200_SEC_TU4);
        for (uint32_t i = 0; i < h->sec[s].count; i++) {
            if (tu[i].plane || tu[i].kind == B200_TU_PCM) continue;
            for (int y = tu[i].y; y < tu[i].y + n && y < h->height; y += 4)
                for (int x = tu[i].x; x < tu[i].x + n && x < h->width; x += 4) o.cbf[(y >> 2) * o.uw + (x >> 2)] = 1;
        }
    }
    const uint32_t *leaf = (const uint32_t *)(o.sec + o.d->off_leaf);
    for (uint32_t i = 0; i < o.d->n_leaf; i++) orc_bs_leaf(&o, leaf[i]);
    const int ctb = 1 << h->log2_ctb_size;
    for (int y0 = 0; y0 < h->height; y0 += ctb)
        for (int x0 = 0; x0 < h->width; x0 += ctb) orc_deblocking_filter_ctb(&o, x0, y0);
    free(o.mvf); free(o.cbf); free(o.vbs); free(o.hbs);
    return 0;
}

/* ------------------------------------------------------------------------------------------
 * SAO.  Reference: hevcdsp_template.c:340-365 (band), :372-567 (edge + border / restore rules);
 * driver hevc_filter.c:197-322.  src = deblocked picture (never modified), dst = output.
 * ---------------------------------------------------------------------------------------- */
void orc_sao_ctb(const B200SaoRec *s, pix_t *dst, const pix_t *src, int stride, int x0, int y0, int w, int h, int bd)
{
    if (s->type == B200_SAO_BAND) {
        int tab[32] = { 0 };
        for (int k = 0; k < 4; k++) tab[(k + s->param) & 31] = s->offset_val[k + 1];
        for (int y = 0; y < h; y++)
            for (int x = 0; x < w; x++) {
                int v = src[(y0 + y) * stride + x0 + x];
                dst[(y0 + y) * stride + x0 + x] = (pix_t)clip_pix(v + tab[v >> (bd - 5)], bd);
            }
        return;
    }
    static const int8_t pos[4][2][2] = { { { -1, 0 }, { 1, 0 } }, { { 0, -1 }, { 0, 1 } }, { { -1, -1 }, { 1, 1 } }, { { 1, -1 }, { -1, 1 } } };
    static const uint8_t edge_idx[5] = { 1, 2, 0, 3, 4 };
    const int cls = s->param;
    const int bl = s->borders & 1, bt = (s->borders >> 1) & 1, br = (s->borders >> 2) & 1, bb = (s->borders >> 3) & 1;
    const int ve0 = s->edges & 1, ve1 = (s->edges >> 1) & 1, he0 = (s->edges >> 2) & 1, he1 = (s->edges >> 3) & 1;
    const int de0 = (s->edges >> 4) & 1, de1 = (s->edges >> 5) & 1, de2 = (s->edges >> 6) & 1, de3 = (s->edges >> 7) & 1;
    /* geometry after the border trimming of :433-471 */
    const int init_x = (cls != 1 && bl) ? 1 : 0, wid = (cls != 1 && br) ? w - 1 : w;
    const int hei = (cls != 0 && bb) ? h - 1 : h;
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const pix_t *c = src + (y0 + y) * stride + x0 + x;
            int v = *c, out;
            int zero_off = 0;                           /* picture-border lines: offset_val[0] (== 0) */
            if (cls != 1 && ((bl && x == 0) || (br && x == w - 1))) zero_off = 1;
            if (cls != 0 && ((bt && y == 0) || (bb && y == h - 1))) zero_off = 1;
            if (zero_off) out = clip_pix(v + s->offset_val[0], bd);
            else {
                int a = c[pos[cls][0][0] + pos[cls][0][1] * stride], b = c[pos[cls][1][0] + pos[cls][1][1] * stride];
                int d0 = (v > a) - (v < a), d1 = (v > b) - (v < b);
                out = clip_pix(v + s->offset_val[edge_idx[2 + d0 + d1]], bd);
            }
            if (s->variant) {                           /* :533-566 not-across-boundary restore */
                const int sul = !de0 && cls == 2 && !bl && !bt, sur = !de1 && cls == 3 && !bt && !br;   /* 2 = SAO_EO_135D, 3 = SAO_EO_45D */
                const int slr = !de2 && cls == 2 && !br && !bb, sll = !de3 && cls == 3 && !bl && !bb;
                int restore = 0;
                if (ve0 && cls != 1 && x == 0 && y >= sul && y < hei - sll) restore = 1;
                if (ve1 && cls != 1 && x == wid - 1 && y >= sur && y < hei - slr) restore = 1;
                if (he0 && cls != 0 && y == 0 && x >= init_x + sul && x < wid - sur) restore = 1;
                if (he1 && cls != 0 && y == hei - 1 && x >= init_x + sll && x < wid - slr) restore = 1;
                if (de0 && cls == 2 && x == 0 && y == 0) restore = 1;
                if (de1 && cls == 3 && x == wid - 1 && y == 0) restore = 1;
                if (de2 && cls == 2 && x == wid - 1 && y == hei - 1) restore = 1;
                if (de3 && cls == 3 && x == 0 && y == hei - 1) restore = 1;
                if (restore) out = v;
            }
            dst[(y0 + y) * stride + x0 + x] = (pix_t)out;
        }
}

/* restore_tqb_pixels (hevc_filter.c:163-193), called after the SAO of a CTB whose type is band or edge: PUs flagged in
 * is_pcm[] (PCM with pcm_loop_filter_disabled, cu_transquant_bypass) get their pre-SAO samples back.  Restated with the two
 * things the reference really does:
 *  - it is called with the LUMA origin of the CTB but the width / height of the CTB in the plane being filtered
 *    (hevc_filter.c:275,316), so for subsampled chroma only the PUs of the first half of the CTB are visited;
 *  - a row of a PU is copied with memcpy(.., min_pu_size >> hshift) -- a length in samples used as bytes, so for
 *    bit depths above 8 only the first half of each row comes back.
 * x0l, y0l: luma origin of the CTB; w, h: size of the CTB in this plane; B: bytes per sample. */
static void orc_restore_tqb(pix_t *dst, const pix_t *src, int stride, int x0l, int y0l, int w, int h, int hs, int vs, int B,
                            int log2_pu, int pu_w, const uint32_t *bits)
{
    const int pu = 1 << log2_pu;
    const int x_min = x0l >> log2_pu, y_min = y0l >> log2_pu, x_max = (x0l + w) >> log2_pu, y_max = (y0l + h) >> log2_pu;
    const int len_samples = (pu >> hs) / B;
    for (int y = y_min; y < y_max; y++)
        for (int x = x_min; x < x_max; x++) {
            const long i = (long)y * pu_w + x;
            if (!((bits[i >> 5] >> (i & 31)) & 1)) continue;
            const int px = (x << log2_pu) >> hs, py = (y << log2_pu) >> vs;
            for (int n = 0; n < (pu >> vs); n++)
                for (int k = 0; k < len_samples; k++) dst[(py + n) * stride + px + k] = src[(py + n) * stride + px + k];
        }
}

/* ------------------------------------------------------------------------------------------
 * Whole-picture executor: the CPU statement of what the GPU stages K1..K5 compute for one blob.
 * planes[slot*3 + c] = uint16 plane of DPB slot `slot`, stride = plane width.
 * Returns 0, or a negative number for a malformed blob.
 * ---------------------------------------------------------------------------------------- */
int orc_execute_blob(const uint8_t *blob, uint16_t **planes, int n_slots)
{
    const B200BlobHeader *h = (const B200BlobHeader *)blob;
    if (h->magic != B200_BLOB_MAGIC || h->version != B200_BLOB_VERSION) return -1;
    if (h->cur_slot >= n_slots) return -2;
    const int bd = h->bit_depth, cfi = h->chroma_format_idc;
    int pw[3], ph[3];
    for (int p = 0; p < 3; p++) b200_plane_dims(h->width, h->height, cfi, p, &pw[p], &ph[p]);
    pix_t **cur = planes + 3 * h->cur_slot;

    const int16_t *pool = (const int16_t *)(blob + h->sec[B200_SEC_COEFF].off);
    /* parked residuals (intra TUs): sized by a first pass over the PARK records */
    size_t park_len = 8;
    for (int s = B200_SEC_TU4; s <= B200_SEC_TU32; s++) {
        const B200TuRec *tu = (const B200TuRec *)(blob + h->sec[s].off);
        for (uint32_t i = 0; i < h->sec[s].count; i++)
            if (tu[i].flags & B200_TUF_PARK) {
                uint32_t po = 0;
                b200_tu_data(&tu[i], pool, &po);
                if ((size_t)po + (1u << (2 * tu[i].log2)) > park_len) park_len = (size_t)po + (1u << (2 * tu[i].log2));
            }
    }
    const B200CcpRec *ccp = (const B200CcpRec *)(blob + h->ccp.off);
    const uint32_t n_ccp = (h->flags & B200_FRAME_CCP) ? h->ccp.count : 0;
    for (uint32_t i = 0; i < n_ccp; i++) {
        const size_t nn = (size_t)1 << (2 * ccp[i].log2);
        if ((ccp[i].flags & B200_CCPF_TO_PARK) && ccp[i].off_out + nn > park_len) park_len = ccp[i].off_out + nn;
    }
    int16_t *parked = (int16_t *)calloc(park_len, sizeof(int16_t));
    if (!parked) return -3;

    /* K1 inter */
    const B200McRec *mc = (const B200McRec *)(blob + h->sec[B200_SEC_MC].off);
    for (uint32_t i = 0; i < h->sec[B200_SEC_MC].count; i++) {
        const B200McRec *m = &mc[i];
        const int i0 = m->ref0, i1 = (m->flags & B200_MCF_BI) ? m->ref1 : m->ref0;
        if (i0 >= h->n_ref || i1 >= h->n_ref || h->ref_slot[i0] >= n_slots || h->ref_slot[i1] >= n_slots) { free(parked); return -4; }
        const int p = m->plane;
        orc_mc_rec(m, cur[p], pw[p], planes[3 * h->ref_slot[i0] + p], planes[3 * h->ref_slot[i1] + p], pw[p], ph[p], bd);
    }
    /* K2 residual */
    for (int s = B200_SEC_TU4; s <= B200_SEC_TU32; s++) {
        const B200TuRec *tu = (const B200TuRec *)(blob + h->sec[s].off);
        for (uint32_t i = 0; i < h->sec[s].count; i++) {
            const B200TuRec *t = &tu[i];
            int16_t c[32 * 32];
            uint32_t po = 0;
            b200_tu_expand(t, b200_tu_data(t, pool, &po), c);
            const int n = 1 << t->log2, p = t->plane;
            if (t->kind == B200_TU_PCM) {
                for (int y = 0; y < n; y++) for (int x = 0; x < n; x++) cur[p][(t->y + y) * pw[p] + t->x + x] = (pix_t)c[y * n + x];
                continue;
            }
            tu_residual(t, c, bd);
            if (t->flags & B200_TUF_PARK) memcpy(parked + po, c, (size_t)n * n * sizeof(int16_t));
            else orc_add_residual(cur[p] + t->y * pw[p] + t->x, pw[p], c, n, bd);
        }
    }
    /* cross-component prediction (4:4:4 range extension): chroma residual = own residual + (res_scale_val * luma residual) >> 3,
     * in int16 like the reference's coefficient arrays (hevc.c:1325-1327, 1358-1360, hevc_cabac.c:1942-1948), then
     * transform_add -- or, for an intra block, the intra stage below adds it after predicting */
    for (uint32_t i = 0; i < n_ccp; i++) {
        const B200CcpRec *c = &ccp[i];
        const int n = 1 << c->log2, p = c->plane;
        if (p < 1 || p > 2 || c->x + n > pw[p] || c->y + n > ph[p] || c->off_y + (size_t)n * n > park_len ||
            ((c->flags & B200_CCPF_HAS_C) && c->off_c + (size_t)n * n > park_len)) { free(parked); return -8; }
        int16_t r[32 * 32];
        for (int k = 0; k < n * n; k++) {
            const int16_t own = (c->flags & B200_CCPF_HAS_C) ? parked[c->off_c + k] : 0;
            r[k] = (int16_t)(own + ((c->scale * parked[c->off_y + k]) >> 3));
        }
        if (c->flags & B200_CCPF_TO_PARK) memcpy(parked + c->off_out, r, (size_t)n * n * sizeof(int16_t));
        else orc_add_residual(cur[p] + c->y * pw[p] + c->x, pw[p], r, n, bd);
    }
    /* K3 intra, decode order */
    const B200IntraRec *ir = (const B200IntraRec *)(blob + h->sec[B200_SEC_INTRA].off);
    OrcCip cip;
    const int has_cip = (h->flags & B200_FRAME_CIP) && h->cip.count >= 4;
    if (has_cip) {
        const uint32_t *cw = (const uint32_t *)(blob + h->cip.off);
        cip.log2_min_pu = (int)cw[0]; cip.pu_w = (int)cw[1]; cip.pu_h = (int)cw[2]; cip.bits = cw + 4;
        cip.pic_w = h->width; cip.pic_h = h->height;
        if (h->cip.count < B200_CIP_WORDS(cip.pu_w, cip.pu_h)) { free(parked); return -4; }
    }
    for (uint32_t i = 0; i < h->sec[B200_SEC_INTRA].count; i++) {
        const B200IntraRec *r = &ir[i];
        const int p = r->plane;
        if (has_cip) { cip.hs = p && cfi != 3; cip.vs = p && cfi == 1; }
        orc_intra_rec_cip(r, cur[p], pw[p], bd, has_cip ? &cip : NULL);
        if (r->resid_off != B200_NO_RESID)
            orc_add_residual(cur[p] + r->y * pw[p] + r->x, pw[p], parked + r->resid_off, 1 << r->log2, bd);
    }
    free(parked);
    /* K4 deblock */
    if (h->sec[B200_SEC_DBK].count || h->dbd.count) {
        B200DbkLayout L;
        b200_dbk_layout(h->width, h->height, cfi, &L);
        const uint16_t *grid = h->sec[B200_SEC_DBK].count ? (const uint16_t *)(blob + h->sec[B200_SEC_DBK].off) : NULL;
        uint16_t *derived = NULL;
        if (h->dbd.count) {                           /* parameters derived from the records (8f N2); with both present they must agree */
            derived = (uint16_t *)calloc(L.total, sizeof(uint16_t));
            if (!derived) return -3;
            if (orc_dbd_derive(blob, derived)) { free(derived); return -9; }
            if (grid && memcmp(grid, derived, (size_t)L.total * 2)) { free(derived); return -10; }
            grid = derived;
        }
        for (int p = 0; p < 3; p++) deblock_plane(cur[p], pw[p], ph[p], p, grid, &L, bd);
        free(derived);
    }
    /* K5 SAO */
    const uint32_t *tqb_bits = NULL;
    int tqb_log2 = 2, tqb_w = 0;
    if ((h->flags & B200_FRAME_TQB) && h->tqb.count >= 4) {
        const uint32_t *tw = (const uint32_t *)(blob + h->tqb.off);
        if (h->tqb.count < B200_CIP_WORDS(tw[1], tw[2])) return -7;
        tqb_log2 = (int)tw[0]; tqb_w = (int)tw[1]; tqb_bits = tw + 4;
    }
    if (h->sec[B200_SEC_SAO].count) {
        const B200SaoRec *sg = (const B200SaoRec *)(blob + h->sec[B200_SEC_SAO].off);
        const int ctb = 1 << h->log2_ctb_size;
        const int cw = (h->width + ctb - 1) >> h->log2_ctb_size, chh = (h->height + ctb - 1) >> h->log2_ctb_size;
        for (int p = 0; p < 3; p++) {
            const int hs = p && cfi != 3, vs = p && cfi == 1;
            pix_t *copy = (pix_t *)malloc((size_t)pw[p] * ph[p] * sizeof(pix_t));
            if (!copy) return -3;
            memcpy(copy, cur[p], (size_t)pw[p] * ph[p] * sizeof(pix_t));
            for (int cy = 0; cy < chh; cy++)
                for (int cx = 0; cx < cw; cx++) {
                    const B200SaoRec *s = &sg[p * cw * chh + cy * cw + cx];
                    if (s->type == B200_SAO_NONE) continue;
                    const int x0 = (cx << h->log2_ctb_size) >> hs, y0 = (cy << h->log2_ctb_size) >> vs;
                    int w = ctb >> hs, hh = ctb >> vs;
                    if (w > pw[p] - x0) w = pw[p] - x0;
                    if (hh > ph[p] - y0) hh = ph[p] - y0;
                    orc_sao_ctb(s, cur[p], copy, pw[p], x0, y0, w, hh, bd);
                    if (tqb_bits) orc_restore_tqb(cur[p], copy, pw[p], cx << h->log2_ctb_size, cy << h->log2_ctb_size, w, hh, hs, vs,
                                                  bd > 8 ? 2 : 1, tqb_log2, tqb_w, tqb_bits);
                }
            free(copy);
        }
    }
    return 0;
}
