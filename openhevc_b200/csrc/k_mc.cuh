// k_mc.cuh — per-lane code of the inter-prediction stage (K1), put_hevc_{qpel,epel}{,_uni,_bi}{,_w}
// (hevcdsp_template.c:610-1609).  Host + device: kernels.cu strings the phases together with group-local barriers
// (__syncwarp(mask)); tests/emul/kernel_emul.cu (test infrastructure) runs the same phases lane after lane on the CPU.
//
// A tile (<= 16x16, or <= 32x8) is processed by a GROUP of GS lanes: GS = 32 (one warp per tile) for the big tiles,
// GS = 8 (four tiles per warp) for tiles of <= 8x8 samples, which are 3/4 of all tiles in a typical picture.
// Per reference list:
//   W  window: the (w + 7) x (h + 7) neighbourhood (3 instead of 7 for chroma), clamped at the picture border
//      (== emulated_edge_mc, videodsp_template.c:26-100), staged in shared memory as pairs of samples;
//   A  horizontal FIR (if mx): 4 outputs per lane and row, result (int16, the reference's 14-bit intermediate) to `tmp`;
//   B  vertical FIR (if my) or pass-through: lane = column, up to 8 rows per lane -> val[0..7] in registers.
// then the uni / bi / weighted combine and the store.
//
// The stage is issue-bound: the FIRs are therefore written for IDP.2A, the two-way 16-bit x 8-bit dot
// product of sm_90a -- two taps per instruction on samples that stay packed in pairs:
//   * stage A reads six aligned 32-bit words (12 samples) per lane and row; outputs whose first tap falls on an even
//     sample use the words as they are, the others use the five pairs shifted by one sample (PRMT); an 8-tap output
//     is 4 IDP.2A (lo / hi halves of two coefficient registers) instead of 8 IMAD;
//   * when a vertical pass follows, stage A stores its rows interleaved in pairs, tmp[(r / 2, x)] = (row r, row r + 1),
//     so stage B reads eight 32-bit words per lane and again needs 4 IDP.2A per output (7 PRMT for the odd rows);
//   * vertical-only and full-pel blocks keep the scalar path (no horizontal pass that could pair the rows up).
#pragma once
#include "common.cuh"

#define MC_WIN_MAX 640      // (32+7+1) x 15 = 600, (16+7+1) x 23 = 552, + slack for padded reads
#define MC_TMP_MAX 512      // 15 x 32, 23 x 16 plain; 8 row pairs x 32 x 2, 12 row pairs x 16 x 2 interleaved
template <int GS> struct McSmem;
template <> struct McSmem<32> { static constexpr int WIN = MC_WIN_MAX, TMP = MC_TMP_MAX; };
template <> struct McSmem<8>  { static constexpr int WIN = 256 /* 15 x 16 */, TMP = 160 /* 15 x 8, 15 x 10 padded */; };

// ---- filter taps (ff_hevc_qpel_filters / ff_hevc_epel_filters, hevcdsp.c:1028-1042), four per register ----
HD constexpr uint32_t mc_pack4(int a, int b, int c, int d)
{
    return (uint32_t)(a & 0xff) | ((uint32_t)(b & 0xff) << 8) | ((uint32_t)(c & 0xff) << 16) | ((uint32_t)(d & 0xff) << 24);
}
// taps 0..3 (half 0) or 4..7 (half 1) of the 8-tap luma filter of phase f (1..3)
HD uint32_t mc_qpel4(int f, int half)
{
    return f == 1 ? (half ? mc_pack4(17, -5, 1, 0) : mc_pack4(-1, 4, -10, 58))
         : f == 2 ? (half ? mc_pack4(40, -11, 4, -1) : mc_pack4(-1, 4, -11, 40))
         : f == 3 ? (half ? mc_pack4(58, -10, 4, -1) : mc_pack4(0, 1, -5, 17))
                  : (half ? 0u : mc_pack4(0, 0, 0, 64));
}
HD uint32_t mc_epel4(int f)
{
    return f == 1 ? mc_pack4(-2, 58, 10, -2) : f == 2 ? mc_pack4(-4, 54, 16, -2) : f == 3 ? mc_pack4(-6, 46, 28, -4)
         : f == 4 ? mc_pack4(-4, 36, 36, -4) : f == 5 ? mc_pack4(-4, 28, 46, -6) : f == 6 ? mc_pack4(-2, 16, 54, -4)
         : f == 7 ? mc_pack4(-2, 10, 58, -2) : mc_pack4(0, 64, 0, 0);
}
HD int mc_tap(uint32_t c4, int k) { return (int)(int8_t)(c4 >> (8 * k)); }

// d + a.lo16 * b.byte[0|2] + a.hi16 * b.byte[1|3]: IDP.2A.{LO,HI}.{U16,S16}.S8
HD int dp2a_lo_u(uint32_t a, uint32_t b, int d)
{
#ifdef __CUDA_ARCH__
    int r; asm("dp2a.lo.u32.s32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(d)); return r;
#else
    return d + (int)(a & 0xffff) * (int)(int8_t)b + (int)(a >> 16) * (int)(int8_t)(b >> 8);
#endif
}
HD int dp2a_hi_u(uint32_t a, uint32_t b, int d)
{
#ifdef __CUDA_ARCH__
    int r; asm("dp2a.hi.u32.s32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(d)); return r;
#else
    return d + (int)(a & 0xffff) * (int)(int8_t)(b >> 16) + (int)(a >> 16) * (int)(int8_t)(b >> 24);
#endif
}
HD int dp2a_lo_s(uint32_t a, uint32_t b, int d)
{
#ifdef __CUDA_ARCH__
    int r; asm("dp2a.lo.s32.s32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(d)); return r;
#else
    return d + (int)(int16_t)(a & 0xffff) * (int)(int8_t)b + (int)(int16_t)(a >> 16) * (int)(int8_t)(b >> 8);
#endif
}
HD int dp2a_hi_s(uint32_t a, uint32_t b, int d)
{
#ifdef __CUDA_ARCH__
    int r; asm("dp2a.hi.s32.s32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(d)); return r;
#else
    return d + (int)(int16_t)(a & 0xffff) * (int)(int8_t)(b >> 16) + (int)(int16_t)(a >> 16) * (int)(int8_t)(b >> 24);
#endif
}

// ---- one tile ---------------------------------------------------------------------------------------------------------
struct McTile {
    int dx, dy, w, h, plane, flags;
    int sx0, sy0, sx1, sy1, ref0, ref1, frac0, frac1;
    int w0, w1, o0, o1, denom;
    // stage B: lane = column (1 << wsh per row group), `parts` row groups of rows_per rows
    int wsh, parts, rows_per;
    // stage A: 4 outputs per lane, q quads per row, (1 << lsh) lanes per row
    int wpad, lsh, q;
};

template <int GS>
HD McTile mc_decode(const int4 ra, const int4 rb)
{
    McTile t;
    const int mxy = ra.x, whpf = ra.y;
    t.dx = mxy & 0xffff; t.dy = (int)((unsigned)mxy >> 16);
    t.w = whpf & 0xff; t.h = (whpf >> 8) & 0xff;
    if (GS == 8) { t.w = imin(t.w, 8); t.h = imin(t.h, 8); }   // the list order guarantees it; never trust it with shared memory
    t.plane = (whpf >> 16) & 0xff; t.flags = (int)((unsigned)whpf >> 24);
    t.sx0 = (int16_t)(ra.z & 0xffff); t.sy0 = (int16_t)((unsigned)ra.z >> 16); t.sx1 = (int16_t)(ra.w & 0xffff); t.sy1 = (int16_t)((unsigned)ra.w >> 16);
    t.ref0 = rb.x & 0xff; t.ref1 = (rb.x >> 8) & 0xff; t.frac0 = (rb.x >> 16) & 0xff; t.frac1 = (int)((unsigned)rb.x >> 24);
    t.w0 = (int16_t)(rb.y & 0xffff); t.w1 = (int16_t)((unsigned)rb.y >> 16); t.o0 = (int16_t)(rb.z & 0xffff); t.o1 = (int16_t)((unsigned)rb.z >> 16);
    t.denom = rb.w & 0xff;
    const int w = t.w, h = t.h;
    t.wsh = w <= 2 ? 1 : w <= 4 ? 2 : w <= 8 ? 3 : w <= 16 ? 4 : 5;
    t.parts = GS >> t.wsh;
    t.rows_per = ((h + t.parts - 1) / t.parts + 1) & ~1;          // even: row pairs stay aligned for the IDP.2A vertical pass
    t.wpad = (w + 3) & ~3;
    t.q = t.wpad >> 2;
    t.lsh = t.q <= 1 ? 0 : t.q <= 2 ? 1 : t.q <= 4 ? 2 : 3;
    return t;
}

struct McWin {              // geometry of one list's window in shared memory
    int C, R;               // columns / rows the filters need
    int ox, oy;             // picture position of window sample (0, 0) before alignment
    int skew, ax;           // window origin aligned down to an even sample: ax = ox - skew
    int np, Ws;             // sample pairs per row, row stride in samples
};
template <int TAPS>
HD McWin mc_window(const McTile &t, int sx, int sy, int mx, int my)
{
    constexpr int BEFORE = TAPS == 8 ? 3 : 1;
    McWin g;
    g.C = t.w + (mx ? TAPS - 1 : 0); g.R = t.h + (my ? TAPS - 1 : 0);
    g.ox = sx - (mx ? BEFORE : 0); g.oy = sy - (my ? BEFORE : 0);
    g.skew = g.ox & 1; g.ax = g.ox - g.skew;
    g.np = (g.C + g.skew + 1) >> 1; g.Ws = 2 * g.np;
    return g;
}

// ---- phase W -------------------------------------------------------------------------------------------------------------
template <typename PIX, int TAPS, int GS>
HD void mc_load_window(const PlaneDesc &rp, const McTile &t, int sx, int sy, int mx, int my, int gl, uint16_t *win)
{
    const McWin g = mc_window<TAPS>(t, sx, sy, mx, my);
    if (g.ax >= 0 && g.ax + g.Ws <= rp.w && g.oy >= 0 && g.oy + g.R <= rp.h) {
        // interior: one 2-sample load per lane, 1 or 2 rows per pass, no clamping
        const int lpr = g.np <= GS / 2 ? GS / 2 : GS;       // lanes per window row
        const int pi = gl & (lpr - 1), rsub = gl >= lpr ? 1 : 0, rstep = GS / lpr;
        if (pi < g.np) {
            const uint8_t *src = rp.base + (size_t)(g.oy + rsub) * rp.pitch + (size_t)(g.ax + 2 * pi) * sizeof(PIX);
            uint32_t *dst = reinterpret_cast<uint32_t *>(win) + rsub * g.np + pi;
            for (int r = rsub; r < g.R; r += rstep) {
                uint32_t v;
                if (sizeof(PIX) == 2) v = *reinterpret_cast<const uint32_t *>(src);
                else { const uint32_t b2 = *reinterpret_cast<const uint16_t *>(src); v = (b2 & 0xff) | ((b2 & 0xff00) << 8); }
                *dst = v;
                src += (size_t)rstep * rp.pitch; dst += rstep * g.np;
            }
        }
    } else {
        // window hangs over the picture border: clamp sample by sample (== emulated_edge_mc)
        for (int i = gl; i < g.R * g.Ws; i += GS) {
            const int r = i / g.Ws, cc = i - r * g.Ws;
            const int x = clip3i(g.ax + cc, 0, rp.w - 1), y = clip3i(g.oy + r, 0, rp.h - 1);
            win[i] = *px_ptr<PIX>(rp, x, y);
        }
    }
}

// ---- phase A: horizontal FIR ----------------------------------------------------------------------------------------------
template <int TAPS, int GS>
HD void mc_stage_a(const McTile &t, int sx, int sy, int mx, int my, int bd, int gl, const uint16_t *win, int16_t *tmp)
{
    const McWin g = mc_window<TAPS>(t, sx, sy, mx, my);
    const int qi = gl & ((1 << t.lsh) - 1), rstep = GS >> t.lsh;
    if (qi >= t.q) return;
    const uint32_t CA = TAPS == 8 ? mc_qpel4(mx, 0) : mc_epel4(mx), CB = TAPS == 8 ? mc_qpel4(mx, 1) : 0u;
    const int sh = bd - 8;
    const uint32_t *win32 = reinterpret_cast<const uint32_t *>(win);
    constexpr int NW = TAPS == 8 ? 6 : 4;                    // aligned words covering skew + j + k, j < 4, k < TAPS
    for (int r = gl >> t.lsh; r < g.R; r += rstep) {
        uint32_t W[NW], Q[NW - 1];
#pragma unroll
        for (int i = 0; i < NW; i++) W[i] = win32[r * g.np + 2 * qi + i];
#pragma unroll
        for (int i = 0; i < NW - 1; i++) Q[i] = fsr16(W[i], W[i + 1]);      // the pairs that start on an odd sample
        int o[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            // first tap of output j sits on sample e = skew + j of the aligned words
            int acc;
            if (g.skew == 0) {
                const int m = j >> 1;
                if (!(j & 1)) { acc = dp2a_lo_u(W[m], CA, 0); acc = dp2a_hi_u(W[m + 1], CA, acc); if (TAPS == 8) { acc = dp2a_lo_u(W[m + 2], CB, acc); acc = dp2a_hi_u(W[m + 3], CB, acc); } }
                else          { acc = dp2a_lo_u(Q[m], CA, 0); acc = dp2a_hi_u(Q[m + 1], CA, acc); if (TAPS == 8) { acc = dp2a_lo_u(Q[m + 2], CB, acc); acc = dp2a_hi_u(Q[m + 3], CB, acc); } }
            } else {
                const int m = (j + 1) >> 1;
                if (j & 1)    { acc = dp2a_lo_u(W[m], CA, 0); acc = dp2a_hi_u(W[m + 1], CA, acc); if (TAPS == 8) { acc = dp2a_lo_u(W[m + 2], CB, acc); acc = dp2a_hi_u(W[m + 3], CB, acc); } }
                else          { const int n = j >> 1; acc = dp2a_lo_u(Q[n], CA, 0); acc = dp2a_hi_u(Q[n + 1], CA, acc); if (TAPS == 8) { acc = dp2a_lo_u(Q[n + 2], CB, acc); acc = dp2a_hi_u(Q[n + 3], CB, acc); } }
            }
            o[j] = (acc >> sh) & 0xffff;
        }
        if (my) {           // a vertical pass follows: rows interleaved in pairs, element (r, x) at ((r >> 1) * wpad + x) * 2 + (r & 1)
            int16_t *d = tmp + (((r >> 1) * t.wpad + 4 * qi) << 1) + (r & 1);
            d[0] = (int16_t)o[0]; d[2] = (int16_t)o[1]; d[4] = (int16_t)o[2]; d[6] = (int16_t)o[3];
        } else {
            uint32_t *d = reinterpret_cast<uint32_t *>(tmp + r * t.wpad + 4 * qi);
            d[0] = (uint32_t)o[0] | ((uint32_t)o[1] << 16);
            d[1] = (uint32_t)o[2] | ((uint32_t)o[3] << 16);
        }
    }
}

// ---- phase B: vertical FIR (or pass-through), lane = column, up to 8 rows per lane ----------------------------------------
// Loads are unconditional: lanes without rows (y0 >= h) read from row 0, and the rows / columns beyond the tile only
// feed outputs that are never stored.
template <int TAPS, int GS>
HD void mc_stage_b(const McTile &t, int sx, int sy, int mx, int my, int bd, int gl, const uint16_t *win, const int16_t *tmp, int (&val)[8])
{
    const McWin g = mc_window<TAPS>(t, sx, sy, mx, my);
    const int xl = gl & ((1 << t.wsh) - 1);
    int y0 = (gl >> t.wsh) * t.rows_per;
    if (y0 >= t.h) y0 = 0;
    if (mx && my) {
        // both passes: row pairs from stage A, 2 taps per IDP.2A
        const uint32_t CA = TAPS == 8 ? mc_qpel4(my, 0) : mc_epel4(my), CB = TAPS == 8 ? mc_qpel4(my, 1) : 0u;
        constexpr int NP = TAPS == 8 ? 8 : 6;                 // row pairs covering rows y0 .. y0 + 7 + TAPS - 1
        const uint32_t *t32 = reinterpret_cast<const uint32_t *>(tmp);
        uint32_t P[NP], Q[NP - 1];
#pragma unroll
        for (int i = 0; i < NP; i++) P[i] = t32[((y0 >> 1) + i) * t.wpad + xl];
#pragma unroll
        for (int i = 0; i < NP - 1; i++) Q[i] = fsr16(P[i], P[i + 1]);
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const int m = j >> 1;
            int acc;
            if (!(j & 1)) { acc = dp2a_lo_s(P[m], CA, 0); acc = dp2a_hi_s(P[m + 1], CA, acc); if (TAPS == 8) { acc = dp2a_lo_s(P[m + 2], CB, acc); acc = dp2a_hi_s(P[m + 3], CB, acc); } }
            else          { acc = dp2a_lo_s(Q[m], CA, 0); acc = dp2a_hi_s(Q[m + 1], CA, acc); if (TAPS == 8) { acc = dp2a_lo_s(Q[m + 2], CB, acc); acc = dp2a_hi_s(Q[m + 3], CB, acc); } }
            val[j] = acc >> 6;
        }
        return;
    }
    int a[8 + TAPS - 1];
    if (mx) {
        const int16_t *s = tmp + y0 * t.wpad + xl;
#pragma unroll
        for (int k = 0; k < 8 + TAPS - 1; k++) a[k] = s[k * t.wpad];
    } else {
        const uint16_t *s = win + y0 * g.Ws + g.skew + xl;
#pragma unroll
        for (int k = 0; k < 8 + TAPS - 1; k++) a[k] = s[k * g.Ws];
    }
    if (my) {
        const uint32_t CA = TAPS == 8 ? mc_qpel4(my, 0) : mc_epel4(my), CB = TAPS == 8 ? mc_qpel4(my, 1) : 0u;
        int fy[TAPS];
#pragma unroll
        for (int k = 0; k < TAPS; k++) fy[k] = mc_tap(k < 4 ? CA : CB, k & 3);
        const int sh = bd - 8;                                 // vertical only (mx == 0 here)
#pragma unroll
        for (int j = 0; j < 8; j++) {
            int acc = 0;
#pragma unroll
            for (int k = 0; k < TAPS; k++) acc += fy[k] * a[j + k];
            val[j] = acc >> sh;
        }
    } else {
        const int sh = mx ? 0 : 14 - bd;
#pragma unroll
        for (int j = 0; j < 8; j++) val[j] = a[j] << sh;
    }
}

// ---- combine + store (hevcdsp_template.c:626-1136: uni, uni_w, bi, bi_w) ------------------------------------------------------
template <typename PIX>
HD void mc_store(const McTile &t, const PlaneDesc &dp, int bd, int gl, const int (&v0)[8], const int (&v1)[8])
{
    const int shift = 14 - bd, maxv = (1 << bd) - 1;
    const bool bi = t.flags & B200_MCF_BI, weighted = t.flags & B200_MCF_WEIGHTED;
    const bool fullpel0 = t.frac0 == 0;
    const int xl = gl & ((1 << t.wsh) - 1), y0 = (gl >> t.wsh) * t.rows_per;
    if (xl >= t.w) return;
    PIX *d = px_ptr<PIX>(dp, t.dx + xl, t.dy + y0);
#pragma unroll
    for (int j = 0; j < 8; j++) {
        if (j >= t.rows_per || y0 + j >= t.h) break;
        int out;
        if (!bi) {
            if (!weighted) out = fullpel0 ? (v0[j] >> shift) : clip3i((v0[j] + (1 << (shift - 1))) >> shift, 0, maxv);
            else {
                const int s = t.denom + shift;
                out = clip3i(((v0[j] * t.w0 + (1 << (s - 1))) >> s) + t.o0 * (1 << (bd - 8)), 0, maxv);
            }
        } else {
            const int a = (int16_t)v0[j];          // list 0 travels through the reference's int16 tmp[] (hevc.c:1761)
            if (!weighted) out = clip3i((v1[j] + a + (1 << shift)) >> (shift + 1), 0, maxv);
            else {
                const int l2 = t.denom + shift, o = (t.o0 + t.o1) * (1 << (bd - 8)) + 1;
                out = clip3i((v1[j] * t.w1 + a * t.w0 + (o << l2)) >> (l2 + 1), 0, maxv);
            }
        }
        *d = (PIX)out;
        d = reinterpret_cast<PIX *>(reinterpret_cast<uint8_t *>(d) + dp.pitch);
    }
}
