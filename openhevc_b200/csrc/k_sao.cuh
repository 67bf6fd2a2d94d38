// k_sao.cuh — per-thread code of the SAO stage (K5).  Host + device: kernels.cu wraps sao_thread() in the __global__
// kernel; the CPU suite's warp emulator (tests/emul/warp/) compiles kernels.cu for the host, so the packed arithmetic is
// checked against the oracle, through the product's own launcher, before it ever reaches a GPU.
#pragma once
#include "common.cuh"

#ifndef SAO_R
#define SAO_R 2          // rows per thread: 2 rows + 3 blocks per SM leave more warps to hide the loads than 4 rows + 2 blocks
#endif

// 8 consecutive samples (x multiple of 8: 16-byte / 8-byte aligned; rows are padded to the pitch, so a vector that
// starts inside the plane may be read whole), as four registers of two 16-bit samples
template <typename PIX> HD void load8p(const PlaneDesc &pd, int x, int y, uint32_t (&v)[4])
{
    const PIX *s = px_ptr<PIX>(pd, x, y);
    if (sizeof(PIX) == 2) {
        const uint4 q = *reinterpret_cast<const uint4 *>(s);
        v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
    } else {
        const uint2 q = *reinterpret_cast<const uint2 *>(s);
        v[0] = prmt32(q.x, 0, 0x4140); v[1] = prmt32(q.x, 0, 0x4342); v[2] = prmt32(q.y, 0, 0x4140); v[3] = prmt32(q.y, 0, 0x4342);
    }
}
template <typename PIX> HD void store8p(const PlaneDesc &pd, int x, int y, const uint32_t (&v)[4], int nvalid)
{
    PIX *d = px_ptr<PIX>(pd, x, y);
    if (sizeof(PIX) == 2) {
        if (nvalid == 8) *reinterpret_cast<uint4 *>(d) = make_uint4(v[0], v[1], v[2], v[3]);
        else *reinterpret_cast<uint2 *>(d) = make_uint2(v[0], v[1]);            // plane widths are multiples of 4
    } else {
        const uint32_t lo = prmt32(v[0], v[1], 0x6420);
        if (nvalid == 8) *reinterpret_cast<uint2 *>(d) = make_uint2(lo, prmt32(v[2], v[3], 0x6420));
        else *reinterpret_cast<uint32_t *>(d) = lo;
    }
}

struct SaoCtb {                 // one decoded B200SaoRec + the geometry of its CTB in this plane
    int type, cls, borders, edges, variant, tqb;
    int off[5];
    int x0, y0, w, h;           // CTB origin and (picture-clipped) size in samples of the plane
};
HD SaoCtb sao_decode(const uint4 rq, const PlaneDesc &sp, int cx, int cy, int lw, int lh)
{
    SaoCtb t;
    t.type = rq.x & 0xff; t.cls = (rq.x >> 8) & 0xff; t.borders = (rq.x >> 16) & 0xff; t.edges = rq.x >> 24; t.variant = rq.y & 0xff; t.tqb = (rq.y >> 8) & 0xff;
    t.off[0] = (int16_t)(rq.y >> 16); t.off[1] = (int16_t)(rq.z & 0xffff); t.off[2] = (int16_t)(rq.z >> 16); t.off[3] = (int16_t)(rq.w & 0xffff); t.off[4] = (int16_t)(rq.w >> 16);
    t.x0 = cx << lw; t.y0 = cy << lh;
    t.w = imin(1 << lw, sp.w - t.x0); t.h = imin(1 << lh, sp.h - t.y0);
    return t;
}

// The reference rules for one row of 8 samples, sample by sample (edge offset only): used for the outermost rows /
// columns of CTBs that carry border or restore flags, and for CTBs whose offsets do not fit the packed table.  Rare, and
// deliberately self-contained (it reads the record again) so that the packed path carries none of its state in registers.
template <typename PIX>
__host__ __device__ __noinline__ void sao_row_exact(const PlaneDesc &sp, const B200SaoRec *rec, int cx, int cy, int lwlh, int gx, int gy, int maxv, uint32_t (&outp)[4])
{
    const SaoCtb t = sao_decode(LDG128(rec), sp, cx, cy, lwlh & 0xff, lwlh >> 8);
    int c[8], out[8];
    const int yu = imax(gy - 1, 0), yd = imin(gy + 1, sp.h - 1);
    int A[8], Bq[8];
#pragma unroll
    for (int i = 0; i < 8; i++) {
        // positions outside the picture are clamped (they are only ever used by samples that take the `zero` path)
        const int x = imin(gx + i, sp.w - 1), xl = imax(x - 1, 0), xr = imin(x + 1, sp.w - 1);
        c[i] = *px_ptr<PIX>(sp, x, gy);
        const int ya = t.cls == 0 ? gy : yu, yb = t.cls == 0 ? gy : yd;
        const int xa = t.cls == 1 ? x : t.cls == 3 ? xr : xl, xb = t.cls == 1 ? x : t.cls == 3 ? xl : xr;
        A[i] = *px_ptr<PIX>(sp, xa, ya);
        Bq[i] = *px_ptr<PIX>(sp, xb, yb);
    }
    const int cls = t.cls, w = t.w, h = t.h, xs = gx - t.x0, y = gy - t.y0;
    const bool b_l = t.borders & 1, b_t = t.borders & 2, b_r = t.borders & 4, b_b = t.borders & 8;
    const bool zrow = cls != 0 && ((b_t && y == 0) || (b_b && y == h - 1));
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int x = xs + i, v = c[i];
        const bool zero = zrow || (cls != 1 && ((b_l && x == 0) || (b_r && x == w - 1)));
        const int e = (v > A[i]) - (v < A[i]) + (v > Bq[i]) - (v < Bq[i]);      // -2..2
        const int o = zero ? t.off[0] : e == -2 ? t.off[1] : e == -1 ? t.off[2] : e == 0 ? t.off[0] : e == 1 ? t.off[3] : t.off[4];   // edge_idx[] = {1,2,0,3,4}
        out[i] = clip3i(v + o, 0, maxv);
    }
    if (t.variant) {   // not-across-boundary restore, hevcdsp_template.c:533-566 (2 = SAO_EO_135D, 3 = SAO_EO_45D)
        const int edges = t.edges;
        const int init_x = (cls != 1 && b_l) ? 1 : 0, wid = (cls != 1 && b_r) ? w - 1 : w, hei = (cls != 0 && b_b) ? h - 1 : h;
        const bool ve0 = edges & 1, ve1 = edges & 2, he0 = edges & 4, he1 = edges & 8;
        const bool de0 = edges & 16, de1 = edges & 32, de2 = edges & 64, de3 = edges & 128;
        const int sul = !de0 && cls == 2 && !b_l && !b_t, sur = !de1 && cls == 3 && !b_t && !b_r;
        const int slr = !de2 && cls == 2 && !b_r && !b_b, sll = !de3 && cls == 3 && !b_l && !b_b;
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const int x = xs + i;
            bool rs = false;
            rs |= ve0 && cls != 1 && x == 0 && y >= sul && y < hei - sll;
            rs |= ve1 && cls != 1 && x == wid - 1 && y >= sur && y < hei - slr;
            rs |= he0 && cls != 0 && y == 0 && x >= init_x + sul && x < wid - sur;
            rs |= he1 && cls != 0 && y == hei - 1 && x >= init_x + sll && x < wid - slr;
            rs |= de0 && cls == 2 && x == 0 && y == 0;
            rs |= de1 && cls == 3 && x == wid - 1 && y == 0;
            rs |= de2 && cls == 2 && x == wid - 1 && y == hei - 1;
            rs |= de3 && cls == 3 && x == 0 && y == hei - 1;
            if (rs) out[i] = c[i];
        }
    }
#pragma unroll
    for (int k = 0; k < 4; k++) outp[k] = (uint32_t)out[2 * k] | ((uint32_t)out[2 * k + 1] << 16);
}

// restore_tqb_pixels (hevc_filter.c:163-193): after the SAO of a CTB, PUs flagged in is_pcm[] (PCM with the loop filter off,
// cu_transquant_bypass) get their deblocked samples back.  Two things the reference really does are kept:
//  - it is called with the LUMA origin of the CTB but the CTB's width / height in the plane being filtered, so for
//    subsampled chroma only the PUs of the first half of the CTB are visited (x_lim / y_lim below);
//  - a row of a PU is copied with memcpy(.., min_pu_size >> hshift): samples used as bytes, so above 8 bits only the first
//    half of each row comes back (len below).
// Only CTBs marked by the recorder (B200SaoRec.tqb) look at the bitmap: rare streams, a handful of CTBs.
struct TqbDesc {
    const uint32_t *bits;        // one bit per min-PU, row-major; nullptr = nothing to restore in this picture
    int log2_pu, pu_w;
};
HD bool tqb_pu(const TqbDesc &q, int X, int Y)
{
    const long i = (long)Y * q.pu_w + X;
#ifdef __CUDA_ARCH__
    return (__ldg(q.bits + (i >> 5)) >> (i & 31)) & 1;
#else
    return (q.bits[i >> 5] >> (i & 31)) & 1;
#endif
}
// one row of 8 samples at (gx, gy) of a plane with shifts hs / vs: samples of restored PUs take the value of `c` again
HD void sao_restore_row(const TqbDesc &q, const SaoCtb &t, int hs, int vs, int B, int gx, int gy, const uint32_t (&c)[4], uint32_t (&o)[4])
{
    const int l = q.log2_pu;
    const int x_lim = ((t.x0 << hs) + t.w) >> l, y_lim = ((t.y0 << vs) + t.h) >> l;      // luma origin + size in the plane (sic)
    const int len = ((1 << l) >> hs) / B;                                                  // bytes taken for samples (sic)
    const int Y = (gy << vs) >> l;
    if (Y >= y_lim) return;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int px = gx + i, X = (px << hs) >> l;
        if (X < x_lim && px - ((X << l) >> hs) < len && tqb_pu(q, X, Y)) {
            const uint32_t keep = (i & 1) ? 0xffff0000u : 0x0000ffffu;
            o[i >> 1] = (o[i >> 1] & ~keep) | (c[i >> 1] & keep);
        }
    }
}

// out = clip(c + table[idx]) for two samples: idx = 0..4 in each 16-bit half of X
HD uint32_t sao_apply2(uint32_t c, uint32_t X, uint32_t tab_lo, uint32_t tab_hi, uint32_t maxv2)
{
    const uint32_t sel = X | (X >> 8) | 0x7070u;                 // nibbles: idx_lo, 7 (a zero byte), idx_hi, 7
    const uint32_t o = prmt32(tab_lo, tab_hi, sel);                // two offsets, biased by 128, one per half
    return viaddmin_s16x2_relu(c + o, 0xff80ff80u, maxv2);      // imax(imin(c + o - 128, maxv), 0)
}

// Edge offset of class CLS for the 8 x SAO_R samples of one thread.  a / b = the two neighbours of the class
// (hevcdsp_template.c:372-431: pos[][] = {{-1,0},{1,0}}, {{0,-1},{0,1}}, {{-1,-1},{1,1}}, {{1,-1},{-1,1}}).
template <typename PIX, int CLS>
HD void sao_edge_rows(const PlaneDesc &sp, const PlaneDesc &dp, const B200SaoRec *rec, int cx, int cy, int lwlh, int gx, int gy0, int nvalid, int nrows,
                      int maxv, uint32_t tab_lo, uint32_t tab_hi, int exact_rows,
                      const uint32_t (&c)[SAO_R + 2][4], const uint32_t (&sl)[SAO_R + 2], const uint32_t (&sr)[SAO_R + 2],
                      const TqbDesc &tq, const SaoCtb &t, int hsvsB)
{
    const uint32_t maxv2 = (uint32_t)maxv * 0x10001u;
    constexpr int JLO = CLS == 0 ? 1 : 0, JHI = CLS == 0 ? SAO_R : SAO_R + 1;
    uint32_t m[SAO_R + 2][4], mL[SAO_R + 2], mR[SAO_R + 2];
#pragma unroll
    for (int j = JLO; j <= JHI; j++) {
#pragma unroll
        for (int k = 0; k < 4; k++) m[j][k] = vadd2(~c[j][k], 0x00020002u);   // 1 - sample, per half
        mL[j] = (2u + ~sl[j]) << 16;                                           // 1 - left neighbour, in the high half
        mR[j] = 2u + ~sr[j];                                                   // 1 - right neighbour (only the low half is used)
    }
#pragma unroll
    for (int r = 0; r < SAO_R; r++) {
        if (r < nrows) {
            const int j = r + 1;
            uint32_t o[4];
            if ((exact_rows >> r) & 1) {
                sao_row_exact<PIX>(sp, rec, cx, cy, lwlh, gx, gy0 + r, maxv, o);
            } else {
                uint32_t A[4], Bn[4];
                const int ja = CLS == 0 ? j : j - 1, jb = CLS == 0 ? j : j + 1;     // compile-time after unrolling
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    if (CLS == 1) { A[k] = m[ja][k]; Bn[k] = m[jb][k]; }
                    else if (CLS == 3) {
                        A[k] = fsr16(m[ja][k], k < 3 ? m[ja][k < 3 ? k + 1 : 3] : mR[ja]);        // sample i + 1 of the row above
                        Bn[k] = fsl16(k ? m[jb][k ? k - 1 : 0] : mL[jb], m[jb][k]);               // sample i - 1 of the row below
                    } else {
                        A[k] = fsl16(k ? m[ja][k ? k - 1 : 0] : mL[ja], m[ja][k]);                // sample i - 1
                        Bn[k] = fsr16(m[jb][k], k < 3 ? m[jb][k < 3 ? k + 1 : 3] : mR[jb]);       // sample i + 1
                    }
                }
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const uint32_t ua = viaddmin_s16x2_relu(c[j][k], A[k], 0x00020002u);    // sign(c - a) + 1
                    const uint32_t ub = viaddmin_s16x2_relu(c[j][k], Bn[k], 0x00020002u);   // sign(c - b) + 1
                    o[k] = sao_apply2(c[j][k], ua + ub, tab_lo, tab_hi, maxv2);
                }
            }
            if (t.tqb) sao_restore_row(tq, t, hsvsB & 1, (hsvsB >> 1) & 1, hsvsB >> 2, gx, gy0 + r, c[j], o);
            store8p<PIX>(dp, gx, gy0 + r, o, nvalid);
        }
    }
}

// One thread = 8 consecutive samples x SAO_R rows, always inside one CTB (CTBs are >= 8 samples wide in every plane and
// their heights are multiples of 4 or end at the picture edge).  A warp = S strips (one CTB width, or 8 strips) x 32/S
// row groups.
template <typename PIX>
HD void sao_thread(const B200SaoRec *__restrict__ grid, const FrameDesc &src, const FrameDesc &dst, int bd,
                   int log2_ctb, int ctb_w, int ctb_h, int cfi, int4 tile_base, int3 tiles_x, const TqbDesc &tq, int warp, int lane)
{
    if (warp >= tile_base.w) return;                                // tile_base = first tile of plane 0, 1, 2, and the total
    const int plane = warp >= tile_base.z ? 2 : warp >= tile_base.y ? 1 : 0;
    const PlaneDesc sp = plane_of(src, plane), dp = plane_of(dst, plane);
    const int hs = plane && cfi != 3, vs = plane && cfi == 1;
    const int lw = log2_ctb - hs, lh = log2_ctb - vs;
    const int lS = imin(lw - 3, 3);                                  // log2(strips per warp row): CTB width / 8, at most 8
    const int tile = warp - (plane == 2 ? tile_base.z : plane == 1 ? tile_base.y : 0);
    const int ntx = plane == 2 ? tiles_x.z : plane == 1 ? tiles_x.y : tiles_x.x;
    const int ty = tile / ntx, tx = tile - ty * ntx;
    const int gx = ((tx << lS) + (lane & ((1 << lS) - 1))) * 8;
    const int gy0 = ((ty << (5 - lS)) + (lane >> lS)) * SAO_R;
    if (gx >= sp.w || gy0 >= sp.h) return;
    const int cx = gx >> lw, cy = gy0 >> lh;
    const B200SaoRec *rec = grid + (plane * ctb_h + cy) * ctb_w + cx;
    const uint4 rq = LDG128(rec);
    // The rows are fetched BEFORE the record is looked at: whatever the CTB's SAO type, the SAO_R rows are needed (even
    // "off" copies them), and the row above / below and the two outer columns are needed by 3 of the 4 edge classes --
    // issuing them now puts ONE memory latency on the thread's critical path instead of two (record, then rows).
    const int nvalid = imin(8, sp.w - gx);
    uint32_t c[SAO_R + 2][4], sl[SAO_R + 2], sr[SAO_R + 2];
    {
        const int xl = imax(gx - 1, 0), xr = imin(gx + 8, sp.w - 1);
#pragma unroll
        for (int j = 0; j <= SAO_R + 1; j++) {
            const int yy = imin(imax(gy0 + j - 1, 0), sp.h - 1);
            load8p<PIX>(sp, gx, yy, c[j]);
            sl[j] = *px_ptr<PIX>(sp, xl, yy);
            sr[j] = *px_ptr<PIX>(sp, xr, yy);
        }
        if (nvalid < 8) {                          // beyond the plane: replicate, like clamped addressing
#pragma unroll
            for (int j = 0; j <= SAO_R + 1; j++) c[j][2] = c[j][3] = prmt32(c[j][1], 0, 0x3232);
        }
    }
    SaoCtb t = sao_decode(rq, sp, cx, cy, lw, lh);
    if (!tq.bits) t.tqb = 0;                                        // a mark without a bitmap means nothing
    const int nrows = imin(SAO_R, sp.h - gy0);
    const int maxv = (1 << bd) - 1;
    const uint32_t maxv2 = (uint32_t)maxv * 0x10001u;

    if (t.type != B200_SAO_BAND && t.type != B200_SAO_EDGE) {           // no SAO in this CTB: copy through
#pragma unroll
        for (int r = 0; r < SAO_R; r++) if (r < nrows) store8p<PIX>(dp, gx, gy0 + r, c[r + 1], nvalid);
        return;
    }
    bool fits = true;                                                   // offsets representable in the packed table?
#pragma unroll
    for (int k = 0; k < 5; k++) fits &= t.off[k] >= -128 && t.off[k] <= 127;

    if (t.type == B200_SAO_BAND) {
        const int sh = bd - 5;
        if (fits) {
            const uint32_t tab_lo = (uint32_t)((t.off[1] + 128) & 0xff) | ((uint32_t)((t.off[2] + 128) & 0xff) << 8) |
                                    ((uint32_t)((t.off[3] + 128) & 0xff) << 16) | ((uint32_t)((t.off[4] + 128) & 0xff) << 24);
            const uint32_t tab_hi = 128u;                                   // entry 4: no offset
            const uint32_t nb = (uint32_t)((32 - t.cls) & 31) * 0x10001u;   // t.cls = band_position for band CTBs
#pragma unroll
            for (int r = 0; r < SAO_R; r++) {
                if (r >= nrows) break;
                uint32_t o[4];
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const uint32_t band = (c[r + 1][k] >> sh) & 0x001f001fu;
                    const uint32_t kk = vminu2((band + nb) & 0x001f001fu, 0x00040004u);      // (band - position) & 31, 4 = outside
                    o[k] = sao_apply2(c[r + 1][k], kk, tab_lo, tab_hi, maxv2);
                }
                if (t.tqb) sao_restore_row(tq, t, hs, vs, (int)sizeof(PIX), gx, gy0 + r, c[r + 1], o);
                store8p<PIX>(dp, gx, gy0 + r, o, nvalid);
            }
        } else {
#pragma unroll
            for (int r = 0; r < SAO_R; r++) {
                if (r >= nrows) break;
                uint32_t o[4];
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    uint32_t res = 0;
#pragma unroll
                    for (int hlf = 0; hlf < 2; hlf++) {
                        const int v = (c[r + 1][k] >> (16 * hlf)) & 0xffff;
                        const int kk = ((v >> sh) - t.cls) & 31;
                        const int ov = kk < 4 ? clip3i(v + (kk == 0 ? t.off[1] : kk == 1 ? t.off[2] : kk == 2 ? t.off[3] : t.off[4]), 0, maxv) : v;
                        res |= (uint32_t)ov << (16 * hlf);
                    }
                    o[k] = res;
                }
                if (t.tqb) sao_restore_row(tq, t, hs, vs, (int)sizeof(PIX), gx, gy0 + r, c[r + 1], o);
                store8p<PIX>(dp, gx, gy0 + r, o, nvalid);
            }
        }
        return;
    }

    // ---- edge offset ----
    // rows / columns the border rule ("offset 0") or the restore rule can touch: x == 0, x >= w - 2, y == 0, y >= h - 2
    int exact_rows;
    {
        const int cls = t.cls, xs = gx - t.x0, ys = gy0 - t.y0;
        const bool b_l = t.borders & 1, b_t = t.borders & 2, b_r = t.borders & 4, b_b = t.borders & 8, var = t.variant != 0;
        const bool col_exact = !fits || (((b_l && cls != 1) || var) && xs == 0) || (((b_r && cls != 1) || var) && xs + 8 >= t.w - 1);
        const bool top_exact = (b_t && cls != 0) || var, bot_exact = (b_b && cls != 0) || var;
        exact_rows = col_exact ? (1 << SAO_R) - 1 : 0;
#pragma unroll
        for (int r = 0; r < SAO_R; r++) if ((top_exact && ys + r == 0) || (bot_exact && ys + r >= t.h - 2)) exact_rows |= 1 << r;
    }
    const uint32_t tab_lo = (uint32_t)((t.off[1] + 128) & 0xff) | ((uint32_t)((t.off[2] + 128) & 0xff) << 8) |
                            ((uint32_t)((t.off[0] + 128) & 0xff) << 16) | ((uint32_t)((t.off[3] + 128) & 0xff) << 24);
    const uint32_t tab_hi = (uint32_t)((t.off[4] + 128) & 0xff);        // edge_idx[] = {1,2,0,3,4}
    const int lwlh = lw | (lh << 8), hsvsB = hs | (vs << 1) | ((int)sizeof(PIX) << 2);
    switch (t.cls) {
    case 0:  sao_edge_rows<PIX, 0>(sp, dp, rec, cx, cy, lwlh, gx, gy0, nvalid, nrows, maxv, tab_lo, tab_hi, exact_rows, c, sl, sr, tq, t, hsvsB); break;
    case 1:  sao_edge_rows<PIX, 1>(sp, dp, rec, cx, cy, lwlh, gx, gy0, nvalid, nrows, maxv, tab_lo, tab_hi, exact_rows, c, sl, sr, tq, t, hsvsB); break;
    case 2:  sao_edge_rows<PIX, 2>(sp, dp, rec, cx, cy, lwlh, gx, gy0, nvalid, nrows, maxv, tab_lo, tab_hi, exact_rows, c, sl, sr, tq, t, hsvsB); break;
    default: sao_edge_rows<PIX, 3>(sp, dp, rec, cx, cy, lwlh, gx, gy0, nvalid, nrows, maxv, tab_lo, tab_hi, exact_rows, c, sl, sr, tq, t, hsvsB); break;
    }
}

