// k_deblock.cuh — per-thread code of the deblocking stage (K4).  Host + device: kernels.cu wraps the four phases in the
// __global__ kernel (with __syncthreads() between them); the CPU suite's warp emulator (tests/emul/warp/) runs that
// kernel, these functions included, on the host.
//
// hevc_{h,v}_loop_filter_{luma,chroma}, hevcdsp_template.c:1629-1787.  Both directions in ONE pass: tiles are offset
// by (-4,-4) from the 8x8 edge grid, so every sample an edge reads or writes (<= 4 on either side) belongs to exactly
// one tile: load tile -> all vertical edges -> all horizontal edges -> store, no halo, in place.
//
// The stage is issue-bound, so the unit of work is the reference's own unit of decision, the 4-line segment:
//  * one thread = one segment of one edge (4 lines x 8 samples): the decisions (dp0, dq0, dp3, dq3, strong / normal)
//    are computed once, from lines 0 and 3 it already holds -- no shuffles, no redundant per-line decision arithmetic;
//  * a segment without a PRESENT entry (bs == 0, or outside the picture) costs one grid look-up and nothing else;
//  * the tile is moved with 8- / 16-byte shared-memory accesses (4 x 16 B for a vertical-edge segment, 8 x 8 B for
//    a horizontal one) instead of one 2-byte access per sample.
#pragma once
#include "common.cuh"

#define DBK_TW 128
#define DBK_TH 64
#define DBK_PITCH 136            // uint16 units: 272-byte rows keep every 8-sample group 16-byte aligned
#define DBK_THREADS 256

HD int iabs(int v) { return v < 0 ? -v : v; }

// 4 lines of one luma edge segment: p[l][0..3] = P3..P0, p[l][4..7] = Q0..Q3 of line l
HD void dbk_luma_segment(int (&p)[4][8], int beta, int tc, bool no_p, bool no_q, int bd)
{
    beta <<= bd - 8; tc <<= bd - 8;
    const int dp0 = iabs(p[0][1] - 2 * p[0][2] + p[0][3]), dq0 = iabs(p[0][6] - 2 * p[0][5] + p[0][4]);
    const int dp3 = iabs(p[3][1] - 2 * p[3][2] + p[3][3]), dq3 = iabs(p[3][6] - 2 * p[3][5] + p[3][4]);
    const int d0 = dp0 + dq0, d3 = dp3 + dq3;
    if (d0 + d3 >= beta) return;
    const int tc25 = (tc * 5 + 1) >> 1, maxv = (1 << bd) - 1, beta3 = beta >> 3, beta2 = beta >> 2;
    const int sa0 = iabs(p[0][0] - p[0][3]) + iabs(p[0][7] - p[0][4]), sb0 = iabs(p[0][3] - p[0][4]);
    const int sa3 = iabs(p[3][0] - p[3][3]) + iabs(p[3][7] - p[3][4]), sb3 = iabs(p[3][3] - p[3][4]);
    const bool strong = sa0 < beta3 && sb0 < tc25 && sa3 < beta3 && sb3 < tc25 && (d0 << 1) < beta2 && (d3 << 1) < beta2;
    if (strong) {
        const int t2 = tc << 1;
#pragma unroll
        for (int l = 0; l < 4; l++) {
            const int p3 = p[l][0], p2 = p[l][1], p1 = p[l][2], p0 = p[l][3], q0 = p[l][4], q1 = p[l][5], q2 = p[l][6], q3 = p[l][7];
            if (!no_p) {
                p[l][3] = p0 + clip3i(((p2 + 2 * p1 + 2 * p0 + 2 * q0 + q1 + 4) >> 3) - p0, -t2, t2);
                p[l][2] = p1 + clip3i(((p2 + p1 + p0 + q0 + 2) >> 2) - p1, -t2, t2);
                p[l][1] = p2 + clip3i(((2 * p3 + 3 * p2 + p1 + p0 + q0 + 4) >> 3) - p2, -t2, t2);
            }
            if (!no_q) {
                p[l][4] = q0 + clip3i(((p1 + 2 * p0 + 2 * q0 + 2 * q1 + q2 + 4) >> 3) - q0, -t2, t2);
                p[l][5] = q1 + clip3i(((p0 + q0 + q1 + q2 + 2) >> 2) - q1, -t2, t2);
                p[l][6] = q2 + clip3i(((2 * q3 + 3 * q2 + q1 + q0 + p0 + 4) >> 3) - q2, -t2, t2);
            }
        }
    } else {
        const int th = tc >> 1, side = (beta + (beta >> 1)) >> 3, tc10 = 10 * tc;
        const bool mod_p1 = !no_p && dp0 + dp3 < side, mod_q1 = !no_q && dq0 + dq3 < side;
#pragma unroll
        for (int l = 0; l < 4; l++) {
            const int p2 = p[l][1], p1 = p[l][2], p0 = p[l][3], q0 = p[l][4], q1 = p[l][5], q2 = p[l][6];
            int delta = (9 * (q0 - p0) - 3 * (q1 - p1) + 8) >> 4;
            if (iabs(delta) < tc10) {
                delta = clip3i(delta, -tc, tc);
                if (!no_p) p[l][3] = clip3i(p0 + delta, 0, maxv);
                if (!no_q) p[l][4] = clip3i(q0 - delta, 0, maxv);
                if (mod_p1) p[l][2] = clip3i(p1 + clip3i((((p2 + p0 + 1) >> 1) - p1 + delta) >> 1, -th, th), 0, maxv);
                if (mod_q1) p[l][5] = clip3i(q1 + clip3i((((q2 + q0 + 1) >> 1) - q1 - delta) >> 1, -th, th), 0, maxv);
            }
        }
    }
}

HD void dbk_chroma_segment(int (&p)[4][8], int tc, bool no_p, bool no_q, int bd)
{
    tc <<= bd - 8;
    if (tc <= 0) return;
    const int maxv = (1 << bd) - 1;
#pragma unroll
    for (int l = 0; l < 4; l++) {
        const int p1 = p[l][2], p0 = p[l][3], q0 = p[l][4], q1 = p[l][5];
        const int delta = clip3i((((q0 - p0) * 4) + p1 - q1 + 4) >> 3, -tc, tc);
        if (!no_p) p[l][3] = clip3i(p0 + delta, 0, maxv);
        if (!no_q) p[l][4] = clip3i(q0 - delta, 0, maxv);
    }
}

HD uint16_t dbk_entry(const uint16_t *p)
{
#ifdef __CUDA_ARCH__
    return __ldg(p);
#else
    return *p;
#endif
}
// offset / stride of one of the six grids by register selects (an indexed kernel parameter would go through local memory)
HD int dbk_off(const B200DbkLayout &L, int plane, int dir)
{
    return plane == 0 ? L.off[0][dir] : plane == 1 ? L.off[1][dir] : L.off[2][dir];
}
HD int dbk_stride(const B200DbkLayout &L, int plane, int dir)
{
    return plane == 0 ? L.stride[0][dir] : plane == 1 ? L.stride[1][dir] : L.stride[2][dir];
}

// ---- phase 1 / 4: tile <-> picture, 4 samples (one 8-byte shared-memory word pair) at a time ------------------------
template <typename PIX>
HD void dbk_load(uint16_t *t, const PlaneDesc &pd, int bx, int by, int tid)
{
    const int gx0 = DBK_TW * bx - 4, gy0 = DBK_TH * by - 4;
#pragma unroll
    for (int k = 0; k < DBK_TH * (DBK_TW / 4) / DBK_THREADS; k++) {
        const int u = tid + k * DBK_THREADS;
        const int row = u / (DBK_TW / 4), ux = u % (DBK_TW / 4), gx = gx0 + 4 * ux, gy = gy0 + row;
        uint2 v = make_uint2(0u, 0u);
        if (gx >= 0 && gx < pd.w && gy >= 0 && gy < pd.h) {
            const PIX *s = px_ptr<PIX>(pd, gx, gy);
            if (sizeof(PIX) == 2) v = *reinterpret_cast<const uint2 *>(s);
            else { const uint32_t q = *reinterpret_cast<const uint32_t *>(s); v.x = prmt32(q, 0, 0x4140); v.y = prmt32(q, 0, 0x4342); }
        }
        *reinterpret_cast<uint2 *>(t + row * DBK_PITCH + 4 * ux) = v;
    }
}
template <typename PIX>
HD void dbk_store(const uint16_t *t, const PlaneDesc &pd, int bx, int by, int tid)
{
    const int gx0 = DBK_TW * bx - 4, gy0 = DBK_TH * by - 4;
#pragma unroll
    for (int k = 0; k < DBK_TH * (DBK_TW / 4) / DBK_THREADS; k++) {
        const int u = tid + k * DBK_THREADS;
        const int row = u / (DBK_TW / 4), ux = u % (DBK_TW / 4), gx = gx0 + 4 * ux, gy = gy0 + row;
        if (gx >= 0 && gx < pd.w && gy >= 0 && gy < pd.h) {
            const uint2 v = *reinterpret_cast<const uint2 *>(t + row * DBK_PITCH + 4 * ux);
            PIX *s = px_ptr<PIX>(pd, gx, gy);
            if (sizeof(PIX) == 2) *reinterpret_cast<uint2 *>(s) = v;
            else *reinterpret_cast<uint32_t *>(s) = prmt32(v.x, v.y, 0x6420);
        }
    }
}

// ---- phase 2: vertical edges.  thread = (edge column e of 16, segment s of 16) ------------------------------------------
HD void dbk_vertical(uint16_t *t, const uint16_t *grid, const B200DbkLayout &L, const PlaneDesc &pd, int plane, int bx, int by, int tid, int bd)
{
    const int e = tid & 15, s = tid >> 4;
    const int gxe = DBK_TW * bx + 8 * e, gy = DBK_TH * by - 4 + 4 * s;
    if (!(gxe > 0 && gxe < pd.w && gy >= 0 && gy < pd.h)) return;
    const uint32_t en = dbk_entry(grid + dbk_off(L, plane, 0) + (gy >> 2) * dbk_stride(L, plane, 0) + (gxe >> 3));
    if (!(en & B200_DBK_PRESENT)) return;
    uint16_t *base = t + (4 * s) * DBK_PITCH + 8 * e;
    int p[4][8];
#pragma unroll
    for (int l = 0; l < 4; l++) {
        const uint4 q = *reinterpret_cast<const uint4 *>(base + l * DBK_PITCH);
        p[l][0] = q.x & 0xffff; p[l][1] = q.x >> 16; p[l][2] = q.y & 0xffff; p[l][3] = q.y >> 16;
        p[l][4] = q.z & 0xffff; p[l][5] = q.z >> 16; p[l][6] = q.w & 0xffff; p[l][7] = q.w >> 16;
    }
    if (plane == 0) dbk_luma_segment(p, B200_DBK_BETA(en), B200_DBK_TC(en), B200_DBK_NOP(en), B200_DBK_NOQ(en), bd);
    else            dbk_chroma_segment(p, B200_DBK_TC(en), B200_DBK_NOP(en), B200_DBK_NOQ(en), bd);
#pragma unroll
    for (int l = 0; l < 4; l++)
        *reinterpret_cast<uint4 *>(base + l * DBK_PITCH) = make_uint4((uint32_t)p[l][0] | ((uint32_t)p[l][1] << 16), (uint32_t)p[l][2] | ((uint32_t)p[l][3] << 16),
                                                                     (uint32_t)p[l][4] | ((uint32_t)p[l][5] << 16), (uint32_t)p[l][6] | ((uint32_t)p[l][7] << 16));
}

// ---- phase 3: horizontal edges.  thread = (edge row fr of 8, 4-column segment c of 32) --------------------------------------
HD void dbk_horizontal(uint16_t *t, const uint16_t *grid, const B200DbkLayout &L, const PlaneDesc &pd, int plane, int bx, int by, int tid, int bd)
{
    const int c = tid & 31, fr = tid >> 5;
    const int gye = DBK_TH * by + 8 * fr, gx = DBK_TW * bx - 4 + 4 * c;
    if (!(gye > 0 && gye < pd.h && gx >= 0 && gx < pd.w)) return;
    const uint32_t en = dbk_entry(grid + dbk_off(L, plane, 1) + (gye >> 3) * dbk_stride(L, plane, 1) + (gx >> 2));
    if (!(en & B200_DBK_PRESENT)) return;
    uint16_t *base = t + (8 * fr) * DBK_PITCH + 4 * c;
    int p[4][8];                               // p[column][row]: the same "line" layout as for vertical edges
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const uint2 q = *reinterpret_cast<const uint2 *>(base + i * DBK_PITCH);
        p[0][i] = q.x & 0xffff; p[1][i] = q.x >> 16; p[2][i] = q.y & 0xffff; p[3][i] = q.y >> 16;
    }
    if (plane == 0) dbk_luma_segment(p, B200_DBK_BETA(en), B200_DBK_TC(en), B200_DBK_NOP(en), B200_DBK_NOQ(en), bd);
    else            dbk_chroma_segment(p, B200_DBK_TC(en), B200_DBK_NOP(en), B200_DBK_NOQ(en), bd);
#pragma unroll
    for (int i = 1; i < 7; i++)                // rows P3 and Q3 are never modified
        *reinterpret_cast<uint2 *>(base + i * DBK_PITCH) = make_uint2((uint32_t)p[0][i] | ((uint32_t)p[1][i] << 16), (uint32_t)p[2][i] | ((uint32_t)p[3][i] << 16));
}
