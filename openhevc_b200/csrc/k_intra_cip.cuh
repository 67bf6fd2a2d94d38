// k_intra_cip.cuh — constrained_intra_pred for the intra stage (K3): hevcpred_template.c:116-163 (which neighbours
// stay candidates) and :185-249 (samples of inter-coded neighbours are replaced by the nearest intra-coded ones).
// Host + device: k_intra runs both functions on lane 0 of the warp that owns the TU (the rules are a sequential scan
// over at most 129 samples, and constrained_intra_pred streams are rare); the CPU suite's warp emulator (tests/emul/warp/)
// runs k_intra, these functions included, on the host against the oracle.
//
// Arrays: top[-1 .. 2n-1], left[-1 .. 2n-1] as plain int pointers (index -1 = the corner), already holding the
// candidate samples (and the reference's memset pattern everywhere else, :159-161) when cip_substitute() is called.
#pragma once
#include "common.cuh"

struct CipDesc {
    const uint32_t *bits;        // one bit per min-PU, row-major (set = intra); nullptr = picture without constrained_intra_pred
    int log2_pu, pu_w, pu_h;     // sps->log2_min_pu_size, min_pu_width, min_pu_height
    int pic_w, pic_h;            // luma picture size
    int hs_c, vs_c;              // chroma subsampling shifts
};

HD bool cip_pu(const CipDesc &c, int px, int py)
{
    const long i = (long)px + (long)py * c.pu_w;          // linear, like tab_mvf[x + y * min_pu_width]
    if (i < 0 || i >= (long)c.pu_w * c.pu_h) return false;
#ifdef __CUDA_ARCH__
    return (__ldg(c.bits + (i >> 5)) >> (i & 31)) & 1;
#else
    return (c.bits[i >> 5] >> (i & 31)) & 1;
#endif
}

struct CipBlock {                // one TU: luma origin, shifts of its plane, size
    int x0, y0, hs, vs, n;
};
// IS_INTRA(dx, dy): the PU under the sample at offset (dx, dy) (in samples of the TU's plane) from the TU origin
HD bool cip_at(const CipDesc &c, const CipBlock &b, int dx, int dy)
{
    return cip_pu(c, (b.x0 + dx * (1 << b.hs)) >> c.log2_pu, (b.y0 + dy * (1 << b.vs)) >> c.log2_pu);
}

// B200_INF_* availability flags before -> after the constrained-intra rule.  Every SECOND PU along an edge is inspected,
// and the vertical PU count is not bumped to 1 for blocks smaller than a PU -- both as the reference does.
HD int cip_flags(const CipDesc &c, const CipBlock &b, int flags)
{
    const int pu = c.log2_pu, sl_h = b.n << b.hs, sl_v = b.n << b.vs;
    const int cnt_v = sl_v >> pu, cnt_h = imax(sl_h >> pu, 1);
    const bool on_x = (b.x0 & ((1 << pu) - 1)) == 0, on_y = (b.y0 & ((1 << pu) - 1)) == 0;
    const int pxl = (b.x0 - 1) >> pu, pyt = (b.y0 - 1) >> pu;
    int out = flags;
    if ((flags & B200_INF_BOTTOM_LEFT) && on_x) {
        const int py = (b.y0 + sl_v) >> pu, m = imin(cnt_v, c.pu_h - py);
        bool any = false;
        for (int i = 0; i < m; i += 2) any |= cip_pu(c, pxl, py + i);
        if (!any) out &= ~B200_INF_BOTTOM_LEFT;
    }
    if ((flags & B200_INF_LEFT) && on_x) {
        const int py = b.y0 >> pu, m = imin(cnt_v, c.pu_h - py);
        bool any = false;
        for (int i = 0; i < m; i += 2) any |= cip_pu(c, pxl, py + i);
        if (!any) out &= ~B200_INF_LEFT;
    }
    if ((flags & B200_INF_UP_LEFT) && !cip_pu(c, pxl, pyt)) out &= ~B200_INF_UP_LEFT;
    if ((flags & B200_INF_UP) && on_y) {
        const int px = b.x0 >> pu, m = imin(cnt_h, c.pu_w - px);
        bool any = false;
        for (int i = 0; i < m; i += 2) any |= cip_pu(c, px + i, pyt);
        if (!any) out &= ~B200_INF_UP;
    }
    if ((flags & B200_INF_UP_RIGHT) && on_y) {
        const int px = (b.x0 + sl_h) >> pu, m = imin(cnt_h, c.pu_w - px);
        bool any = false;
        for (int i = 0; i < m; i += 2) any |= cip_pu(c, px + i, pyt);
        if (!any) out &= ~B200_INF_UP_RIGHT;
    }
    return out;
}

// value the reference's memset(.., 128, .. * sizeof(pixel)) leaves in samples nobody copied (:159-161)
HD int cip_fill_value(int bd) { return bd > 8 ? 0x8080 : 0x80; }

HD void cip_put4(int *p, int v) { p[0] = v; p[1] = v; p[2] = v; p[3] = v; }

// propagate along the top row towards the corner: every sample of an inter PU takes its right neighbour's value
HD void cip_pull_left(const CipDesc &c, const CipBlock &b, int *top, int from, int stop)
{
    for (int i = from; i > stop; i--)
        if (!cip_at(c, b, i - 1, -1)) top[i - 1] = top[i];
}
// bottom-up pass over the left column in groups of four (keyed on the group's first sample)
HD void cip_sweep_up(const CipDesc &c, const CipBlock &b, int *left, int len)
{
    int carry = left[len - 1];
    for (int i = len - 1; i > -1; i -= 4) {
        if (!cip_at(c, b, -1, i - 3)) cip_put4(left + i - 3, carry);
        else carry = left[i - 3];
    }
}

HD void cip_substitute(const CipDesc &c, const CipBlock &b, int flags, int bottom_left_size, int *top, int *left)
{
    const bool bl = flags & B200_INF_BOTTOM_LEFT, lf = flags & B200_INF_LEFT, ul = flags & B200_INF_UP_LEFT;
    const bool up = flags & B200_INF_UP, ur = flags & B200_INF_UP_RIGHT;
    if (!(bl || lf || ul || up || ur)) return;
    const int n = b.n;
    // how far the scans may go: the candidate ranges, cut at the picture edge
    const int span_x = ur ? 2 * n : n, span_y = bl ? 2 * n : n;
    const int len_x = b.x0 + (span_x << b.hs) < c.pic_w ? span_x : (c.pic_w - b.x0) >> b.hs;
    const int len_y = b.y0 + (span_y << b.vs) < c.pic_h ? span_y : (c.pic_h - b.y0) >> b.vs;
    if (bl || lf || ul) {
        int j = n + (bl ? bottom_left_size : 0) - 1;
        while (j > -1 && !cip_at(c, b, -1, j)) j--;
        if (!cip_at(c, b, -1, j)) {                     // nothing intra on the left, corner included: start from the top row
            int k = 0;
            while (k < len_x && !cip_at(c, b, k, -1)) k++;
            cip_pull_left(c, b, top, k, -1);
        }
    } else {
        int k = 0;
        while (k < len_x && !cip_at(c, b, k, -1)) k++;
        if (k > 0) {
            if (b.x0 > 0) cip_pull_left(c, b, top, k, -1);
            else { cip_pull_left(c, b, top, k, 0); top[-1] = top[0]; }
        }
    }
    left[-1] = top[-1];
    if (bl || lf) {                                     // top-down pass over the left column, groups of four
        int carry = left[-1];
        for (int i = 0; i < len_y; i += 4) {
            if (!cip_at(c, b, -1, i)) cip_put4(left + i, carry);
            else carry = left[i + 3];
        }
    }
    if (!lf) for (int i = 0; i < n; i += 4) cip_put4(left + i, left[-1]);
    if (!bl) { const int v = left[n - 1]; for (int i = 0; i < n; i += 4) cip_put4(left + n + i, v); }
    if (b.x0 != 0 && b.y0 != 0) {
        cip_sweep_up(c, b, left, len_y);
        if (!cip_at(c, b, -1, -1)) left[-1] = left[0];
    } else if (b.x0 == 0) {
        for (int i = 0; i < len_y; i += 4) cip_put4(left + i, 0);
    } else {
        cip_sweep_up(c, b, left, len_y);
    }
    top[-1] = left[-1];
    if (b.y0 != 0) {                                    // left-to-right pass over the top row
        int carry = left[-1];
        for (int i = 0; i < len_x; i += 4) {
            if (!cip_at(c, b, i, -1)) cip_put4(top + i, carry);
            else carry = top[i + 3];
        }
    }
}
