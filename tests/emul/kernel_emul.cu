// kernel_emul.cu — TEST INFRASTRUCTURE.  Runs the per-thread code of the CUDA kernels (the __host__ __device__ functions
// of openhevc_b200/csrc/k_*.cuh, the very source the GPU executes) on the CPU, one "thread" after the other, on host
// memory.  tests/test_kernel_emul_cpu.py compares the result with the oracle: arithmetic identities of the packed
// 16x2 paths, tile / lane geometry and border rules are checked here, without a GPU.  Nothing in the product links this.
#include "../../openhevc_b200/csrc/k_sao.cuh"
#include "../../openhevc_b200/csrc/k_deblock.cuh"
#include "../../openhevc_b200/csrc/k_intra_cip.cuh"
#include <vector>

static void describe(FrameDesc &f, uint8_t *const planes[3], const int pitch[3], int width, int height, int cfi)
{
    for (int p = 0; p < 3; p++) {
        const int hs = p && cfi != 3, vs = p && cfi == 1;
        f.p[p].base = planes[p]; f.p[p].pitch = pitch[p]; f.p[p].w = width >> hs; f.p[p].h = height >> vs;
    }
}

// same geometry as launch_sao() in kernels.cu
extern "C" int emul_sao(const B200SaoRec *grid, uint8_t *const src_planes[3], uint8_t *const dst_planes[3], const int pitch[3],
                        int width, int height, int cfi, int bd, int log2_ctb, const uint32_t *tqb_words)
{
    TqbDesc tq;
    tq.bits = nullptr; tq.log2_pu = 2; tq.pu_w = 0;
    if (tqb_words) { tq.bits = tqb_words + 4; tq.log2_pu = (int)tqb_words[0]; tq.pu_w = (int)tqb_words[1]; }
    FrameDesc src, dst;
    describe(src, src_planes, pitch, width, height, cfi);
    describe(dst, dst_planes, pitch, width, height, cfi);
    const int ctb_w = (width + (1 << log2_ctb) - 1) >> log2_ctb, ctb_h = (height + (1 << log2_ctb) - 1) >> log2_ctb;
    int base[4] = { 0, 0, 0, 0 }, ntx[3];
    for (int p = 0; p < 3; p++) {
        const int hs = p && cfi != 3;
        const int lS = (log2_ctb - hs - 3) < 3 ? (log2_ctb - hs - 3) : 3;
        const int tw = 8 << lS, th = (32 >> lS) * SAO_R;
        ntx[p] = (src.p[p].w + tw - 1) / tw;
        base[p + 1] = base[p] + ntx[p] * ((src.p[p].h + th - 1) / th);
    }
    const int blocks = (base[3] + 7) / 8;
    const int4 tb = make_int4(base[0], base[1], base[2], base[3]);
    const int3 tx = make_int3(ntx[0], ntx[1], ntx[2]);
    for (int warp = 0; warp < blocks * 8; warp++)
        for (int lane = 0; lane < 32; lane++) {
            if (bd > 8) sao_thread<uint16_t>(grid, src, dst, bd, log2_ctb, ctb_w, ctb_h, cfi, tb, tx, tq, warp, lane);
            else        sao_thread<uint8_t>(grid, src, dst, bd, log2_ctb, ctb_w, ctb_h, cfi, tb, tx, tq, warp, lane);
        }
    return 0;
}

// same geometry as launch_deblock() / k_deblock in kernels.cu: phases separated by __syncthreads() there, by loops here
extern "C" int emul_deblock(const uint16_t *grid, uint8_t *const planes[3], const int pitch[3], int width, int height, int cfi, int bd)
{
    FrameDesc f;
    describe(f, planes, pitch, width, height, cfi);
    B200DbkLayout L;
    b200_dbk_layout(width, height, cfi, &L);
    std::vector<uint16_t> tile(DBK_TH * DBK_PITCH + 8);
    uint16_t *t = (uint16_t *)(((uintptr_t)tile.data() + 15) & ~(uintptr_t)15);
    const int gx = (f.p[0].w + 4 + DBK_TW - 1) / DBK_TW, gy = (f.p[0].h + 4 + DBK_TH - 1) / DBK_TH;
    for (int plane = 0; plane < 3; plane++)
        for (int by = 0; by < gy; by++)
            for (int bx = 0; bx < gx; bx++) {
                const PlaneDesc pd = plane_of(f, plane);
                if (DBK_TW * bx - 4 >= pd.w || DBK_TH * by - 4 >= pd.h) continue;
                for (int tid = 0; tid < DBK_THREADS; tid++) { if (bd > 8) dbk_load<uint16_t>(t, pd, bx, by, tid); else dbk_load<uint8_t>(t, pd, bx, by, tid); }
                for (int tid = 0; tid < DBK_THREADS; tid++) dbk_vertical(t, grid, L, pd, plane, bx, by, tid, bd);
                for (int tid = 0; tid < DBK_THREADS; tid++) dbk_horizontal(t, grid, L, pd, plane, bx, by, tid, bd);
                for (int tid = 0; tid < DBK_THREADS; tid++) { if (bd > 8) dbk_store<uint16_t>(t, pd, bx, by, tid); else dbk_store<uint8_t>(t, pd, bx, by, tid); }
            }
    return 0;
}

// constrained_intra_pred: cip_flags() + the gather k_intra performs with those flags (restated here with plain loops: the
// kernel's gather is warp-cooperative and goes through the edge records) + cip_substitute().  Output like
// orc_debug_cip_refs(): index 0 holds [-1].
extern "C" int emul_cip_refs(const uint32_t *cip_words, const B200IntraRec *r, const uint16_t *plane, int stride, int pic_w, int pic_h, int cfi, int bd,
                             int *top65, int *left65, int *flags_out)
{
    CipDesc cd;
    cd.bits = cip_words + 4; cd.log2_pu = (int)cip_words[0]; cd.pu_w = (int)cip_words[1]; cd.pu_h = (int)cip_words[2];
    cd.pic_w = pic_w; cd.pic_h = pic_h; cd.hs_c = cfi != 3; cd.vs_c = cfi == 1;
    CipBlock cb;
    cb.hs = r->plane ? cd.hs_c : 0; cb.vs = r->plane ? cd.vs_c : 0;
    cb.x0 = r->x << cb.hs; cb.y0 = r->y << cb.vs; cb.n = 1 << r->log2;
    const int n = cb.n, fl = cip_flags(cd, cb, r->flags);
    int tbuf[8 + 66 + 8], lbuf[8 + 66 + 8];
    int *top = tbuf + 9, *left = lbuf + 9;
    for (int i = -1; i < 64; i++) top[i] = left[i] = i < 0 ? 128 : cip_fill_value(bd);
    const uint16_t *src = plane + (size_t)r->y * stride + r->x;
    if (fl & B200_INF_UP_LEFT) top[-1] = left[-1] = src[-stride - 1];
    if (fl & B200_INF_UP) for (int i = 0; i < n; i++) top[i] = src[-stride + i];
    if (fl & B200_INF_UP_RIGHT) for (int i = 0; i < n; i++) top[n + i] = src[-stride + n + imin(i, r->top_right_size - 1)];
    if (fl & B200_INF_LEFT) for (int i = 0; i < n; i++) left[i] = src[(size_t)i * stride - 1];
    if (fl & B200_INF_BOTTOM_LEFT) for (int i = 0; i < n; i++) left[n + i] = src[(size_t)(n + imin(i, r->bottom_left_size - 1)) * stride - 1];
    cip_substitute(cd, cb, fl, r->bottom_left_size, top, left);
    for (int i = -1; i < 64; i++) { top65[i + 1] = top[i]; left65[i + 1] = left[i]; }
    *flags_out = fl & 31;
    return 0;
}
