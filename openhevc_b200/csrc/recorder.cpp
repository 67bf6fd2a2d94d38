// recorder.cpp — host side of the drop-in: turns the reference's per-block table calls into
// one packed work-list blob per picture (include/b200hevc_worklist.h).  Pure host code.
//
// Blob layout produced here:  header | deblock grids | SAO grid | coefficient pool (grows while
// recording) | TU4 | TU8 | TU16 | TU32 | INTRA | MC   (lists appended by b200_rec_finish).
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <vector>
#if defined(__SSE2__)
#include <emmintrin.h>
#endif
#include "../../include/b200hevc.h"

struct B200Rec {
    B200Config cfg;
    int pw[3], ph[3];
    B200DbkLayout dbk;
    int ctb_w, ctb_h;
    uint8_t *blob = nullptr;
    bool pinned = false;
    uint64_t cap = 0, cap_max = 0;
    uint32_t off_dbk, off_sao, off_pool;
    uint32_t ncoef = 0;
    uint32_t npark = 0;          // int16 used in the parked-residual pool
    std::vector<B200TuRec> tu[4];
    std::vector<B200IntraRec> intra;
    // MC: whole prediction blocks in decode order, which the device cuts into tiles (k_mc_expand).  mc_tiles[] counts the tiles
    // per bucket of the wire format ([0] tiles of any shape, [1 + B200_MC_SMALL_KEY] tiles of <= 8x8 samples by (chroma, bi)); a
    // block's pad[] holds the index of its first tile in its bucket.  A plain array: this is the hottest append of the recorder.
    struct McBlocks { B200McRec *p = nullptr; size_t n = 0, cap = 0; } mcb;
    uint32_t mc_tiles[5] = { 0, 0, 0, 0, 0 };
    std::vector<uint32_t> cip;   // B200CipHeader + bitmap of a constrained_intra_pred picture (b200_rec_set_cip), else empty
    std::vector<B200CcpRec> ccp; // cross-component prediction records (b200_rec_ccp), executed between the residual and the intra stage
    std::vector<uint32_t> tqb;   // B200CipHeader + bitmap of the PUs restore_tqb_pixels gives their deblocked samples back (b200_rec_set_tqb)
    std::vector<uint32_t> leaf;  // on-device deblocking derivation: one word per ff_hevc_deblocking_boundary_strengths() call (b200_rec_bs_leaf)
    std::vector<uint32_t> dbd;   // ... and the finished B200DbdHeader + arrays (b200_rec_set_dbd), else empty
    int last_intra[3];
    bool any_dbk = false, any_sao = false, open = false;
    bool merged = false;         // holds lists of several recording threads: intra records need re-ordering at finish
    int cur_slot = 0, poc = 0;
    uint8_t ref_slot[16];
    int n_ref = 0;
    uint64_t nbytes = 0;
};

// Decode order -> dependency-level order.  level(TU) = 1 + max level of the 4x4 units it reads (0 for units no intra
// TU of this picture writes); sorting by level (stable) is still a topological order of the intra dependencies, and
// it puts the TUs that can run concurrently next to each other, so the device needs only a small in-flight window
// (few warps polling) to expose all the parallelism the picture has.  O(n * neighbours), host only.
extern "C" int b200_intra_level_order(const B200IntraRec *recs, uint32_t n, int width, int height, int cfi, uint32_t *perm)
{
    if (!recs || !perm) return B200_EINVAL;
    // scratch kept per thread: a picture needs ~3 MB of unit maps, and fresh vectors would be mmap'ed, faulted in and
    // unmapped again for every picture (this runs on the decoding thread, between two pictures)
    static thread_local std::vector<uint32_t> lvl[3], level, start;
    int fs[3];
    for (int p = 0; p < 3; p++) {
        int pw, ph;
        b200_plane_dims(width, height, cfi, p, &pw, &ph);
        fs[p] = pw / 4 + 2;
        // the unit maps stay allocated and CLEAN between calls (a picture with a few intra blocks must not pay for zeroing ~3 MB
        // of maps): whatever a call writes it resets before it returns
        const size_t need = (size_t)fs[p] * (ph / 4 + 2);
        if (lvl[p].size() != need) lvl[p].assign(need, 0);
    }
    auto undo = [&](uint32_t upto) {
        for (uint32_t i = 0; i < upto; i++) {
            const B200IntraRec &r = recs[i];
            const int s = fs[r.plane], u = 1 << (r.log2 - 2), ux = r.x >> 2, uy = r.y >> 2;
            for (int y = 0; y < u; y++) for (int x = 0; x < u; x++) lvl[r.plane][(size_t)(uy + y) * s + ux + x] = 0;
        }
    };
    level.assign(n, 0);
    uint32_t maxl = 0;
    for (uint32_t i = 0; i < n; i++) {
        const B200IntraRec &r = recs[i];
        if (r.plane > 2 || r.log2 < 2 || r.log2 > 5) { undo(i); return B200_EINVAL; }
        std::vector<uint32_t> &L = lvl[r.plane];
        const int s = fs[r.plane], u = 1 << (r.log2 - 2), ux = r.x >> 2, uy = r.y >> 2, nn = 1 << r.log2;
        if ((size_t)(uy + u) * s + ux + u >= L.size() + s) { undo(i); return B200_EINVAL; }
        uint32_t m = 0;
        if ((r.flags & B200_INF_UP_LEFT) && ux && uy) m = L[(size_t)(uy - 1) * s + ux - 1];
        if (uy) {
            int cnt = (r.flags & B200_INF_UP) ? u : 0, from = (r.flags & B200_INF_UP) ? 0 : u;
            if (r.flags & B200_INF_UP_RIGHT) cnt = u + (r.top_right_size + 3) / 4;
            for (int k = from; k < cnt; k++) { const size_t idx = (size_t)(uy - 1) * s + ux + k; if (idx < L.size() && L[idx] > m) m = L[idx]; }
        }
        if (ux) {
            int cnt = (r.flags & B200_INF_LEFT) ? u : 0, from = (r.flags & B200_INF_LEFT) ? 0 : u;
            if (r.flags & B200_INF_BOTTOM_LEFT) cnt = u + (r.bottom_left_size + 3) / 4;
            for (int k = from; k < cnt; k++) { const size_t idx = (size_t)(uy + k) * s + ux - 1; if (idx < L.size() && L[idx] > m) m = L[idx]; }
        }
        (void)nn;
        level[i] = m + 1;
        if (level[i] > maxl) maxl = level[i];
        for (int y = 0; y < u; y++) for (int x = 0; x < u; x++) L[(size_t)(uy + y) * s + ux + x] = m + 1;
    }
    undo(n);
    start.assign(maxl + 2, 0);
    for (uint32_t i = 0; i < n; i++) start[level[i] + 1]++;
    for (uint32_t k = 0; k <= maxl; k++) start[k + 1] += start[k];
    for (uint32_t i = 0; i < n; i++) perm[start[level[i]]++] = i;
    return (int)maxl;
}

extern "C" int b200_rec_set_refs(B200Rec *r, const uint8_t *slots, int n)
{
    if (!r || !r->open || n < 0 || n > 16 || (n && !slots)) return B200_EINVAL;
    r->n_ref = n;
    if (n) memcpy(r->ref_slot, slots, (size_t)n);
    return 0;
}

// Largest blob a picture of this geometry can produce: every sample coded (one int16 each; with 4:4:4 cross-component
// prediction every luma block travels twice, the second time park-only), a TU + intra + MC record and the two-int16 park
// prefix per 4x4 unit, the grids, slack for the section alignment.  The device arenas (engine.cu) and the recorder's
// growth limit are both this number.
extern "C" uint64_t b200_worst_blob_bytes(const B200Config *c)
{
    if (!c) return 0;
    uint64_t samples = 0, luma = 0;
    for (int p = 0; p < 3; p++) { int w, h; b200_plane_dims(c->width, c->height, c->chroma_format_idc, p, &w, &h); samples += (uint64_t)w * h; if (!p) luma = (uint64_t)w * h; }
    B200DbkLayout L;
    b200_dbk_layout(c->width, c->height, c->chroma_format_idc, &L);
    const int ctb = 1 << c->log2_ctb_size;
    const uint64_t nctb = (uint64_t)((c->width + ctb - 1) >> c->log2_ctb_size) * ((c->height + ctb - 1) >> c->log2_ctb_size);
    const uint64_t u = samples / 16 + (c->chroma_format_idc == 3 ? luma / 16 : 0);
    uint64_t v = 4096 + (samples + (c->chroma_format_idc == 3 ? luma : 0)) * 2 + u * (16 + 16 + 32 + 16 + 32) + (uint64_t)L.total * 2 + nctb * 3 * 16 +
                 (samples >> 4) /* CIP + TQB bitmaps */ + luma / 16 * 4 + luma / 64 + luma / 16 + nctb * 2 /* DBD: leaves, QP, PCM, offsets */ + (1u << 20);
    if (c->max_blob_bytes && c->max_blob_bytes < v) v = c->max_blob_bytes;
    return (v + 4095) & ~(uint64_t)4095;
}

// The blob starts at a fraction of the worst case and grows on demand (pinned memory is expensive to allocate: a worst-case
// 4K blob is ~100 MB, a typical one 1-10 MB, and every decoding thread owns two recorders).
static int rec_grow(B200Rec *r, uint64_t need)
{
    if (need <= r->cap) return 0;
    if (need > r->cap_max) return B200_ENOMEM;
    uint64_t cap = r->cap * 2 > need ? r->cap * 2 : need;
    if (cap > r->cap_max) cap = r->cap_max;
    cap = (cap + 4095) & ~(uint64_t)4095;
    uint8_t *nb = r->pinned ? (uint8_t *)b200_host_alloc(cap) : nullptr;
    const bool np = nb != nullptr;
    if (!nb && posix_memalign((void **)&nb, 4096, cap)) return B200_ENOMEM;
    const uint64_t used = (uint64_t)r->off_pool + (uint64_t)r->ncoef * 2;
    memcpy(nb, r->blob, used < r->cap ? used : r->cap);
    if (r->pinned) b200_host_free(r->blob); else free(r->blob);
    r->blob = nb; r->cap = cap; r->pinned = np;
    return 0;
}

extern "C" int b200_rec_create(const B200Config *cfg, B200Rec **out)
{
    if (!cfg || !out || cfg->width < 16 || cfg->height < 16 || (cfg->width & 7) || (cfg->height & 7) ||
        cfg->chroma_format_idc < 1 || cfg->chroma_format_idc > 3 || cfg->bit_depth < 8 || cfg->bit_depth > 12 ||
        cfg->log2_ctb_size < 4 || cfg->log2_ctb_size > 6)
        return B200_EINVAL;
    B200Rec *r = new B200Rec();
    r->cfg = *cfg;
    for (int p = 0; p < 3; p++) b200_plane_dims(cfg->width, cfg->height, cfg->chroma_format_idc, p, &r->pw[p], &r->ph[p]);
    b200_dbk_layout(cfg->width, cfg->height, cfg->chroma_format_idc, &r->dbk);
    const int ctb = 1 << cfg->log2_ctb_size;
    r->ctb_w = (cfg->width + ctb - 1) >> cfg->log2_ctb_size;
    r->ctb_h = (cfg->height + ctb - 1) >> cfg->log2_ctb_size;
    r->off_dbk = 256;
    r->off_sao = b200_align_u32(r->off_dbk + r->dbk.total * 2, 256);
    r->off_pool = b200_align_u32(r->off_sao + (uint32_t)(3 * r->ctb_w * r->ctb_h) * 16, 256);
    r->cap_max = b200_worst_blob_bytes(cfg);
    r->cap = (r->off_pool + (r->cap_max >> 4) + (2u << 20) + 4095) & ~(uint64_t)4095;
    if (r->cap > r->cap_max) r->cap = r->cap_max;
    if (r->cap < (uint64_t)r->off_pool + (1u << 17)) { delete r; return B200_EINVAL; }     // max_blob_bytes below the fixed sections
    r->blob = (uint8_t *)b200_host_alloc(r->cap);           // pinned when a GPU is present
    r->pinned = r->blob != nullptr;
    if (!r->blob && posix_memalign((void **)&r->blob, 4096, r->cap)) { delete r; return B200_ENOMEM; }
    *out = r;
    return 0;
}

extern "C" void b200_rec_destroy(B200Rec *r)
{
    if (!r) return;
    if (r->pinned) b200_host_free(r->blob); else free(r->blob);
    free(r->mcb.p);
    delete r;
}

extern "C" int b200_rec_begin(B200Rec *r, int cur_slot, int poc)
{
    if (!r || cur_slot < 0 || cur_slot > 255) return B200_EINVAL;
    memset(r->blob + r->off_sao, 0, r->off_pool - r->off_sao);            // the deblock grids (1 MB at 4K) are cleared by the first call that needs them
    for (int s = 0; s < 4; s++) r->tu[s].clear();
    r->intra.clear(); r->mcb.n = 0; for (int k = 0; k < 5; k++) r->mc_tiles[k] = 0; r->cip.clear(); r->tqb.clear(); r->ccp.clear(); r->leaf.clear(); r->dbd.clear();
    r->ncoef = 0; r->npark = 0; r->any_dbk = r->any_sao = false;
    r->last_intra[0] = r->last_intra[1] = r->last_intra[2] = -1;
    r->cur_slot = cur_slot; r->poc = poc; r->open = true; r->nbytes = 0; r->n_ref = 0; r->merged = false;
    return 0;
}

static int16_t *pool_take(B200Rec *r, int n, uint32_t *off)
{
    const uint32_t o = (r->ncoef + 7) & ~7u;
    if ((uint64_t)r->off_pool + ((uint64_t)o + n) * 2 + (1u << 16) > r->cap && rec_grow(r, (uint64_t)r->off_pool + ((uint64_t)o + n) * 2 + (1u << 16))) return nullptr;
    *off = o;
    r->ncoef = o + n;
    return (int16_t *)(r->blob + r->off_pool) + o;
}

// intra_linked: -1 = link to the preceding intra record of the plane if it matches (the normal case), 0 = never, 1 = must;
// 2 = PARK the residual without linking it to anything (cross-component prediction), park offset returned in *park_out
static int rec_tu_impl(B200Rec *r, int plane, int x, int y, int log2, int kind, int flags, int col_limit,
                       const int16_t *coeffs, int intra_linked, uint32_t *park_out)
{
    if (!r || !r->open || !coeffs || plane < 0 || plane > 2 || log2 < 2 || log2 > 5 || kind < 0 || kind > B200_TU_PCM) return B200_EINVAL;
    const int n = 1 << log2;
    if (x < 0 || y < 0 || x + n > r->pw[plane] || y + n > r->ph[plane]) return B200_EINVAL;
    if (kind == B200_TU_DST && log2 != 2) return B200_EINVAL;
    // rdpcm follows transform skip or bypass only (hevc_cabac.c:1873,1892); the device would apply it in another order
    if ((flags & (B200_TUF_RDPCM | B200_TUF_RDPCM_VERT)) && kind != B200_TU_SKIP && kind != B200_TU_BYPASS) return B200_EINVAL;
    // residual of an intra TU: park it, the intra kernel adds it right after predicting the block
    const int li = r->last_intra[plane];
    bool link = false;
    if (li >= 0 && kind != B200_TU_PCM) {
        const B200IntraRec &ir = r->intra[li];
        link = ir.x == x && ir.y == y && ir.log2 == log2 && ir.resid_off == B200_NO_RESID;
        if (intra_linked == 0 || intra_linked == 2) link = false;
    }
    const bool park_only = intra_linked == 2 && kind != B200_TU_PCM;
    if (intra_linked == 2 && !park_only) return B200_EINVAL;
    const bool parked = link || park_only;
    // sparse transport (SURVEY.md §8f N1): most dequantised coefficients are zero, send (position, value) pairs.
    // One pass, four coefficients per test (the block is 8-byte aligned scratch of the decoder, hevc.h:1063): pairs are
    // written straight into the pool while they stay below the size of a dense block, else the block is copied whole.
    const int nn = n * n;
    uint32_t off;
    int16_t *dst = pool_take(r, (parked ? 2 : 0) + nn, &off);         // room for either form; the unused tail is given back
    if (!dst) return B200_ENOMEM;
    int16_t *pairs = dst + (parked ? 2 : 0);
    int nnz = 0;
    bool sparse = kind != B200_TU_PCM;
    if (sparse) {
        const int limit = (nn - 1) / 2;                                // sparse iff 2 * nnz < nn
#if defined(__SSE2__)
        {   // eight coefficients per test; the decoder's scratch is mostly zeros
            const __m128i zero = _mm_setzero_si128();
            for (int q = 0; q < nn / 8 && nnz <= limit; q++) {
                const __m128i v = _mm_loadu_si128((const __m128i *)(coeffs + 8 * q));
                unsigned m = 0xffffu & ~(unsigned)_mm_movemask_epi8(_mm_cmpeq_epi16(v, zero));     // two bits per non-zero coefficient
                while (m) {
                    const int k = __builtin_ctz(m) >> 1;
                    m &= ~(3u << (2 * k));
                    if (nnz < limit) { pairs[2 * nnz] = (int16_t)(8 * q + k); pairs[2 * nnz + 1] = coeffs[8 * q + k]; }
                    nnz++;
                }
            }
        }
#else
        if (((uintptr_t)coeffs & 7) == 0) {
            const uint64_t *w = (const uint64_t *)coeffs;
            for (int q = 0; q < nn / 4 && nnz <= limit; q++) {
                const uint64_t v = w[q];
                if (!v) continue;
                for (int k = 0; k < 4; k++) {
                    const int16_t c = (int16_t)(v >> (16 * k));
                    if (c) { if (nnz < limit) { pairs[2 * nnz] = (int16_t)(4 * q + k); pairs[2 * nnz + 1] = c; } nnz++; }
                }
            }
        } else {
            for (int i = 0; i < nn && nnz <= limit; i++)
                if (coeffs[i]) { if (nnz < limit) { pairs[2 * nnz] = (int16_t)i; pairs[2 * nnz + 1] = coeffs[i]; } nnz++; }
        }
#endif
        sparse = nnz <= limit && 2 * nnz < nn;
    }
    r->ncoef = off + (parked ? 2 : 0) + (sparse ? 2 * nnz : nn);      // give the unused tail back
    B200TuRec t;
    memset(&t, 0, sizeof(t));
    if (parked) {
        const uint32_t po = (r->npark + 7) & ~7u;
        r->npark = po + n * n;
        dst[0] = (int16_t)(po & 0xffff); dst[1] = (int16_t)(po >> 16);
        dst += 2;
        if (link) r->intra[li].resid_off = po;
        if (park_out) *park_out = po;
        t.flags |= B200_TUF_PARK;
    }
    if (sparse) t.nnz = (uint16_t)nnz;                                 // the pairs are in place
    else {
        memcpy(dst, coeffs, (size_t)nn * 2);
        t.nnz = B200_TU_DENSE;
    }
    t.x = (uint16_t)x; t.y = (uint16_t)y; t.plane = (uint8_t)plane; t.log2 = (uint8_t)log2; t.kind = (uint8_t)kind;
    t.flags |= (uint8_t)(flags & (B200_TUF_RDPCM | B200_TUF_RDPCM_VERT));
    t.col_limit = (uint8_t)(col_limit < 0 ? 0 : col_limit > 255 ? 255 : col_limit);
    t.coeff_off = off;
    if (intra_linked == 1 && !link) return B200_ESTATE;
    r->tu[log2 - 2].push_back(t);
    return 0;
}

extern "C" int b200_rec_tu(B200Rec *r, int plane, int x, int y, int log2, int kind, int flags, int col_limit,
                           const int16_t *coeffs, int intra_linked)
{
    if (intra_linked < -1 || intra_linked > 1) return B200_EINVAL;
    return rec_tu_impl(r, plane, x, y, log2, kind, flags, col_limit, coeffs, intra_linked, nullptr);
}

extern "C" int b200_rec_tu_parked(B200Rec *r, int plane, int x, int y, int log2, int kind, int flags, int col_limit, const int16_t *coeffs,
                                  uint32_t *park_off)
{
    if (!park_off) return B200_EINVAL;
    return rec_tu_impl(r, plane, x, y, log2, kind, flags, col_limit, coeffs, 2, park_off);
}

// cross-component prediction of one chroma block (hevc.c:1295-1360): see B200CcpRec
extern "C" int b200_rec_ccp(B200Rec *r, int plane, int x, int y, int log2, int scale, uint32_t off_y, int has_c, uint32_t off_c)
{
    if (!r || !r->open || plane < 1 || plane > 2 || log2 < 2 || log2 > 5 || r->cfg.chroma_format_idc != 3) return B200_EINVAL;
    const int n = 1 << log2, as = scale < 0 ? -scale : scale;
    if (x < 0 || y < 0 || x + n > r->pw[plane] || y + n > r->ph[plane] || (as != 1 && as != 2 && as != 4 && as != 8)) return B200_EINVAL;
    if ((uint64_t)off_y + n * n > r->npark || (has_c && (uint64_t)off_c + n * n > r->npark)) return B200_EINVAL;
    B200CcpRec c;
    memset(&c, 0, sizeof(c));
    c.x = (uint16_t)x; c.y = (uint16_t)y; c.plane = (uint8_t)plane; c.log2 = (uint8_t)log2; c.scale = (int8_t)scale;
    c.off_y = off_y; c.off_c = has_c ? off_c : 0;
    c.flags = has_c ? B200_CCPF_HAS_C : 0;
    const int li = r->last_intra[plane];
    if (li >= 0) {                                  // intra predicted block: the intra stage adds the combined residual after predicting
        B200IntraRec &ir = r->intra[li];
        if (ir.x == x && ir.y == y && ir.log2 == log2 && ir.resid_off == B200_NO_RESID) {
            const uint32_t po = (r->npark + 7) & ~7u;
            r->npark = po + n * n;
            ir.resid_off = po;
            c.off_out = po;
            c.flags |= B200_CCPF_TO_PARK;
        }
    }
    r->ccp.push_back(c);
    return 0;
}

extern "C" int b200_rec_pcm(B200Rec *r, int plane, int x, int y, int log2, const int16_t *samples)
{
    return b200_rec_tu(r, plane, x, y, log2, B200_TU_PCM, 0, 0, samples, 0);
}

extern "C" int b200_rec_intra(B200Rec *r, int plane, int x, int y, int log2, int mode, int flags, int top_right_size, int bottom_left_size)
{
    if (!r || !r->open || plane < 0 || plane > 2 || log2 < 2 || log2 > 5 || mode < 0 || mode > 34) return B200_EINVAL;
    const int n = 1 << log2;
    if (x < 0 || y < 0 || (x & 3) || (y & 3) || x + n > r->pw[plane] || y + n > r->ph[plane]) return B200_EINVAL;
    B200IntraRec ir;
    memset(&ir, 0, sizeof(ir));
    ir.x = (uint16_t)x; ir.y = (uint16_t)y; ir.plane = (uint8_t)plane; ir.log2 = (uint8_t)log2; ir.mode = (uint8_t)mode;
    ir.flags = (uint8_t)flags;
    ir.top_right_size = (uint8_t)((flags & B200_INF_UP_RIGHT) ? top_right_size : 0);
    ir.bottom_left_size = (uint8_t)((flags & B200_INF_BOTTOM_LEFT) ? bottom_left_size : 0);
    ir.resid_off = B200_NO_RESID;
    r->last_intra[plane] = (int)r->intra.size();
    r->intra.push_back(ir);
    return 0;
}

static inline int mc_push(B200Rec *r, const B200McRec &t)
{
    B200Rec::McBlocks &bk = r->mcb;
    if (bk.n == bk.cap) {
        const size_t cap = bk.cap ? 2 * bk.cap : 4096;
        B200McRec *np = (B200McRec *)realloc(bk.p, cap * sizeof(B200McRec));
        if (!np) return B200_ENOMEM;
        bk.p = np; bk.cap = cap;
    }
    bk.p[bk.n++] = t;
    return 0;
}
// bucket all tiles of a w x h block fall into, or -1 when they differ (never for the prediction-block shapes of HEVC)
static inline int mc_block_bucket(int w, int h, int flags, int *ntiles)
{
    const int twmax = B200_MC_TILE_WMAX(h);
    int n = 0, bucket = -2;
    for (int tx = 0; tx < w;) {
        const int tw = w - tx > twmax ? twmax : w - tx, maxh = B200_MC_TILE_HMAX(tw);
        for (int ty = 0; ty < h; ty += maxh) {
            const int th = h - ty > maxh ? maxh : h - ty;
            const int k = B200_MC_IS_SMALL(tw, th) ? 1 + B200_MC_SMALL_KEY(flags) : 0;
            if (bucket == -2) bucket = k; else if (bucket != k) bucket = -1;
            n++;
        }
        tx += tw;
    }
    *ntiles = n;
    return bucket;
}

extern "C" int b200_rec_mc(B200Rec *r, const B200McRec *b)
{
    if (!r || !r->open || !b || b->plane > 2 || !b->w || !b->h || b->w > 64 || b->h > 64) return B200_EINVAL;
    if (b->x + b->w > r->pw[b->plane] || b->y + b->h > r->ph[b->plane]) return B200_EINVAL;
    {   // the block travels whole; the device cuts it (k_mc_expand) exactly like the loop below
        int ntiles;
        const int k = mc_block_bucket(b->w, b->h, b->flags, &ntiles);
        if (k >= 0 && r->mc_tiles[k] + (uint32_t)ntiles < (1u << 24)) {
            B200McRec t = *b;
            const uint32_t off = r->mc_tiles[k];
            t.pad[0] = (uint8_t)off; t.pad[1] = (uint8_t)(off >> 8); t.pad[2] = (uint8_t)(off >> 16);
            r->mc_tiles[k] += (uint32_t)ntiles;
            return mc_push(r, t);
        }
    }
    // a block whose tiles differ in kind: every tile as a block of its own.  Tiles of <= 16 x 16 samples (blocks taller than
    // 8 rows: the squarer tile has the smaller filter halo) or <= 32 x 8: one warp each on the device, tiles of <= 8 x 8 four
    // per warp
    const int twmax = B200_MC_TILE_WMAX(b->h);
    for (int tx = 0; tx < b->w;) {
        const int tw = b->w - tx > twmax ? twmax : b->w - tx;
        const int maxh = B200_MC_TILE_HMAX(tw);
        for (int ty = 0; ty < b->h; ty += maxh) {
            const int th = b->h - ty > maxh ? maxh : b->h - ty;
            B200McRec t = *b;
            t.x = (uint16_t)(b->x + tx); t.y = (uint16_t)(b->y + ty); t.w = (uint8_t)tw; t.h = (uint8_t)th;
            t.sx0 = (int16_t)(b->sx0 + tx); t.sy0 = (int16_t)(b->sy0 + ty);
            t.sx1 = (int16_t)(b->sx1 + tx); t.sy1 = (int16_t)(b->sy1 + ty);
            const int k = B200_MC_IS_SMALL(tw, th) ? 1 + B200_MC_SMALL_KEY(b->flags) : 0;
            const uint32_t off = r->mc_tiles[k]++;
            t.pad[0] = (uint8_t)off; t.pad[1] = (uint8_t)(off >> 8); t.pad[2] = (uint8_t)(off >> 16);
            if (int rc = mc_push(r, t)) return rc;
        }
        tx += tw;
    }
    return 0;
}

// Slice / WPP / tile worker threads of ONE picture record into their own B200Rec (lock-free appends, SURVEY.md §8b);
// at frame end the owner folds them into its recorder.  `s` must have its reference table set (b200_rec_set_refs);
// indices are re-mapped into d's table, pool offsets relocated.  s is closed afterwards.
extern "C" int b200_rec_merge(B200Rec *d, B200Rec *s)
{
    if (!d || !s || d == s || !d->open || !s->open) return B200_EINVAL;
    if (d->cfg.width != s->cfg.width || d->cfg.height != s->cfg.height || d->cfg.chroma_format_idc != s->cfg.chroma_format_idc ||
        d->cfg.bit_depth != s->cfg.bit_depth || d->cfg.log2_ctb_size != s->cfg.log2_ctb_size || d->cur_slot != s->cur_slot)
        return B200_EINVAL;
    uint8_t map[16];
    for (int i = 0; i < s->n_ref; i++) {
        int j = 0;
        while (j < d->n_ref && d->ref_slot[j] != s->ref_slot[i]) j++;
        if (j == d->n_ref) {
            if (d->n_ref == 16) return B200_ENOTSUP;
            d->ref_slot[d->n_ref++] = s->ref_slot[i];
        }
        map[i] = (uint8_t)j;
    }
    const uint32_t base = (d->ncoef + 7) & ~7u, pbase = (d->npark + 7) & ~7u;
    if (rec_grow(d, (uint64_t)d->off_pool + ((uint64_t)base + s->ncoef) * 2 + (1u << 16))) return B200_ENOMEM;
    int16_t *dp = (int16_t *)(d->blob + d->off_pool);
    if (s->ncoef) memcpy(dp + base, s->blob + s->off_pool, (size_t)s->ncoef * 2);
    d->ncoef = base + s->ncoef;
    d->npark = pbase + s->npark;
    for (int k = 0; k < 4; k++)
        for (B200TuRec t : s->tu[k]) {
            t.coeff_off += base;
            if (t.flags & B200_TUF_PARK) {
                const uint32_t po = ((uint32_t)(uint16_t)dp[t.coeff_off] | ((uint32_t)(uint16_t)dp[t.coeff_off + 1] << 16)) + pbase;
                dp[t.coeff_off] = (int16_t)(po & 0xffff); dp[t.coeff_off + 1] = (int16_t)(po >> 16);
            }
            d->tu[k].push_back(t);
        }
    for (B200CcpRec c : s->ccp) {
        c.off_y += pbase;
        if (c.flags & B200_CCPF_HAS_C) c.off_c += pbase;
        if (c.flags & B200_CCPF_TO_PARK) c.off_out += pbase;
        d->ccp.push_back(c);
    }
    for (B200IntraRec ir : s->intra) {
        if (ir.resid_off != B200_NO_RESID) ir.resid_off += pbase;
        d->intra.push_back(ir);
    }
    {
        B200Rec::McBlocks &db = d->mcb;
        const B200Rec::McBlocks &sb = s->mcb;
        if (db.n + sb.n > db.cap) {
            const size_t cap = db.n + sb.n + 4096;
            B200McRec *np = (B200McRec *)realloc(db.p, cap * sizeof(B200McRec));
            if (!np) return B200_ENOMEM;
            db.p = np; db.cap = cap;
        }
        for (size_t i = 0; i < sb.n; i++) {
            B200McRec m = sb.p[i];
            if (m.ref0 >= s->n_ref || ((m.flags & B200_MCF_BI) && m.ref1 >= s->n_ref)) return B200_EINVAL;
            m.ref0 = map[m.ref0];
            if (m.flags & B200_MCF_BI) m.ref1 = map[m.ref1];
            // the block's tiles now follow the tiles d already has in that bucket
            int nt;
            const int bk = mc_block_bucket(m.w, m.h, m.flags, &nt);
            if (bk < 0) return B200_EINVAL;
            const uint32_t off = ((uint32_t)m.pad[0] | ((uint32_t)m.pad[1] << 8) | ((uint32_t)m.pad[2] << 16)) + d->mc_tiles[bk];
            if (off + (uint32_t)nt >= (1u << 24)) return B200_ENOTSUP;
            m.pad[0] = (uint8_t)off; m.pad[1] = (uint8_t)(off >> 8); m.pad[2] = (uint8_t)(off >> 16);
            db.p[db.n++] = m;
        }
    }
    for (int k = 0; k < 5; k++) d->mc_tiles[k] += s->mc_tiles[k];
    d->leaf.insert(d->leaf.end(), s->leaf.begin(), s->leaf.end());
    if (s->any_dbk) {
        if (!d->any_dbk) memset(d->blob + d->off_dbk, 0, d->off_sao - d->off_dbk);
        uint16_t *dg = (uint16_t *)(d->blob + d->off_dbk);
        const uint16_t *sg = (const uint16_t *)(s->blob + s->off_dbk);
        for (uint32_t i = 0; i < d->dbk.total; i++) if (sg[i]) dg[i] = sg[i];
        d->any_dbk = true;
    }
    if (s->any_sao) {
        uint64_t *dg = (uint64_t *)(d->blob + d->off_sao);
        const uint64_t *sg = (const uint64_t *)(s->blob + s->off_sao);
        for (int i = 0; i < 3 * d->ctb_w * d->ctb_h; i++) if (sg[2 * i] | sg[2 * i + 1]) { dg[2 * i] = sg[2 * i]; dg[2 * i + 1] = sg[2 * i + 1]; }
        d->any_sao = true;
    }
    d->last_intra[0] = d->last_intra[1] = d->last_intra[2] = -1;
    d->merged = true;
    s->open = false;
    return 0;
}

extern "C" int b200_rec_deblock(B200Rec *r, int plane, int vertical, int x, int y, int beta, const int tc[2],
                                const uint8_t no_p[2], const uint8_t no_q[2])
{
    if (!r || !r->open || plane < 0 || plane > 2 || !tc || !no_p || !no_q) return B200_EINVAL;
    if (x < 0 || y < 0 || x >= r->pw[plane] || y >= r->ph[plane]) return B200_EINVAL;
    if (vertical ? ((x & 7) || (y & 3) || !x) : ((y & 7) || (x & 3) || !y)) return B200_EINVAL;
    if (beta < 0 || beta > 127 || tc[0] < 0 || tc[0] > 63 || tc[1] < 0 || tc[1] > 63) return B200_ENOTSUP;
    if (!r->any_dbk) memset(r->blob + r->off_dbk, 0, r->off_sao - r->off_dbk);
    uint16_t *g = (uint16_t *)(r->blob + r->off_dbk) + r->dbk.off[plane][vertical ? 0 : 1];
    const int gs = (int)r->dbk.stride[plane][vertical ? 0 : 1];
    for (int j = 0; j < 2; j++) {
        const int sx = vertical ? x : x + 4 * j, sy = vertical ? y + 4 * j : y;
        if (sx >= r->pw[plane] || sy >= r->ph[plane]) continue;
        const int idx = vertical ? (sy >> 2) * gs + (sx >> 3) : (sy >> 3) * gs + (sx >> 2);
        g[idx] = B200_DBK_PACK(tc[j], plane ? 0 : beta, no_p[j] != 0, no_q[j] != 0);
    }
    r->any_dbk = true;
    return 0;
}

extern "C" int b200_rec_sao(B200Rec *r, int plane, int x, int y, const B200SaoRec *p)
{
    if (!r || !r->open || !p || plane < 0 || plane > 2 || x < 0 || y < 0 || x >= r->pw[plane] || y >= r->ph[plane]) return B200_EINVAL;
    const int hs = plane && r->cfg.chroma_format_idc != 3, vs = plane && r->cfg.chroma_format_idc == 1;
    const int cx = (x << hs) >> r->cfg.log2_ctb_size, cy = (y << vs) >> r->cfg.log2_ctb_size;
    B200SaoRec *g = (B200SaoRec *)(r->blob + r->off_sao);
    g[(plane * r->ctb_h + cy) * r->ctb_w + cx] = *p;
    if (p->type != B200_SAO_NONE) r->any_sao = true;
    return 0;
}

// pps->constrained_intra_pred_flag: the PU types of the picture (MvField.pred_flag == PF_INTRA, one byte per min-PU,
// row-major), as they stand when every CTB has been parsed
extern "C" int b200_rec_set_cip(B200Rec *r, int log2_min_pu_size, int min_pu_width, int min_pu_height, const uint8_t *is_intra)
{
    if (!r || !r->open || !is_intra || log2_min_pu_size < 2 || log2_min_pu_size > 5 || min_pu_width <= 0 || min_pu_height <= 0 ||
        min_pu_width != (r->cfg.width >> log2_min_pu_size) || min_pu_height != (r->cfg.height >> log2_min_pu_size)) return B200_EINVAL;
    r->cip.assign(B200_CIP_WORDS(min_pu_width, min_pu_height), 0u);
    r->cip[0] = (uint32_t)log2_min_pu_size; r->cip[1] = (uint32_t)min_pu_width; r->cip[2] = (uint32_t)min_pu_height;
    for (int y = 0; y < min_pu_height; y++)
        for (int x = 0; x < min_pu_width; x++)
            if (is_intra[(size_t)y * min_pu_width + x]) { const size_t i = (size_t)y * min_pu_width + x; r->cip[4 + (i >> 5)] |= 1u << (i & 31); }
    return 0;
}

// streams with transquant_bypass_enable / pcm_loop_filter_disabled AND SAO: s->is_pcm[] (one byte per min-PU, row-major,
// non-zero = the PU keeps its deblocked samples), once all CTBs are parsed (hevc_filter.c:163-193)
extern "C" int b200_rec_set_tqb(B200Rec *r, int log2_min_pu_size, int min_pu_width, int min_pu_height, const uint8_t *is_pcm)
{
    if (!r || !r->open || !is_pcm || log2_min_pu_size < 2 || log2_min_pu_size > 5 || min_pu_width <= 0 || min_pu_height <= 0 ||
        min_pu_width != (r->cfg.width >> log2_min_pu_size) || min_pu_height != (r->cfg.height >> log2_min_pu_size)) return B200_EINVAL;
    bool any = false;
    r->tqb.assign(B200_CIP_WORDS(min_pu_width, min_pu_height), 0u);
    r->tqb[0] = (uint32_t)log2_min_pu_size; r->tqb[1] = (uint32_t)min_pu_width; r->tqb[2] = (uint32_t)min_pu_height;
    for (int y = 0; y < min_pu_height; y++)
        for (int x = 0; x < min_pu_width; x++)
            if (is_pcm[(size_t)y * min_pu_width + x]) { const size_t i = (size_t)y * min_pu_width + x; r->tqb[4 + (i >> 5)] |= 1u << (i & 31); any = true; }
    if (!any) r->tqb.clear();                               // nothing to restore in this picture
    return 0;
}

// ---- deblocking parameters derived on the device (B200DbdHeader, include/b200hevc_worklist.h) ----
// one call of ff_hevc_deblocking_boundary_strengths(s, x0, y0, log2_size): top / left = that edge of the block takes part
// (hevc_filter.c:832-839, 870-877, evaluated by the caller)
extern "C" int b200_rec_bs_leaf(B200Rec *r, int x0, int y0, int log2, int top, int left)
{
    if (!r || !r->open || log2 < 2 || log2 > 6 || x0 < 0 || y0 < 0 || (x0 & 3) || (y0 & 3) || x0 >= r->cfg.width || y0 >= r->cfg.height) return B200_EINVAL;
    r->leaf.push_back(B200_DBD_LEAF(x0, y0, log2, top, left));
    return 0;
}

extern "C" int b200_rec_set_dbd(B200Rec *r, const B200DbdInput *in)
{
    if (!r || !r->open || !in || !in->qp_y || !in->ctb_offsets) return B200_EINVAL;
    const int W = r->cfg.width, H = r->cfg.height;
    if (in->log2_min_cb_size < 3 || in->log2_min_cb_size > 6 || in->min_cb_width != (W >> in->log2_min_cb_size) || in->min_cb_height != (H >> in->log2_min_cb_size)) return B200_EINVAL;
    if (in->is_pcm && (in->log2_min_pu_size < 2 || in->log2_min_pu_size > 5 || in->min_pu_width != (W >> in->log2_min_pu_size) || in->min_pu_height != (H >> in->log2_min_pu_size)))
        return B200_EINVAL;
    const uint32_t nqp = (uint32_t)in->min_cb_width * in->min_cb_height, nctb = (uint32_t)r->ctb_w * r->ctb_h;
    const uint32_t npcm = in->is_pcm ? (uint32_t)in->min_pu_width * in->min_pu_height : 0;
    B200DbdHeader h;
    memset(&h, 0, sizeof(h));
    h.flags = in->is_pcm ? B200_DBDF_PCM : 0;
    h.log2_min_cb_size = (uint32_t)in->log2_min_cb_size; h.min_cb_width = (uint32_t)in->min_cb_width; h.min_cb_height = (uint32_t)in->min_cb_height;
    h.log2_min_pu_size = (uint32_t)in->log2_min_pu_size; h.min_pu_width = (uint32_t)in->min_pu_width; h.min_pu_height = (uint32_t)in->min_pu_height;
    h.cb_qp_offset = in->cb_qp_offset; h.cr_qp_offset = in->cr_qp_offset;
    h.n_leaf = (uint32_t)r->leaf.size();
    uint32_t o = sizeof(B200DbdHeader);
    h.off_leaf = o; o = b200_align_u32(o + 4 * h.n_leaf, 16);
    h.off_qp = o;   o = b200_align_u32(o + nqp, 16);
    h.off_ctb = o;  o = b200_align_u32(o + 2 * nctb, 16);
    h.off_pcm = o;  o = b200_align_u32(o + npcm, 16);
    r->dbd.assign(o / 4, 0u);
    uint8_t *b = (uint8_t *)r->dbd.data();
    memcpy(b, &h, sizeof(h));
    if (h.n_leaf) memcpy(b + h.off_leaf, r->leaf.data(), 4 * (size_t)h.n_leaf);
    memcpy(b + h.off_qp, in->qp_y, nqp);
    memcpy(b + h.off_ctb, in->ctb_offsets, 2 * (size_t)nctb);
    if (npcm) memcpy(b + h.off_pcm, in->is_pcm, npcm);
    return 0;
}

extern "C" int b200_rec_finish(B200Rec *r, const void **blob, uint64_t *nbytes)
{
    if (!r || !r->open || !blob || !nbytes) return B200_EINVAL;
    {   // room for the lists and the optional sections behind the pool, before any pointer into the blob is taken
        uint64_t need = b200_align_u32(r->off_pool + ((r->ncoef + 7) & ~7u) * 2, 256);
        for (int s = 0; s < 4; s++) need += ((uint64_t)r->tu[s].size() * 16 + 255) & ~(uint64_t)255;
        need += (((uint64_t)r->intra.size() * 16 + 255) & ~(uint64_t)255) + (((uint64_t)r->mcb.n * 32 + 255) & ~(uint64_t)255);
        need += r->cip.size() * 4 + r->tqb.size() * 4 + r->dbd.size() * 4 + r->ccp.size() * sizeof(B200CcpRec) + 5 * 256;
        if (rec_grow(r, need)) return B200_ENOMEM;
    }
    B200BlobHeader *h = (B200BlobHeader *)r->blob;
    memset(h, 0, sizeof(*h));
    h->magic = B200_BLOB_MAGIC; h->version = B200_BLOB_VERSION;
    h->poc = r->poc;
    h->width = (uint16_t)r->cfg.width; h->height = (uint16_t)r->cfg.height;
    h->chroma_format_idc = (uint8_t)r->cfg.chroma_format_idc; h->bit_depth = (uint8_t)r->cfg.bit_depth;
    h->log2_ctb_size = (uint8_t)r->cfg.log2_ctb_size; h->cur_slot = (uint8_t)r->cur_slot;
    h->flags = (r->any_dbk ? B200_FRAME_HAS_DEBLOCK : 0) | (r->any_sao ? B200_FRAME_HAS_SAO : 0);
    h->n_ref = (uint8_t)r->n_ref;
    memcpy(h->ref_slot, r->ref_slot, (size_t)r->n_ref);
    h->sec[B200_SEC_DBK].off = r->off_dbk; h->sec[B200_SEC_DBK].count = r->any_dbk ? r->dbk.total : 0;
    h->sec[B200_SEC_SAO].off = r->off_sao; h->sec[B200_SEC_SAO].count = r->any_sao ? (uint32_t)(3 * r->ctb_w * r->ctb_h) : 0;
    h->sec[B200_SEC_COEFF].off = r->off_pool; h->sec[B200_SEC_COEFF].count = (r->ncoef + 7) & ~7u;
    uint64_t o = b200_align_u32(r->off_pool + h->sec[B200_SEC_COEFF].count * 2, 256);
    uint64_t need = o;
    for (int s = 0; s < 4; s++) need += ((uint64_t)r->tu[s].size() * 16 + 255) & ~(uint64_t)255;
    need += (((uint64_t)r->intra.size() * 16 + 255) & ~(uint64_t)255) + (((uint64_t)r->mcb.n * 32 + 255) & ~(uint64_t)255);
    if (need > r->cap) return B200_ENOMEM;
    for (int s = 0; s < 4; s++) {
        h->sec[B200_SEC_TU4 + s].off = (uint32_t)o; h->sec[B200_SEC_TU4 + s].count = (uint32_t)r->tu[s].size();
        if (!r->tu[s].empty()) memcpy(r->blob + o, r->tu[s].data(), r->tu[s].size() * 16);
        o = (o + r->tu[s].size() * 16 + 255) & ~(uint64_t)255;
    }
    h->sec[B200_SEC_INTRA].off = (uint32_t)o; h->sec[B200_SEC_INTRA].count = (uint32_t)r->intra.size();
    if (r->merged) {
        // each CTB was recorded by one thread in decode order; CTB raster order between them is a topological order of
        // the intra dependencies (they reach up / left / up-right CTBs only), which is all the level sort needs
        const int lc = r->cfg.log2_ctb_size, cfi = r->cfg.chroma_format_idc, cw = r->ctb_w;
        auto key = [&](const B200IntraRec &a) {
            const int hs = a.plane && cfi != 3, vs = a.plane && cfi == 1;
            return (((int)a.y << vs) >> lc) * cw + (((int)a.x << hs) >> lc);
        };
        std::stable_sort(r->intra.begin(), r->intra.end(), [&](const B200IntraRec &a, const B200IntraRec &b) { return key(a) < key(b); });
    }
    if (!r->intra.empty()) {
        static thread_local std::vector<uint32_t> perm;
        perm.resize(r->intra.size());
        B200IntraRec *dst = (B200IntraRec *)(r->blob + o);
        b200_intra_level_order(r->intra.data(), (uint32_t)r->intra.size(), r->cfg.width, r->cfg.height, r->cfg.chroma_format_idc, perm.data());
        for (size_t i = 0; i < perm.size(); i++) dst[i] = r->intra[perm[i]];
    }
    o = (o + r->intra.size() * 16 + 255) & ~(uint64_t)255;
    h->sec[B200_SEC_MC].off = (uint32_t)o; h->sec[B200_SEC_MC].count = (uint32_t)r->mcb.n;
    if (r->mcb.n) {                                          // whole blocks: mc_big_count stays 0, the tile counts tell the device the cut
        memcpy(r->blob + o, r->mcb.p, r->mcb.n * sizeof(B200McRec));
        for (int k = 0; k < 5; k++) h->mc_tile_count[k] = r->mc_tiles[k];
    }
    o = (o + r->mcb.n * 32 + 255) & ~(uint64_t)255;
    if (!r->cip.empty()) {                                   // constrained_intra_pred picture: B200CipHeader + intra bitmap
        if (o + r->cip.size() * 4 + 256 > r->cap) return B200_ENOMEM;
        h->cip.off = (uint32_t)o; h->cip.count = (uint32_t)r->cip.size();
        h->flags |= B200_FRAME_CIP;
        memcpy(r->blob + o, r->cip.data(), r->cip.size() * 4);
        o = (o + r->cip.size() * 4 + 255) & ~(uint64_t)255;
    }
    if (!r->ccp.empty()) {                                   // cross-component prediction records
        if (o + r->ccp.size() * sizeof(B200CcpRec) + 256 > r->cap) return B200_ENOMEM;
        h->ccp.off = (uint32_t)o; h->ccp.count = (uint32_t)r->ccp.size();
        h->flags |= B200_FRAME_CCP;
        memcpy(r->blob + o, r->ccp.data(), r->ccp.size() * sizeof(B200CcpRec));
        o = (o + r->ccp.size() * sizeof(B200CcpRec) + 255) & ~(uint64_t)255;
    }
    if (!r->tqb.empty() && r->any_sao) {                     // restore_tqb_pixels only ever runs behind the SAO of a CTB
        if (o + r->tqb.size() * 4 + 256 > r->cap) return B200_ENOMEM;
        h->tqb.off = (uint32_t)o; h->tqb.count = (uint32_t)r->tqb.size();
        h->flags |= B200_FRAME_TQB;
        memcpy(r->blob + o, r->tqb.data(), r->tqb.size() * 4);
        o = (o + r->tqb.size() * 4 + 255) & ~(uint64_t)255;
        // mark the CTBs that contain such PUs (all three planes): the SAO kernel looks at the bitmap only there
        const int lp = (int)r->tqb[0], pw_ = (int)r->tqb[1], ph_ = (int)r->tqb[2], per = (1 << r->cfg.log2_ctb_size) >> lp;
        B200SaoRec *g = (B200SaoRec *)(r->blob + r->off_sao);
        for (int cy = 0; cy < r->ctb_h; cy++)
            for (int cx = 0; cx < r->ctb_w; cx++) {
                bool any = false;
                for (int y = cy * per; y < (cy + 1) * per && y < ph_ && !any; y++)
                    for (int x = cx * per; x < (cx + 1) * per && x < pw_; x++) {
                        const size_t i = (size_t)y * pw_ + x;
                        if ((r->tqb[4 + (i >> 5)] >> (i & 31)) & 1) { any = true; break; }
                    }
                if (any) for (int pl = 0; pl < 3; pl++) g[(pl * r->ctb_h + cy) * r->ctb_w + cx].tqb = 1;
            }
    }
    if (!r->dbd.empty()) {                                   // deblocking parameters derived on the device
        if (o + r->dbd.size() * 4 + 256 > r->cap) return B200_ENOMEM;
        h->dbd.off = (uint32_t)o; h->dbd.count = (uint32_t)r->dbd.size();
        memcpy(r->blob + o, r->dbd.data(), r->dbd.size() * 4);
        o = (o + r->dbd.size() * 4 + 255) & ~(uint64_t)255;
        h->flags |= B200_FRAME_HAS_DEBLOCK;
    }
    h->total_bytes = (uint32_t)o;
    r->nbytes = o; r->open = false;
    *blob = r->blob; *nbytes = o;
    return 0;
}
