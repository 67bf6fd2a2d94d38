// kernels.cu — hand-written sm_90a kernels for openHEVC's pixel-reconstruction path.
//
// One kernel per stage, each consuming one section of the per-frame work list
// (include/b200hevc_worklist.h):
//   K1 k_mc        put_hevc_{qpel,epel}{,_uni,_bi}{,_w}        hevcdsp_template.c:610-1609
//   K2 k_residual  idct / idct_dc / idct_4x4_luma / transform_skip / rdpcm + transform_add   :45-326
//   K3 k_intra     intra_pred + pred_planar / pred_dc / pred_angular (+ fused residual add)   hevcpred_template.c:30-538
//   K4 k_deblock   hevc_{h,v}_loop_filter_{luma,chroma}                                       hevcdsp_template.c:1629-1787
//   K5 k_sao       sao_band_filter / sao_edge_filter[0,1]                                     :340-567
// All arithmetic is integer and bit-exact with the reference's C templates (tests/ compare with
// oracle/, which is pinned against the reference build).  No tensor cores: the path is HBM / L2
// bound integer work (SURVEY.md §8d).
#include "common.cuh"
#include <stdlib.h>

// Kernel launches go through one macro so that tests/emul/ can compile this very file for the CPU (warp-lockstep fibers,
// -DB200_EMUL) and run whole pictures through the same launchers; for nvcc it is the plain launch syntax.
#ifndef B200_EMUL
#define B200_LAUNCH(grid, block, smem, stream, ...) __VA_ARGS__<<<grid, block, smem, stream>>>
#endif

// --------------------------------------------------------------------------------------------
// constants
// --------------------------------------------------------------------------------------------
__constant__ int8_t c_qpel[4][8] = { { 0, 0, 0, 64, 0, 0, 0, 0 }, { -1, 4, -10, 58, 17, -5, 1, 0 },
                                     { -1, 4, -11, 40, 40, -11, 4, -1 }, { 0, 1, -5, 17, 58, -10, 4, -1 } };
__constant__ int8_t c_epel[8][4] = { { 0, 64, 0, 0 }, { -2, 58, 10, -2 }, { -4, 54, 16, -2 }, { -6, 46, 28, -4 },
                                     { -4, 36, 36, -4 }, { -4, 28, 46, -6 }, { -2, 16, 54, -4 }, { -2, 10, 58, -2 } };
__constant__ int8_t c_intra_angle[33] = { 32, 26, 21, 17, 13, 9, 5, 2, 0, -2, -5, -9, -13, -17, -21, -26, -32,
                                          -26, -21, -17, -13, -9, -5, -2, 0, 2, 5, 9, 13, 17, 21, 26, 32 };
__constant__ int16_t c_inv_angle[15] = { -4096, -1638, -910, -630, -482, -390, -315, -256, -315, -390, -482, -630, -910, -1638, -4096 };

// HEVC core transform coefficient T[k][n] = sign * |64*sqrt2*cos((2n+1)k*pi/64)| (standardised integers).
// Evaluated at compile time after full unrolling: the butterflies below carry their multipliers as immediates.
__host__ __device__ constexpr int hevc_cos(int j)
{
    constexpr int t[33] = { 64, 90, 90, 90, 89, 88, 87, 85, 83, 82, 80, 78, 75, 73, 70, 67, 64,
                            61, 57, 54, 50, 46, 43, 38, 36, 31, 25, 22, 18, 13, 9, 4, 0 };
    return t[j];
}
__host__ __device__ constexpr int hevc_T(int k, int n)
{
    int m = ((2 * n + 1) * k) & 127;
    return m <= 32 ? hevc_cos(m) : m <= 64 ? -hevc_cos(64 - m) : m < 96 ? -hevc_cos(m - 64) : hevc_cos(128 - m);
}

// --------------------------------------------------------------------------------------------
// K0: work-list validation.  A record is an index into device memory (picture, coefficient pool, reference table):
// none of them is trusted.  Checking ~300 k records costs the submitting host thread about a millisecond per 4K
// picture -- more than everything else it does -- and a few microseconds here, one record per thread.  A bad record
// closes the picture's GATE (gate[1]): every kernel that consumes records returns at once, so a malformed list is
// rejected, not executed; gate[3] latches the failing sections until b200_sync() reports them.
// gate layout (uint32, one per compute lane): [0] K3 ticket, [1] gate of the picture in progress, [2] K3 time-out latch,
// [3] validation latch, [6] tiles k_mc_expand wrote for the picture in progress (k_validate compares and clears it).
// --------------------------------------------------------------------------------------------
// Error latches are mirrored into mapped host memory (engine.cu: gate[4..5] = device address of this lane's host word), so that
// the host can notice a rejected picture without synchronising with the device (b200_poll_errors).
__device__ __forceinline__ void latch_host(uint32_t *gate, uint32_t code)
{
    uint32_t *hp = *reinterpret_cast<uint32_t *const *>(gate + 4);
    if (hp) { *reinterpret_cast<volatile uint32_t *>(hp) = code; __threadfence_system(); }
}

struct ValidateArgs {
    const uint8_t *blob;                 // device copy of the blob
    B200Section sec[B200_SEC_COUNT];
    int pw[3], ph[3];
    uint32_t ncoef, mc_big, n_ref;
    unsigned long long arena_bytes;
    const uint8_t *mc; uint32_t mc_count;      // the MC tile records: the blob's section, or the list k_mc_expand wrote
    uint32_t mc_tag;                           // list k_mc_expand wrote: the stamp every tile of this picture carries; else 0
};

__global__ void __launch_bounds__(256) k_validate(ValidateArgs a, uint32_t *gate)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t bad = 0;
#pragma unroll
    for (int s = B200_SEC_TU4; s <= B200_SEC_TU32; s++) {
        if (i >= a.sec[s].count) continue;
        const int4 raw = __ldg(reinterpret_cast<const int4 *>(a.blob + a.sec[s].off) + i);
        B200TuRec t;
        memcpy(&t, &raw, 16);
        const int n = 4 << (s - B200_SEC_TU4);
        const int pl = t.plane > 2 ? 0 : t.plane;
        const int pw = pl == 0 ? a.pw[0] : pl == 1 ? a.pw[1] : a.pw[2], ph = pl == 0 ? a.ph[0] : pl == 1 ? a.ph[1] : a.ph[2];
        const unsigned long long need = (unsigned long long)t.coeff_off + ((t.flags & B200_TUF_PARK) ? 2 : 0) + (t.nnz == B200_TU_DENSE ? n * n : 2ull * t.nnz);
        if (t.plane > 2 || (1 << t.log2) != n || t.x + n > pw || t.y + n > ph || need > a.ncoef ||
            (t.nnz != B200_TU_DENSE && (int)t.nnz > n * n) || (t.kind == B200_TU_PCM && t.nnz != B200_TU_DENSE) ||
            t.kind > B200_TU_PCM || (t.kind == B200_TU_DST && n != 4) ||
            ((t.flags & (B200_TUF_RDPCM | B200_TUF_RDPCM_VERT)) && t.kind != B200_TU_SKIP && t.kind != B200_TU_BYPASS))
            bad |= 1u << s;
    }
    if (i < a.sec[B200_SEC_INTRA].count) {
        const int4 raw = __ldg(reinterpret_cast<const int4 *>(a.blob + a.sec[B200_SEC_INTRA].off) + i);
        B200IntraRec r;
        memcpy(&r, &raw, 16);
        const int n = 1 << (r.log2 & 7);
        const int pl = r.plane > 2 ? 0 : r.plane;
        const int pw = pl == 0 ? a.pw[0] : pl == 1 ? a.pw[1] : a.pw[2], ph = pl == 0 ? a.ph[0] : pl == 1 ? a.ph[1] : a.ph[2];
        if (r.plane > 2 || r.log2 < 2 || r.log2 > 5 || r.mode > 34 || (r.x & 3) || (r.y & 3) || r.x + n > pw || r.y + n > ph ||
            (r.resid_off != B200_NO_RESID && ((unsigned long long)r.resid_off + n * n) * 2 > a.arena_bytes) ||
            ((r.flags & B200_INF_UP_RIGHT) && (r.top_right_size < 1 || r.top_right_size > n || r.x + n + r.top_right_size > pw)) ||
            ((r.flags & B200_INF_BOTTOM_LEFT) && (r.bottom_left_size < 1 || r.bottom_left_size > n || r.y + n + r.bottom_left_size > ph)) ||
            ((r.flags & (B200_INF_UP | B200_INF_UP_RIGHT | B200_INF_UP_LEFT)) && r.y == 0) ||
            ((r.flags & (B200_INF_LEFT | B200_INF_BOTTOM_LEFT | B200_INF_UP_LEFT)) && r.x == 0))
            bad |= 1u << B200_SEC_INTRA;
    }
    if (i < a.mc_count) {
        const int4 *p = reinterpret_cast<const int4 *>(a.mc) + 2 * (size_t)i;
        const int4 ra = __ldg(p), rb = __ldg(p + 1);
        B200McRec m;
        memcpy(&m, &ra, 16);
        memcpy(reinterpret_cast<uint8_t *>(&m) + 16, &rb, 16);
        const int maxf = (m.flags & B200_MCF_CHROMA) ? 7 : 3;
        const int pl = m.plane > 2 ? 0 : m.plane;
        const int pw = pl == 0 ? a.pw[0] : pl == 1 ? a.pw[1] : a.pw[2], ph = pl == 0 ? a.ph[0] : pl == 1 ? a.ph[1] : a.ph[2];
        if (m.plane > 2 || !m.w || !m.h || m.w > 32 || m.w * m.h > 256 || m.x + m.w > pw || m.y + m.h > ph ||
            m.ref0 >= a.n_ref || ((m.flags & B200_MCF_BI) && m.ref1 >= a.n_ref) ||
            (m.frac0 & 15) > maxf || (m.frac0 >> 4) > maxf || (m.frac1 & 15) > maxf || (m.frac1 >> 4) > maxf || m.denom > 7 ||
            ((m.w > 16) ? m.h > 8 : m.h > 16) || (i >= a.mc_big && !B200_MC_IS_SMALL(m.w, m.h)) ||
            (a.mc_tag && ((uint32_t)rb.w >> 8) != a.mc_tag))
            bad |= 1u << B200_SEC_MC;
    }
    // A place of the tile list that no block of this picture wrote still holds a tile of an earlier picture (without this
    // picture's stamp, rejected above).  Every place stamped and as many tiles written as there are places: no place was
    // written twice either, i.e. no two blocks claimed the same places.
    if (i == 0 && a.mc_tag) {
        if (gate[6] != a.mc_count) bad |= 1u << B200_SEC_MC;
        gate[6] = 0;
    }
    if (bad) { gate[1] = 1u; atomicOr(gate + 3, bad); latch_host(gate, bad); }
}

int launch_validate(cudaStream_t st, const uint8_t *blob_dev, const B200BlobHeader &h, const int pw[3], const int ph[3], unsigned long long arena_bytes, uint32_t *gate,
                    const B200McRec *mc_tiles, uint32_t mc_count, uint32_t mc_big, uint32_t mc_tag)
{
    ValidateArgs a;
    a.blob = blob_dev;
    a.mc = mc_tiles ? reinterpret_cast<const uint8_t *>(mc_tiles) : blob_dev + h.sec[B200_SEC_MC].off;
    a.mc_count = mc_tiles ? mc_count : h.sec[B200_SEC_MC].count;
    uint32_t most = a.mc_count;
    for (int s = 0; s < B200_SEC_COUNT; s++) { a.sec[s] = h.sec[s]; if (s >= B200_SEC_TU4 && s <= B200_SEC_INTRA && h.sec[s].count > most) most = h.sec[s].count; }
    for (int p = 0; p < 3; p++) { a.pw[p] = pw[p]; a.ph[p] = ph[p]; }
    a.ncoef = h.sec[B200_SEC_COEFF].count; a.mc_big = mc_tiles ? mc_big : h.mc_big_count; a.n_ref = h.n_ref; a.arena_bytes = arena_bytes;
    a.mc_tag = mc_tiles ? mc_tag : 0;
    if (!most) return 0;
    B200_LAUNCH((most + 255) / 256, 256, 0, st, k_validate)(a, gate);
    return 1;
}

// --------------------------------------------------------------------------------------------
// K2: residual.  N lanes per TU (one column, then one row each); 32/N TUs per warp.
// 1-D inverse DCT as register butterflies (even/odd decomposition), transposition through
// a padded shared tile.  The int16 clip between the two stages is kept (Appendix A.2).
// --------------------------------------------------------------------------------------------
template <int N> struct Idct1D {
    static constexpr int STEP = 32 / N;
    __device__ __forceinline__ static void run(const int (&v)[N], int (&out)[N])
    {
        int ein[N / 2], e[N / 2];
#pragma unroll
        for (int j = 0; j < N / 2; j++) ein[j] = v[2 * j];
        Idct1D<N / 2>::run(ein, e);
#pragma unroll
        for (int k = 0; k < N / 2; k++) {
            int o = 0;
#pragma unroll
            for (int j = 1; j < N; j += 2) o += hevc_T(j * STEP, k) * v[j];
            out[k] = e[k] + o;
            out[N - 1 - k] = e[k] - o;
        }
    }
};
template <> struct Idct1D<4> {
    __device__ __forceinline__ static void run(const int (&v)[4], int (&out)[4])
    {
        const int e0 = 64 * (v[0] + v[2]), e1 = 64 * (v[0] - v[2]);
        const int o0 = 83 * v[1] + 36 * v[3], o1 = 36 * v[1] - 83 * v[3];
        out[0] = e0 + o0; out[1] = e1 + o1; out[2] = e1 - o1; out[3] = e0 - o0;
    }
};

// which inputs the reference's pruned butterflies read for a given `end` (hevcdsp_template.c:223-277)
template <int N> __device__ __forceinline__ bool idct_keep(int j, int end)
{
    if (N == 4) return true;
    if (N == 8 || N == 16) return !(j & 1) || j < end;
    if (j & 1) return j < end;
    if ((j & 3) == 2) return (j >> 1) < end / 2;
    return true;
}

template <int N> __device__ __forceinline__ void dst4_1d(const int (&v)[N], int (&out)[N])
{
    if (N == 4) {   // inverse DST-VII, hevcdsp_template.c:170-183
        const int c0 = v[0] + v[2], c1 = v[2] + v[3], c2 = v[0] - v[3], c3 = 74 * v[1];
        out[0] = 29 * c0 + 55 * c1 + c3;
        out[1] = 55 * c2 - 29 * c1 + c3;
        out[2] = 74 * (v[0] - v[2] + v[3]);
        out[3] = 55 * c0 + 29 * c2 - c3;
    }
}

#define RESID_TILE_INTS (32 * 33)      // per warp: the largest padded tile (one 32x32 TU)

// One warp's share of the TUs of size N: `blk` = index of the 4-warp block within the list of this size.
template <typename PIX, int N>
__device__ __forceinline__ void residual_warp(const B200TuRec *__restrict__ recs, int count, const int16_t *__restrict__ pool,
                                              int16_t *__restrict__ parked, const FrameDesc &f, int bd, int *tile_w, int blk)
{
    constexpr int G = 32 / N;            // TUs per warp
    constexpr int TS = N * (N + 1);      // padded tile
    static_assert(G * TS <= RESID_TILE_INTS, "tile buffer too small");
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane / N, col = lane % N;
    const int ti = (blk * 4 + warp) * G + g;
    const bool active = ti < count;
    int *tile = tile_w + g * TS;

    B200TuRec rec;
    if (active) {
        const int4 raw = __ldg(reinterpret_cast<const int4 *>(recs + ti));
        memcpy(&rec, &raw, 16);
    } else {
        memset(&rec, 0, 16);
        rec.kind = B200_TU_BYPASS;
    }
    const int16_t *c = pool + rec.coeff_off;
    const int kind = rec.kind;
    uint32_t park_off = 0;
    if (active && (rec.flags & B200_TUF_PARK)) { park_off = (uint32_t)(uint16_t)c[0] | ((uint32_t)(uint16_t)c[1] << 16); c += 2; }
    const bool sparse = rec.nnz != B200_TU_DENSE;
    int v[N], t[N];
    // sparse transport: (position, value) pairs are scattered into the zeroed tile, then every lane picks up its column
#pragma unroll
    for (int j = 0; j < N; j++) tile[j * (N + 1) + col] = 0;
    __syncwarp();
    if (active && sparse)
        for (int e = col; e < rec.nnz; e += N) {
            const int pos = (uint16_t)c[2 * e] & (N * N - 1);
            tile[(pos / N) * (N + 1) + (pos % N)] = c[2 * e + 1];
        }
    __syncwarp();
    const int c00 = !active ? 0 : sparse ? tile[0] : c[0];
    if (active && !sparse) {
#pragma unroll
        for (int j = 0; j < N; j++) v[j] = c[j * N + col];
    } else {
#pragma unroll
        for (int j = 0; j < N; j++) v[j] = tile[j * (N + 1) + col];
    }
    __syncwarp();
    const int lim_row = min((int)rec.col_limit, N);
    // ---- first stage (columns) ----
    if (kind == B200_TU_IDCT) {
        int lim = min((int)rec.col_limit + 4, N);
        if (lim < N && col > 0) lim -= 4 * ((col - 1) >> 2);
#pragma unroll
        for (int j = 0; j < N; j++) if (!idct_keep<N>(j, lim)) v[j] = 0;
        int o[N];
        Idct1D<N>::run(v, o);
#pragma unroll
        for (int j = 0; j < N; j++) t[j] = clip16i((o[j] + 64) >> 7);
    } else if (kind == B200_TU_DST) {
        int o[N];
        dst4_1d<N>(v, o);
#pragma unroll
        for (int j = 0; j < N; j++) t[j] = clip16i((o[j] + 64) >> 7);
    } else if (kind == B200_TU_DC) {
        const int shift = 14 - bd;
        const int dc = active ? (((c00 + 1) >> 1) + (1 << (shift - 1))) >> shift : 0;
#pragma unroll
        for (int j = 0; j < N; j++) t[j] = (int16_t)dc;
    } else if (kind == B200_TU_SKIP) {
        const int shift = 15 - bd - rec.log2;
#pragma unroll
        for (int j = 0; j < N; j++) t[j] = shift > 0 ? (int16_t)((v[j] + (1 << (shift - 1))) >> shift) : (int16_t)(v[j] << -shift);
    } else {
#pragma unroll
        for (int j = 0; j < N; j++) t[j] = v[j];
    }
    if ((rec.flags & (B200_TUF_RDPCM | B200_TUF_RDPCM_VERT)) == (B200_TUF_RDPCM | B200_TUF_RDPCM_VERT)) {
#pragma unroll
        for (int j = 1; j < N; j++) t[j] = (int16_t)(t[j] + t[j - 1]);   // running sum down the column, int16 wrap
    }
    // ---- transpose ----
#pragma unroll
    for (int j = 0; j < N; j++) tile[j * (N + 1) + col] = t[j];
    __syncwarp();
#pragma unroll
    for (int j = 0; j < N; j++) v[j] = tile[col * (N + 1) + j];          // lane now owns row `col`
    // ---- second stage (rows) ----
    if (kind == B200_TU_IDCT || kind == B200_TU_DST) {
        int o[N];
        if (kind == B200_TU_IDCT) {
#pragma unroll
            for (int j = 0; j < N; j++) if (!idct_keep<N>(j, lim_row)) v[j] = 0;
            Idct1D<N>::run(v, o);
        } else {
            dst4_1d<N>(v, o);
        }
        const int shift = 20 - bd, add = 1 << (shift - 1);
#pragma unroll
        for (int j = 0; j < N; j++) t[j] = clip16i((o[j] + add) >> shift);
    } else {
#pragma unroll
        for (int j = 0; j < N; j++) t[j] = v[j];
    }
    if ((rec.flags & (B200_TUF_RDPCM | B200_TUF_RDPCM_VERT)) == B200_TUF_RDPCM) {
#pragma unroll
        for (int j = 1; j < N; j++) t[j] = (int16_t)(t[j] + t[j - 1]);   // running sum along the row
    }
    __syncwarp();
#pragma unroll
    for (int j = 0; j < N; j++) tile[col * (N + 1) + j] = t[j];          // tile[row][x]
    __syncwarp();
    if (!active) return;
    // ---- output: rows of N consecutive samples per TU ----
    if (rec.flags & B200_TUF_PARK) {
        int16_t *pk = parked + park_off;           // the blob stays read-only: parked residuals live in their own pool
#pragma unroll
        for (int y = 0; y < N; y++) pk[y * N + col] = (int16_t)tile[y * (N + 1) + col];
    } else {
        const PlaneDesc pd = plane_of(f, rec.plane);
        const int maxv = (1 << bd) - 1;
        const bool pcm = kind == B200_TU_PCM;
#pragma unroll
        for (int y = 0; y < N; y++) {
            PIX *d = px_ptr<PIX>(pd, rec.x + col, rec.y + y);
            const int r = tile[y * (N + 1) + col];
            *d = (PIX)(pcm ? r : clip3i((int)*d + r, 0, maxv));
        }
    }
}

// All four TU sizes in ONE launch: separate launches ran back to back although none of them fills the machine (the
// 32x32 list is a few hundred CTAs).  Largest TUs first, so that the long-running warps
// start first and the small ones fill in behind them.
struct ResidualLists {
    const B200TuRec *recs[4];            // 4x4, 8x8, 16x16, 32x32
    int count[4];
    int nblk[4];                         // CTAs of 4 warps per list
};

template <typename PIX>
__global__ void __launch_bounds__(128) k_residual(ResidualLists L, const int16_t *__restrict__ pool, int16_t *__restrict__ parked, FrameDesc f, int bd,
                                                  const uint32_t *__restrict__ gate)
{
    if (__ldg(gate + 1)) return;         // the picture's work list failed validation (k_validate)
    __shared__ int tile_s[4][RESID_TILE_INTS];
    int *tile_w = tile_s[threadIdx.x >> 5];
    int b = blockIdx.x;
    if (b < L.nblk[3]) { residual_warp<PIX, 32>(L.recs[3], L.count[3], pool, parked, f, bd, tile_w, b); return; }
    b -= L.nblk[3];
    if (b < L.nblk[2]) { residual_warp<PIX, 16>(L.recs[2], L.count[2], pool, parked, f, bd, tile_w, b); return; }
    b -= L.nblk[2];
    if (b < L.nblk[1]) { residual_warp<PIX, 8>(L.recs[1], L.count[1], pool, parked, f, bd, tile_w, b); return; }
    b -= L.nblk[1];
    residual_warp<PIX, 4>(L.recs[0], L.count[0], pool, parked, f, bd, tile_w, b);
}


// --------------------------------------------------------------------------------------------
// K2b: cross-component prediction (4:4:4 range extension; hevc.c:1295-1360, hevc_cabac.c:1942-1948), only launched for pictures
// that carry B200CcpRec records.  chroma residual = own residual (parked by K2, if the block has coefficients) +
// (res_scale_val * luma residual) >> 3 (the luma block parked by K2 through a second, unlinked record), in int16 like the
// reference's coefficient arrays; added to the picture like transform_add, or parked again for the intra stage.
// The records are validated here (one CTA per record): a bad one closes the picture's gate like K0 does.
// --------------------------------------------------------------------------------------------
template <typename PIX>
__global__ void __launch_bounds__(128) k_ccp(const B200CcpRec *__restrict__ recs, int count, int16_t *__restrict__ parked, FrameDesc f, int bd,
                                             uint32_t *gate, unsigned long long arena_bytes)
{
    if (__ldg(gate + 1)) return;
    const int i = blockIdx.x;
    if (i >= count) return;
    const int4 *rp = reinterpret_cast<const int4 *>(recs + i);
    const int4 ra = __ldg(rp);
    const int x = ra.x & 0xffff, y = (unsigned)ra.x >> 16;
    const int plane = ra.y & 0xff, log2 = (ra.y >> 8) & 0xff, scale = (int8_t)((ra.y >> 16) & 0xff), flags = (unsigned)ra.y >> 24;
    const uint32_t off_y = (uint32_t)ra.z, off_c = (uint32_t)ra.w, off_out = (uint32_t)__ldg(reinterpret_cast<const int *>(rp + 1));
    const int n = 1 << (log2 & 7), nn = n * n;
    const int pl = plane == 2 ? 2 : 1;
    const PlaneDesc pd = plane_of(f, pl);
    const unsigned long long cap = arena_bytes / 2;                           // int16 entries of the parked pool
    if ((plane != 1 && plane != 2) || log2 < 2 || log2 > 5 || x + n > pd.w || y + n > pd.h || (unsigned long long)off_y + nn > cap ||
        ((flags & B200_CCPF_HAS_C) && (unsigned long long)off_c + nn > cap) || ((flags & B200_CCPF_TO_PARK) && (unsigned long long)off_out + nn > cap)) {
        if (threadIdx.x == 0) { gate[1] = 1u; atomicOr(gate + 3, 1u << B200_SEC_COUNT); latch_host(gate, 1u << B200_SEC_COUNT); }
        return;
    }
    const int maxv = (1 << bd) - 1;
    for (int k = threadIdx.x; k < nn; k += 128) {
        const int own = (flags & B200_CCPF_HAS_C) ? parked[off_c + k] : 0;
        const int r = (int16_t)(own + ((scale * (int)parked[off_y + k]) >> 3));
        if (flags & B200_CCPF_TO_PARK) parked[off_out + k] = (int16_t)r;
        else {
            PIX *d = px_ptr<PIX>(pd, x + (k & (n - 1)), y + (k >> log2));
            *d = (PIX)clip3i((int)*d + r, 0, maxv);
        }
    }
}

// --------------------------------------------------------------------------------------------
// K1: inter prediction.  One warp per tile record (<= 256 samples, <= 32 wide).
// Reference window staged in shared memory with clamped addressing (== emulated_edge_mc),
// separable FIR with the 14-bit intermediate of the reference.
// --------------------------------------------------------------------------------------------
#define MC_WIN_MAX 640      // (32+7+1) x 15 = 600, (16+7+1) x 23 = 552, + slack for padded reads
#define MC_TMP_MAX 512      // 15 x 32, 23 x 16
template <int GS> struct McSmem;
template <> struct McSmem<32> { static constexpr int WIN = MC_WIN_MAX, TMP = MC_TMP_MAX; };
template <> struct McSmem<8>  { static constexpr int WIN = 256 /* 15 x 16 */, TMP = 160 /* 15 x 8 */; };

// K1a: prediction blocks -> tiles.  The host records ONE record per table call (a block of up to 64x64 samples, hevc.c:1641-1949)
// instead of cutting it into up to 24 tiles itself (6-9 % of the hooked decoder's host time, and 60 % of the upload of a lightly
// coded picture): one thread per block writes the block's tiles -- the cut of B200_MC_TILE_WMAX / _HMAX, the one definition the
// recorder's fallback uses too -- into the lane's tile list at the place the host reserved (bucket base + B200McRec.pad), laid
// out like a B200_SEC_MC section in tile mode.  Only memory safety is checked here (index inside the bucket); the tiles are
// validated like any other list by k_validate, which runs behind this kernel.  Each tile carries the picture's stamp in its pad
// bytes (k_mc reads no pad), and gate[6] counts the tiles written: with both, k_validate also rejects a list whose blocks leave
// places of the tile list unwritten or claim the same places twice.
struct McExpandArgs {
    const B200McRec *blocks; uint32_t n_blocks;
    B200McRec *tiles;
    uint32_t base[5], count[5];
    uint32_t tag;                        // 24 bits, never 0
};
__global__ void __launch_bounds__(256) k_mc_expand(McExpandArgs a, uint32_t *gate)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const int4 *p = reinterpret_cast<const int4 *>(a.blocks) + 2 * (size_t)min(i, a.n_blocks - 1);
    const int4 ra = __ldg(p), rb = __ldg(p + 1);
    const int x = ra.x & 0xffff, y = (unsigned)ra.x >> 16, w = ra.y & 0xff, h = (ra.y >> 8) & 0xff, flags = (unsigned)ra.y >> 24;
    const int sx0 = (int16_t)(ra.z & 0xffff), sy0 = (int16_t)((unsigned)ra.z >> 16), sx1 = (int16_t)(ra.w & 0xffff), sy1 = (int16_t)((unsigned)ra.w >> 16);
    const uint32_t off = ((unsigned)rb.w >> 8) & 0xffffff;            // pad[0..2]
    bool bad = !w || !h || w > 64 || h > 64;
    int bucket = -1;
    uint32_t k = 0;
    if (i < a.n_blocks && !bad) {
        const int twmax = B200_MC_TILE_WMAX(h);
        for (int tx = 0; tx < w && !bad;) {
            const int tw = w - tx > twmax ? twmax : w - tx, maxh = B200_MC_TILE_HMAX(tw);
            for (int ty = 0; ty < h; ty += maxh) {
                const int th = h - ty > maxh ? maxh : h - ty;
                const int b = B200_MC_IS_SMALL(tw, th) ? 1 + B200_MC_SMALL_KEY(flags) : 0;
                if (bucket < 0) bucket = b;
                const uint32_t cnt = bucket == 0 ? a.count[0] : bucket == 1 ? a.count[1] : bucket == 2 ? a.count[2] : bucket == 3 ? a.count[3] : a.count[4];
                const uint32_t bs = bucket == 0 ? a.base[0] : bucket == 1 ? a.base[1] : bucket == 2 ? a.base[2] : bucket == 3 ? a.base[3] : a.base[4];
                if (b != bucket || off + k >= cnt) { bad = true; break; }
                int4 ta = ra, tb = rb;
                ta.x = ((x + tx) & 0xffff) | ((y + ty) << 16);
                ta.y = (ra.y & 0xffff0000) | tw | (th << 8);
                ta.z = ((sx0 + tx) & 0xffff) | ((sy0 + ty) << 16);
                ta.w = ((sx1 + tx) & 0xffff) | ((sy1 + ty) << 16);
                tb.w = (rb.w & 0xff) | (int)(a.tag << 8);                 // denom; pad = the picture's stamp
                int4 *o = reinterpret_cast<int4 *>(a.tiles + bs + off + k);
                o[0] = ta; o[1] = tb;
                k++;
            }
            tx += tw;
        }
    }
    uint32_t n = k;                                                   // tiles written by the warp: one atomic per warp
#pragma unroll
    for (int s = 16; s; s >>= 1) n += __shfl_xor_sync(0xffffffffu, n, s);
    if ((threadIdx.x & 31) == 0 && n) atomicAdd(gate + 6, n);
    if (i < a.n_blocks && bad) { gate[1] = 1u; atomicOr(gate + 3, 1u << B200_SEC_MC); latch_host(gate, 1u << B200_SEC_MC); }
}
int launch_mc_expand(cudaStream_t st, const B200McRec *blocks, uint32_t n_blocks, B200McRec *tiles, const uint32_t count[5], uint32_t tag, uint32_t *gate)
{
    if (!n_blocks) return 0;
    McExpandArgs a;
    a.blocks = blocks; a.n_blocks = n_blocks; a.tiles = tiles; a.tag = tag;
    uint32_t o = 0;
    for (int k = 0; k < 5; k++) { a.base[k] = o; a.count[k] = count[k]; o += count[k]; }
    B200_LAUNCH((n_blocks + 255) / 256, 256, 0, st, k_mc_expand)(a, gate);
    return 1;
}

__device__ __forceinline__ int ref_slot_of(const RefTable &rt, int i)
{
    const uint64_t w = (i & 8) ? rt.w[1] : rt.w[0];      // no runtime indexing of the parameter struct (would go through local memory)
    return (int)((w >> (8 * (i & 7))) & 0xff);
}

// a reference plane, from the DPB's descriptor table
__device__ __forceinline__ PlaneDesc ref_plane(const FrameDesc *__restrict__ dpb, int slot, int plane)
{
    return dpb[slot].p[plane];
}

struct McGeom {
    int w, h;
    int wsh, parts, rows_per;   // stage B: lane = column (1 << wsh per row group), `parts` row groups of rows_per rows
    int wpad, lsh, q;           // stage A: 4 outputs per lane, q quads per row, (1 << lsh) lanes per row
    int ts;                     // row stride of the 16-bit intermediate in shared memory (= wpad)
};

// A tile is processed by a GROUP of GS lanes: GS = 32 (one warp per tile) for the big tiles, GS = 8 (four tiles per
// warp) for tiles of <= 8x8 samples, which are 3/4 of all tiles in a typical picture but would leave most of a warp
// idle.  `gl` = lane within the group, `gmask` = the group's lanes: every barrier below is group-local, so the
// groups of one warp may take different branches (uni/bi, luma/chroma, fractional or not).
//
// One reference list of one tile: fills val[j] (j < rows_per) with the 14-bit intermediate of sample
// (x = gl & (wpw-1), y = part * rows_per + j), exactly the value put_hevc_{q,e}pel* would hold.
// the window of reference samples one list of one tile needs, as it lies in shared memory
struct McWin {
    int R;                      // rows
    int ox, oy;                 // picture position of its first sample (before the even alignment)
    int skew, ax;               // origin aligned down to an even sample: ax = ox - skew
    int np, Ws;                 // sample pairs per row, shared-memory row stride (samples)
};
template <int TAPS>
__device__ __forceinline__ McWin mc_win(int sx, int sy, int mx, int my, const McGeom &g)
{
    constexpr int BEFORE = TAPS == 8 ? 3 : 1;
    McWin m;
    const int C = g.w + (mx ? TAPS - 1 : 0);
    m.R = g.h + (my ? TAPS - 1 : 0);
    m.ox = sx - (mx ? BEFORE : 0); m.oy = sy - (my ? BEFORE : 0);
    m.skew = m.ox & 1; m.ax = m.ox - m.skew;
    m.np = (C + m.skew + 1) >> 1; m.Ws = 2 * m.np;
    return m;
}
__device__ __forceinline__ bool mc_win_interior(const McWin &m, const PlaneDesc &rp)
{
    return m.ax >= 0 && m.ax + m.Ws <= rp.w && m.oy >= 0 && m.oy + m.R <= rp.h;
}
// window hangs over the picture border: clamp sample by sample (== emulated_edge_mc)
template <typename PIX, int GS>
__device__ __forceinline__ void mc_win_clamped(const McWin &m, const PlaneDesc &rp, int gl, uint16_t *win)
{
    for (int i = gl; i < m.R * m.Ws; i += GS) {
        const int r = i / m.Ws, cc = i - r * m.Ws;
        const int x = clip3i(m.ax + cc, 0, rp.w - 1), y = clip3i(m.oy + r, 0, rp.h - 1);
        win[i] = __ldg(px_ptr<PIX>(rp, x, y));
    }
}
template <typename PIX>
__device__ __forceinline__ uint32_t mc_ld_pair(const uint8_t *src)          // two neighbouring samples as two 16-bit halves
{
    if (sizeof(PIX) == 2) return __ldg(reinterpret_cast<const uint32_t *>(src));
    const uint32_t t = __ldg(reinterpret_cast<const uint16_t *>(src));
    return (t & 0xff) | ((t & 0xff00) << 8);
}

// the FIRs of one list on a window that is complete in shared memory
template <int TAPS, int GS>
__device__ __forceinline__ void mc_list_fir(const McWin &m, int mx, int my, const McGeom &g, int bd, int gl, unsigned gmask,
                                            const uint16_t *win, int16_t *tmp, int (&val)[8])
{
    const int R = m.R, Ws = m.Ws, skew = m.skew;
    const int8_t *fxp = TAPS == 8 ? c_qpel[mx] : c_epel[mx];
    const int8_t *fyp = TAPS == 8 ? c_qpel[my] : c_epel[my];
    if (mx) {
        // stage A: horizontal FIR, 4 outputs per lane, rows per pass = GS >> lsh
        int fx[TAPS];
#pragma unroll
        for (int k = 0; k < TAPS; k++) fx[k] = fxp[k];
        const int qi = gl & ((1 << g.lsh) - 1), rstep = GS >> g.lsh;
        if (qi < g.q) {
            const int sh = bd - 8;
            for (int r = gl >> g.lsh; r < R; r += rstep) {
                const uint16_t *s = win + r * Ws + skew + 4 * qi;
                int p[TAPS + 3];
#pragma unroll
                for (int k = 0; k < TAPS + 3; k++) p[k] = s[k];
                int o[4];
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    int acc = 0;
#pragma unroll
                    for (int k = 0; k < TAPS; k++) acc += fx[k] * p[j + k];
                    o[j] = (acc >> sh) & 0xffff;
                }
                uint32_t *d = reinterpret_cast<uint32_t *>(tmp + r * g.ts + 4 * qi);
                d[0] = (uint32_t)o[0] | ((uint32_t)o[1] << 16);
                d[1] = (uint32_t)o[2] | ((uint32_t)o[3] << 16);
            }
        }
        __syncwarp(gmask);
    }
    // stage B: vertical FIR (or pass-through), lane = column, up to 8 rows per lane with a register sliding window
    // Loads are unconditional: every index stays inside the group's buffers (sized for the worst tile shape), and the
    // rows / columns beyond the tile only feed outputs that are never stored.
    const int xl = gl & ((1 << g.wsh) - 1), y0 = (gl >> g.wsh) * g.rows_per;
    int a[8 + TAPS - 1];
    if (mx) {
        const int16_t *s = tmp + y0 * g.ts + xl;
#pragma unroll
        for (int k = 0; k < 8 + TAPS - 1; k++) a[k] = s[k * g.ts];
    } else {
        const uint16_t *s = win + y0 * Ws + skew + xl;
#pragma unroll
        for (int k = 0; k < 8 + TAPS - 1; k++) a[k] = s[k * Ws];
    }
    if (my) {
        int fy[TAPS];
#pragma unroll
        for (int k = 0; k < TAPS; k++) fy[k] = fyp[k];
        const int sh = mx ? 6 : bd - 8;
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

// B200McRec fields straight from the two 16-byte halves of the record
struct McRec {
    int dx, dy, w, h, plane, flags, sx0, sy0, sx1, sy1, ref0, ref1, frac0, frac1, w0, w1, o0, o1, denom;
};
template <int GS>
__device__ __forceinline__ McRec mc_rec(const int4 ra, const int4 rb)
{
    McRec t;
    const int mxy = ra.x, whpf = ra.y;
    t.dx = mxy & 0xffff; t.dy = (unsigned)mxy >> 16;
    t.w = whpf & 0xff; t.h = (whpf >> 8) & 0xff;
    if (GS == 8) { t.w = min(t.w, 8); t.h = min(t.h, 8); }          // the list order guarantees it; never trust it with shared memory
    t.plane = (whpf >> 16) & 0xff; t.flags = (unsigned)whpf >> 24;
    t.sx0 = (int16_t)(ra.z & 0xffff); t.sy0 = (int16_t)((unsigned)ra.z >> 16); t.sx1 = (int16_t)(ra.w & 0xffff); t.sy1 = (int16_t)((unsigned)ra.w >> 16);
    t.ref0 = rb.x & 0xff; t.ref1 = (rb.x >> 8) & 0xff; t.frac0 = (rb.x >> 16) & 0xff; t.frac1 = (unsigned)rb.x >> 24;
    t.w0 = (int16_t)(rb.y & 0xffff); t.w1 = (int16_t)((unsigned)rb.y >> 16); t.o0 = (int16_t)(rb.z & 0xffff); t.o1 = (int16_t)((unsigned)rb.z >> 16);
    t.denom = rb.w & 0xff;
    return t;
}
template <int GS>
__device__ __forceinline__ McGeom mc_geom(int w, int h)
{
    McGeom g;
    g.w = w; g.h = h;
    g.wsh = w <= 2 ? 1 : w <= 4 ? 2 : w <= 8 ? 3 : w <= 16 ? 4 : 5;
    g.parts = GS >> g.wsh;
    g.rows_per = (h + g.parts - 1) / g.parts;
    g.wpad = (w + 3) & ~3;
    g.q = g.wpad >> 2;
    g.lsh = g.q <= 1 ? 0 : g.q <= 2 ? 1 : g.q <= 4 ? 2 : 3;
    g.ts = g.wpad;
    return g;
}
// combine the lists' 14-bit intermediates (hevcdsp_template.c put_hevc_*_uni / _bi / _w) and store the tile
template <typename PIX>
__device__ __forceinline__ void mc_store(const McRec &t, const McGeom &g, const PlaneDesc &dp, int bd, int gl, const int (&v0)[8], const int (&v1)[8])
{
    const bool bi = t.flags & B200_MCF_BI, weighted = t.flags & B200_MCF_WEIGHTED;
    const int w = t.w, h = t.h, w0 = t.w0, w1 = t.w1, o0 = t.o0, o1 = t.o1, denom = t.denom;
    const int shift = 14 - bd, maxv = (1 << bd) - 1;
    const bool fullpel0 = t.frac0 == 0;
    const int xl = gl & ((1 << g.wsh) - 1), y0 = (gl >> g.wsh) * g.rows_per;
    if (xl >= w) return;
    PIX *d = px_ptr<PIX>(dp, t.dx + xl, t.dy + y0);
#pragma unroll
    for (int j = 0; j < 8; j++) {
        if (j >= g.rows_per || y0 + j >= h) break;
        int out;
        if (!bi) {
            if (!weighted) out = fullpel0 ? (v0[j] >> shift) : clip3i((v0[j] + (1 << (shift - 1))) >> shift, 0, maxv);
            else {
                const int s = denom + shift;
                out = clip3i(((v0[j] * w0 + (1 << (s - 1))) >> s) + o0 * (1 << (bd - 8)), 0, maxv);
            }
        } else {
            const int a = (int16_t)v0[j];          // list 0 travels through the reference's int16 tmp[] (hevc.c:1761)
            if (!weighted) out = clip3i((v1[j] + a + (1 << shift)) >> (shift + 1), 0, maxv);
            else {
                const int l2 = denom + shift, o = (o0 + o1) * (1 << (bd - 8)) + 1;
                out = clip3i((v1[j] * w1 + a * w0 + (o << l2)) >> (l2 + 1), 0, maxv);
            }
        }
        *d = (PIX)out;
        d = reinterpret_cast<PIX *>(reinterpret_cast<uint8_t *>(d) + dp.pitch);
    }
}

// The window loads of BOTH lists are issued before anything waits for them.  Fetching a window in passes of a few 4-byte loads
// per lane, and the second list only after the first has been filtered, costs several dependent round trips to L2 / HBM per
// bi-predicted tile in a stage that waits on exactly those loads (long scoreboard, DRAM at 10 %).  Here a lane issues up to
// 2 x 15 loads back to back into registers, then commits them to the two shared-memory windows.
#define MC_PASSES 15          // 32x8 tiles: 15 rows, one per pass; 16x16 tiles: 23 rows, two per pass; 8-lane groups: <= 15 rows
template <typename PIX, int GS>
__device__ __forceinline__ void mc_issue(const McWin &m, const PlaneDesc &rp, int gl, uint32_t (&v)[MC_PASSES])
{
    const int np = m.np;
    const int lpr = np <= GS / 2 ? GS / 2 : GS;         // lanes per window row
    const int pi = min(gl & (lpr - 1), np - 1), rsub = gl >= lpr ? 1 : 0, rstep = GS / lpr;
    // unconditional loads: lanes and passes beyond the window re-read its last pair / last row (never committed), so the
    // loop is straight-line code and every load is in flight before the first one is needed
    const uint8_t *src = rp.base + (size_t)m.oy * rp.pitch + (size_t)(m.ax + 2 * pi) * sizeof(PIX);
#pragma unroll
    for (int i = 0; i < MC_PASSES; i++) v[i] = mc_ld_pair<PIX>(src + (size_t)min(rsub + i * rstep, m.R - 1) * rp.pitch);
}
template <typename PIX, int GS>
__device__ __forceinline__ void mc_commit(const McWin &m, const PlaneDesc &rp, int gl, const uint32_t (&v)[MC_PASSES], uint16_t *win)
{
    const int np = m.np;
    const int lpr = np <= GS / 2 ? GS / 2 : GS;
    const int pi = gl & (lpr - 1), rsub = gl >= lpr ? 1 : 0, rstep = GS / lpr;
    if (pi >= np) return;
    uint32_t *dst = reinterpret_cast<uint32_t *>(win) + rsub * np + pi;
#pragma unroll
    for (int i = 0; i < MC_PASSES; i++)
        if (rsub + i * rstep < m.R) dst[i * rstep * np] = v[i];
    // taller windows than any valid tile produces (the validation kernel bounds w and h): finish row by row
    for (int r = rsub + MC_PASSES * rstep; r < m.R; r += rstep)
        dst[(r - rsub) * np] = mc_ld_pair<PIX>(rp.base + (size_t)(m.oy + r) * rp.pitch + (size_t)(m.ax + 2 * pi) * sizeof(PIX));
}

template <typename PIX, int GS>
__global__ void __launch_bounds__(256, 3) k_mc(const B200McRec *__restrict__ recs, int count, FrameDesc cur, const FrameDesc *__restrict__ dpb, RefTable rt, int bd,
                                         const uint32_t *__restrict__ gate)
{
    if (__ldg(gate + 1)) return;         // the picture's work list failed validation (k_validate)
    constexpr int NG = 256 / GS;                           // groups per CTA
    __shared__ __align__(16) uint16_t win_s[NG][2][McSmem<GS>::WIN];
    __shared__ __align__(16) int16_t tmp_s[NG][McSmem<GS>::TMP];
    const int grp = threadIdx.x / GS, gl = threadIdx.x & (GS - 1);
    const unsigned gmask = GS == 32 ? 0xffffffffu : (((1u << GS) - 1u) << ((threadIdx.x & 31) & ~(GS - 1)));
    const int ri = blockIdx.x * NG + grp;
    if (ri >= count) return;                               // whole groups leave: the barriers are group-local
    const int4 *rp4 = reinterpret_cast<const int4 *>(recs + ri);
    const McRec t = mc_rec<GS>(__ldg(rp4), __ldg(rp4 + 1));
    const bool chroma = t.flags & B200_MCF_CHROMA, bi = t.flags & B200_MCF_BI;
    const McGeom g = mc_geom<GS>(t.w, t.h);
    const int mx0 = t.frac0 & 15, my0 = t.frac0 >> 4, mx1 = t.frac1 & 15, my1 = t.frac1 >> 4;
    const PlaneDesc rp0 = ref_plane(dpb, ref_slot_of(rt, t.ref0), t.plane);
    const PlaneDesc rp1 = bi ? ref_plane(dpb, ref_slot_of(rt, t.ref1), t.plane) : rp0;
    const McWin m0 = chroma ? mc_win<4>(t.sx0, t.sy0, mx0, my0, g) : mc_win<8>(t.sx0, t.sy0, mx0, my0, g);
    const McWin m1 = chroma ? mc_win<4>(t.sx1, t.sy1, mx1, my1, g) : mc_win<8>(t.sx1, t.sy1, mx1, my1, g);
    const bool in0 = mc_win_interior(m0, rp0), in1 = bi && mc_win_interior(m1, rp1);      // uniform over the group
    uint16_t *win0 = win_s[grp][0], *win1 = win_s[grp][1];
    uint32_t r0[MC_PASSES], r1[MC_PASSES];
    if (in0) mc_issue<PIX, GS>(m0, rp0, gl, r0);
    if (in1) mc_issue<PIX, GS>(m1, rp1, gl, r1);
    if (!in0) mc_win_clamped<PIX, GS>(m0, rp0, gl, win0);
    if (bi && !in1) mc_win_clamped<PIX, GS>(m1, rp1, gl, win1);
    if (in0) mc_commit<PIX, GS>(m0, rp0, gl, r0, win0);
    if (in1) mc_commit<PIX, GS>(m1, rp1, gl, r1, win1);
    __syncwarp(gmask);
    int v0[8], v1[8];
    if (chroma) mc_list_fir<4, GS>(m0, mx0, my0, g, bd, gl, gmask, win0, tmp_s[grp], v0);
    else        mc_list_fir<8, GS>(m0, mx0, my0, g, bd, gl, gmask, win0, tmp_s[grp], v0);
    if (bi) {
        __syncwarp(gmask);                                 // list 0's stage B has read tmp
        if (chroma) mc_list_fir<4, GS>(m1, mx1, my1, g, bd, gl, gmask, win1, tmp_s[grp], v1);
        else        mc_list_fir<8, GS>(m1, mx1, my1, g, bd, gl, gmask, win1, tmp_s[grp], v1);
    }
    mc_store<PIX>(t, g, plane_of(cur, t.plane), bd, gl, v0, v1);
}


// --------------------------------------------------------------------------------------------
// K3: intra prediction.  Persistent warps take TUs in dependency-level order from an atomic counter.
// Neighbouring TUs exchange their border samples through per-4x4-unit *edge records* (bottom row and
// right column, 4 samples + valid bits in one 8-byte word each): the record IS the message, so a
// dependent TU polls the very data it needs -- no separate flag, no fence on either side, one L2
// round trip per wavefront step.  The picture itself is written with plain stores for the later stages.
// Prediction + parked residual are fused, so the serial chain is short.
// --------------------------------------------------------------------------------------------
// debug: per-TU timestamps (ns, %globaltimer) [grab, -, neighbours in, predicted, -, published]; null = off
__device__ unsigned long long *g_intra_trace = nullptr;
#ifndef B200_EMUL
__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
#endif
#define TRACE(slot) do { if (tr && lane == 0) tr[slot] = gtime(); } while (0)
int set_intra_trace(unsigned long long *p) { return (int)cudaMemcpyToSymbol(g_intra_trace, &p, sizeof(p)); }

// relaxed, GPU-scope accesses for the flags and edge records other warps poll.  8-byte edge words: naturally aligned 64-bit
// accesses are single-copy atomic, so a reader sees a whole record or none.  (tests/emul/ supplies CPU versions of the four:
// plain accesses, the loads also yield to the other emulated warps.)
#ifndef B200_EMUL
__device__ __forceinline__ uint32_t ld_relaxed(const uint32_t *p)
{
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed(uint32_t *p, uint32_t v)
{
    asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint2 ld_edge(const uint2 *p)
{
    uint2 v;
    asm volatile("ld.relaxed.gpu.global.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_edge(uint2 *p, uint2 v)
{
    asm volatile("st.relaxed.gpu.global.v2.u32 [%0], {%1, %2};" ::"l"(p), "r"(v.x), "r"(v.y) : "memory");
}
#endif
#define EDGE_VALID 0x8000u
__device__ __forceinline__ uint2 edge_pack(int a, int b, int c, int d)
{
    return make_uint2((uint32_t)a | EDGE_VALID | (((uint32_t)b | EDGE_VALID) << 16), (uint32_t)c | EDGE_VALID | (((uint32_t)d | EDGE_VALID) << 16));
}
__device__ __forceinline__ int edge_elem(uint2 v, int i)
{
    const uint32_t w = (i & 2) ? v.y : v.x;
    return (int)((w >> ((i & 1) * 16)) & 0x7fff);
}

__device__ __forceinline__ B200IntraRec decode_intra(const int4 raw)
{
    B200IntraRec r;
    r.x = (uint16_t)(raw.x & 0xffff); r.y = (uint16_t)((unsigned)raw.x >> 16);
    r.plane = (uint8_t)(raw.y & 0xff); r.log2 = (uint8_t)((raw.y >> 8) & 0xff); r.mode = (uint8_t)((raw.y >> 16) & 0xff); r.flags = (uint8_t)((unsigned)raw.y >> 24);
    r.top_right_size = (uint8_t)(raw.z & 0xff); r.bottom_left_size = (uint8_t)((raw.z >> 8) & 0xff); r.pad[0] = r.pad[1] = 0;
    r.resid_off = (uint32_t)raw.w;
    return r;
}

#include "k_intra_cip.cuh"

struct IntraEdges {
    uint2 *e[3];        // per plane: [2 * unit] = bottom row of the 4x4 unit, [2 * unit + 1] = its right column
    int stride[3];      // units per row
};
__device__ __forceinline__ uint2 *edges_of(const IntraEdges &ed, int plane) { return plane == 0 ? ed.e[0] : plane == 1 ? ed.e[1] : ed.e[2]; }
__device__ __forceinline__ int estride_of(const IntraEdges &ed, int plane) { return plane == 0 ? ed.stride[0] : plane == 1 ? ed.stride[1] : ed.stride[2]; }

// records of every unit from the picture as it stands after K1/K2 (inter blocks are final at that point)
template <typename PIX>
__global__ void k_intra_edges_init(FrameDesc f, IntraEdges ed)
{
    const int plane = blockIdx.z;
    const PlaneDesc pd = plane_of(f, plane);
    const int ux = blockIdx.x * blockDim.x + threadIdx.x, uy = blockIdx.y;
    if (4 * ux >= pd.w || 4 * uy >= pd.h) return;
    const PIX *b = px_ptr<PIX>(pd, 4 * ux, 4 * uy + 3);
    const int r0 = *px_ptr<PIX>(pd, 4 * ux + 3, 4 * uy), r1 = *px_ptr<PIX>(pd, 4 * ux + 3, 4 * uy + 1), r2 = *px_ptr<PIX>(pd, 4 * ux + 3, 4 * uy + 2);
    const uint2 bot = edge_pack(b[0], b[1], b[2], b[3]), rgt = edge_pack(r0, r1, r2, b[3]);
    uint4 *dst = reinterpret_cast<uint4 *>(edges_of(ed, plane) + 2 * ((size_t)uy * estride_of(ed, plane) + ux));
    *dst = make_uint4(bot.x, bot.y, rgt.x, rgt.y);
}

// units an intra TU of this picture will write: not valid yet
__global__ void k_intra_prepass(const B200IntraRec *__restrict__ recs, int count, IntraEdges ed, const uint32_t *__restrict__ gate)
{
    if (__ldg(gate + 1)) return;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const B200IntraRec r = decode_intra(__ldg(reinterpret_cast<const int4 *>(recs + i)));
    const int u = 1 << (r.log2 - 2), ux = r.x >> 2, uy = r.y >> 2;
    uint2 *e = edges_of(ed, r.plane);
    const int fs = estride_of(ed, r.plane);
    for (int y = 0; y < u; y++)
        for (int x = 0; x < u; x++) *reinterpret_cast<uint4 *>(e + 2 * ((size_t)(uy + y) * fs + ux + x)) = make_uint4(0, 0, 0, 0);
}

// Poll until every lane of the warp has its record(s).  Executed by all 32 lanes with a uniform (vote) exit so the
// warp leaves the loop CONVERGED -- a per-lane `while (!valid)` lets lanes leave one by one and the rest of the TU
// then runs as diverged fragments, several times slower.  A malformed list (dependency cycle)
// must not hang the GPU: give up after ~0.3 s and latch an error in counter[2].
// `pa_alt`: alternative source of record a (the up-left corner sample is the last element of BOTH halves of its unit,
// and depending on the neighbour's geometry only the bottom row or only the right column of that unit is published).
__device__ __forceinline__ void fetch_edges(const uint2 *pa, const uint2 *pa_alt, uint2 &va, const uint2 *pb, uint2 &vb, uint32_t *counter)
{
    bool ha = pa == nullptr, hb = pb == nullptr;
    uint32_t spins = 0;
    va = vb = make_uint2(0, 0);
    for (;;) {
        if (!ha) {
            // (every 16-bit half carries EDGE_VALID: both words of the record must have arrived -- the two halves of a vector
            // access are two accesses to the memory model)
            va = ld_edge(pa); ha = va.x & va.y & EDGE_VALID;
            if (!ha && pa_alt) { const uint2 t = ld_edge(pa_alt); if (t.x & t.y & EDGE_VALID) { va = t; ha = true; } }
        }
        if (!hb) { vb = ld_edge(pb); hb = vb.x & vb.y & EDGE_VALID; }
        if (__all_sync(0xffffffffu, ha && hb)) break;
        __nanosleep(20);
        if ((++spins & 1023) == 0) {
            const bool abort = spins > (1u << 21) || ld_relaxed(counter + 2) != 0;
            if (__any_sync(0xffffffffu, abort)) { st_relaxed(counter + 2, 1u); latch_host(counter, 0x80000000u); break; }
        }
    }
}

// publish the bottom row / right column of a finished TU: sb[x] = row n-1, sr[y] = column n-1 (shared memory)
__device__ __forceinline__ void publish_edges(uint2 *e, int fs, int ux, int uy, int u, const uint16_t *sb, const uint16_t *sr, int lane)
{
    if (lane < u) st_edge(e + 2 * ((size_t)(uy + u - 1) * fs + ux + lane), edge_pack(sb[4 * lane], sb[4 * lane + 1], sb[4 * lane + 2], sb[4 * lane + 3]));
    else if (lane >= 8 && lane < 8 + u) {
        const int k = lane - 8;
        st_edge(e + 2 * ((size_t)(uy + k) * fs + ux + u - 1) + 1, edge_pack(sr[4 * k], sr[4 * k + 1], sr[4 * k + 2], sr[4 * k + 3]));
    }
}

// Fast path for 4x4 / 8x8 intra TUs (the bulk of every dependency chain): the <= 33 reference samples live one per
// lane in two registers (fT: lane k = top[k-1], fL: lane k = left[k]); substitution, [1 2 1] smoothing and the
// predictors use warp shuffles only, so one wavefront step is ~150 instructions.
template <typename PIX>
__device__ __forceinline__ void intra_small(const B200IntraRec &r, const int16_t *__restrict__ pool, const PlaneDesc &pd, int bd,
                                            uint2 *e, int fs, uint32_t *counter, int lane, uint16_t *sbr, unsigned long long *tr)
{
    const unsigned FULL = 0xffffffffu;
    const int n = 1 << r.log2, n2 = 2 * n, x0 = r.x, y0 = r.y, maxv = (1 << bd) - 1;
    const bool ul = r.flags & B200_INF_UP_LEFT, up = r.flags & B200_INF_UP, ur = r.flags & B200_INF_UP_RIGHT;
    const bool lf = r.flags & B200_INF_LEFT, bl = r.flags & B200_INF_BOTTOM_LEFT;
    const int trs = r.top_right_size, bls = r.bottom_left_size;
    const int npx = n * n;
    const int16_t *res = r.resid_off != B200_NO_RESID ? pool + r.resid_off : nullptr;
    int rs0 = 0, rs1 = 0;                                  // residual prefetch (independent of the neighbours)
    if (res) { if (lane < npx) rs0 = res[lane]; if (lane + 32 < npx) rs1 = res[lane + 32]; }
    // ---- neighbours: lane k polls the record holding top[k-1] and the one holding left[k] ----
    int gT = 0, gL = 0;
    {
        const int t = lane - 1;
        const bool needT = lane == 0 ? ul : t < n ? up : (t < n2 && ur);
        const bool needL = lane < n ? lf : (lane < n2 && bl);
        const int tx = x0 + (lane == 0 ? -1 : min(t, n + trs - 1)), ly = y0 + min(lane, n + bls - 1);
        const uint2 *pT = needT ? e + 2 * ((size_t)((y0 - 1) >> 2) * fs + (tx >> 2)) : nullptr;
        const uint2 *pL = needL ? e + 2 * ((size_t)(ly >> 2) * fs + ((x0 - 1) >> 2)) + 1 : nullptr;
        uint2 vT, vL;
        fetch_edges(pT, (lane == 0 && pT) ? pT + 1 : nullptr, vT, pL, vL, counter);
        if (needT) gT = edge_elem(vT, tx & 3);
        if (needL) gL = edge_elem(vL, ly & 3);
    }
    TRACE(2);
    // ---- substitution (hevcpred_template.c:250-286), closed form on broadcast scalars ----
    const int g_corner = __shfl_sync(FULL, gT, 0), g_top0 = __shfl_sync(FULL, gT, 1), g_topn1 = __shfl_sync(FULL, gT, n), g_topn = __shfl_sync(FULL, gT, n + 1);
    const int g_left0 = __shfl_sync(FULL, gL, 0), g_leftn1 = __shfl_sync(FULL, gL, n - 1), g_leftn = __shfl_sync(FULL, gL, n);
    const int sub = lf ? g_leftn1 : ul ? g_corner : up ? g_top0 : ur ? g_topn : (1 << (bd - 1));
    const int bl0 = bl ? g_leftn : sub, l0 = lf ? g_left0 : bl0, corner = ul ? g_corner : l0, un1 = up ? g_topn1 : corner;
    int fT, fL;
    {
        const int t = lane - 1;
        fT = t < 0 ? corner : t < n ? (up ? gT : corner) : (ur ? gT : un1);
        fL = lane < n ? (lf ? gL : bl0) : (bl ? gL : sub);
    }
    const int mode = r.mode;
    // ---- [1 2 1] smoothing (:288-327); strong smoothing needs 32x32, never here ----
    if ((r.flags & B200_INF_FILTER) && mode != 1 && n == 8) {
        const int d26 = abs(mode - 26), d10 = abs(mode - 10);
        if (min(d26, d10) > 7) {
            const int tm = __shfl_up_sync(FULL, fT, 1), tp = __shfl_down_sync(FULL, fT, 1);
            const int lm = __shfl_up_sync(FULL, fL, 1), lp = __shfl_down_sync(FULL, fL, 1);
            const int top0 = __shfl_sync(FULL, fT, 1), left0 = __shfl_sync(FULL, fL, 0);
            int qT, qL;
            if (lane == 0) qT = (left0 + 2 * corner + top0 + 2) >> 2;
            else if (lane == n2) qT = fT;                                  // top[2n-1]
            else qT = (tp + 2 * fT + tm + 2) >> 2;
            if (lane == n2 - 1) qL = fL;
            else qL = (lp + 2 * fL + (lane == 0 ? corner : lm) + 2) >> 2;
            fT = qT; fL = qL;
        }
    }
#define TOPS(i) __shfl_sync(FULL, fT, ((i) + 1) & 31)
#define LEFTS(i) __shfl_sync(FULL, fL, (i) & 31)
    const int cornerf = __shfl_sync(FULL, fT, 0);
    int dc = 0;
    if (mode == 1) {
        int sum = (lane < n ? fL : 0) + ((lane >= 1 && lane <= n) ? fT : 0);
#pragma unroll
        for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(FULL, sum, o);
        dc = (sum + n) >> (r.log2 + 1);
    }
    const int angle = mode >= 2 ? c_intra_angle[mode - 2] : 0;
    const bool vertical = mode >= 18;
    const int inv = (mode >= 11 && mode <= 25) ? c_inv_angle[mode - 11] : 0;
    const bool edge = r.plane == 0;                                       // n < 32 always here
    const int topn_f = TOPS(n), leftn_f = LEFTS(n), top0_f = TOPS(0), left0_f = LEFTS(0);
    uint16_t *sb = sbr, *sr = sbr + 32;
#pragma unroll
    for (int it = 0; it < 2; it++) {
        const int i = lane + 32 * it;
        if (it * 32 >= npx) break;                                         // uniform
        const int y = (i >> r.log2) & (n - 1), x = i & (n - 1);
        const int ty = TOPS(x), lx = LEFTS(y);                             // top[x], left[y]
        int v;
        if (mode == 0) {
            v = ((n - 1 - x) * lx + (x + 1) * topn_f + (n - 1 - y) * ty + (y + 1) * leftn_f + n) >> (r.log2 + 1);
        } else if (mode == 1) {
            v = dc;
            if (edge) {
                if (x == 0 && y == 0) v = (left0_f + 2 * dc + top0_f + 2) >> 2;
                else if (y == 0) v = (ty + 3 * dc + 2) >> 2;
                else if (x == 0) v = (lx + 3 * dc + 2) >> 2;
            }
        } else {
            const int a = vertical ? y : x, b = vertical ? x : y;
            const int pos = (a + 1) * angle, id = pos >> 5, fact = pos & 31;
            const int k0 = b + id + 1, k1 = k0 + 1;                        // ref[k] = main[k-1]; k < 0: projected side sample
            // source of ref[k]: main[k-1] (k>=0) or side[j], j = -1 + ((k*inv+128)>>8); index -1 of either array is the corner (fT lane 0)
            const int j0 = k0 >= 0 ? k0 - 1 : -1 + ((k0 * inv + 128) >> 8), j1 = k1 >= 0 ? k1 - 1 : -1 + ((k1 * inv + 128) >> 8);
            const bool t0 = (k0 >= 0) == vertical, t1 = (k1 >= 0) == vertical;   // read from the top register?
            const int a0 = __shfl_sync(FULL, fT, (j0 + 1) & 31), b0 = __shfl_sync(FULL, fL, j0 & 31);
            const int a1 = __shfl_sync(FULL, fT, (j1 + 1) & 31), b1 = __shfl_sync(FULL, fL, j1 & 31);
            const int r0 = (t0 || j0 < 0) ? a0 : b0, r1 = (t1 || j1 < 0) ? a1 : b1;
            v = fact ? ((32 - fact) * r0 + fact * r1 + 16) >> 5 : r0;
            if (edge) {
                if (mode == 26 && x == 0) v = clip3i(top0_f + ((lx - cornerf) >> 1), 0, maxv);
                if (mode == 10 && y == 0) v = clip3i(left0_f + ((ty - cornerf) >> 1), 0, maxv);
            }
        }
        if (i < npx) {
            if (res) v = clip3i(v + (it ? rs1 : rs0), 0, maxv);
            *px_ptr<PIX>(pd, x0 + x, y0 + y) = (PIX)v;
            if (y == n - 1) sb[x] = (uint16_t)v;
            if (x == n - 1) sr[y] = (uint16_t)v;
        }
    }
#undef TOPS
#undef LEFTS
    TRACE(3);
    __syncwarp();
    publish_edges(e, fs, x0 >> 2, y0 >> 2, n >> 2, sb, sr, lane);
    __syncwarp();
    TRACE(5);
}

template <typename PIX>
__global__ void __launch_bounds__(128) k_intra(const B200IntraRec *__restrict__ recs, int count, const int16_t *__restrict__ pool,
                                               FrameDesc f, int bd, IntraEdges ed, uint32_t *counter, CipDesc cipd)
{
    if (ld_relaxed(counter + 1)) return;               // the picture's work list failed validation (k_validate)
    const bool cip = cipd.bits != nullptr;             // constrained_intra_pred picture (rare): every TU takes the general path
    __shared__ int s_g[4][2][66];     // gathered   [0]=top [1]=left, element [k] holds index k-1
    __shared__ int s_f[4][2][66];     // substituted
    __shared__ int s_ff[4][2][66];    // smoothed
    __shared__ uint16_t s_st[4][2][64];   // staging: neighbour samples by position / border of the finished TU
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int maxv = (1 << bd) - 1;
    for (;;) {
        int idx = 0;
        if (lane == 0) idx = atomicAdd(counter, 1u);
        idx = __shfl_sync(0xffffffffu, idx, 0);
        if (idx >= count) break;
        const B200IntraRec r = decode_intra(__ldg(reinterpret_cast<const int4 *>(recs + idx)));
        uint2 *e = edges_of(ed, r.plane);
        const int fs = estride_of(ed, r.plane);
        if (r.log2 <= 3 && !cip) {
            unsigned long long *tr = g_intra_trace ? g_intra_trace + 8ull * idx : nullptr;
            TRACE(0);
            intra_small<PIX>(r, pool, plane_of(f, r.plane), bd, e, fs, counter, lane, &s_st[warp][0][0], tr);
            continue;
        }
        const int n = 1 << r.log2, n2 = 2 * n, x0 = r.x, y0 = r.y;
        const PlaneDesc pd = plane_of(f, r.plane);
        // availability: final in the record, except under constrained_intra_pred, where the record holds the flags BEFORE
        // the rule and lane 0 applies hevcpred_template.c:116-163 with the picture's intra bitmap
        int aflags = r.flags;
        CipBlock cb;
        if (cip) {
            const int hs = r.plane ? cipd.hs_c : 0, vs = r.plane ? cipd.vs_c : 0;
            cb.x0 = x0 << hs; cb.y0 = y0 << vs; cb.hs = hs; cb.vs = vs; cb.n = n;
            int fl = 0;
            if (lane == 0) fl = cip_flags(cipd, cb, r.flags);
            aflags = __shfl_sync(0xffffffffu, fl, 0);
        }
        const bool ul = aflags & B200_INF_UP_LEFT, up = aflags & B200_INF_UP, ur = aflags & B200_INF_UP_RIGHT;
        const bool lf = aflags & B200_INF_LEFT, bl = aflags & B200_INF_BOTTOM_LEFT;
        const int trs = r.top_right_size, bls = r.bottom_left_size;
        uint16_t *stg_t = s_st[warp][0], *stg_l = s_st[warp][1];
        // ---- neighbours: lane k fetches the bottom row of top unit k (4 samples), lane k the right column of left unit k;
        //      16x16: 8 + 8 units, 32x32: 16 + 16 units; the corner comes with the up-left unit's bottom row ----
        int g_corner = 0;
        {
            const int nu = n2 >> 2;                                            // units along 2n samples
            const int ot = 4 * lane, ol = 4 * lane;
            const bool needT = lane < nu && ((ot < n && up) || (ot >= n && ur && ot < n + trs));
            const bool needL = lane < nu && ((ol < n && lf) || (ol >= n && bl && ol < n + bls));
            const uint2 *pT = needT ? e + 2 * ((size_t)((y0 - 1) >> 2) * fs + ((x0 + ot) >> 2)) : nullptr;
            const uint2 *pL = needL ? e + 2 * ((size_t)((y0 + ol) >> 2) * fs + ((x0 - 1) >> 2)) + 1 : nullptr;
            uint2 vT, vL, vC, vD;
            fetch_edges(pT, nullptr, vT, pL, vL, counter);
            const uint2 *pC = (lane == 0 && ul) ? e + 2 * ((size_t)((y0 - 1) >> 2) * fs + ((x0 - 1) >> 2)) : nullptr;
            fetch_edges(pC, pC ? pC + 1 : nullptr, vC, nullptr, vD, counter);
            if (lane < 16) {
#pragma unroll
                for (int k = 0; k < 4; k++) { stg_t[4 * lane + k] = needT ? (uint16_t)edge_elem(vT, k) : 0; stg_l[4 * lane + k] = needL ? (uint16_t)edge_elem(vL, k) : 0; }
            }
            g_corner = __shfl_sync(0xffffffffu, pC ? edge_elem(vC, 3) : 0, 0);
        }
        __syncwarp();
        // ---- the reference arrays, with the replication of the last in-picture sample (hevcpred_template.c:170-183) ----
        int *gt = s_g[warp][0], *gl = s_g[warp][1];
        const int nofill = cip ? cip_fill_value(bd) : 0;       // what the reference leaves in samples nobody copied (:159-161)
        for (int k = lane; k <= n2; k += 32) {
            const int t = k - 1;
            int tv = nofill, lv = nofill;
            if (t < 0) { tv = lv = cip ? 128 : 0; if (ul) tv = lv = g_corner; }
            else {
                if (t < n ? up : ur) tv = stg_t[t < n ? t : min(t, n + trs - 1)];
                if (t < n ? lf : bl) lv = stg_l[t < n ? t : min(t, n + bls - 1)];
            }
            gt[k] = tv; gl[k] = lv;
        }
        __syncwarp();
        if (cip) {                                               // :185-249, a sequential scan: one lane
            if (lane == 0) cip_substitute(cipd, cb, aflags, bls, gt + 1, gl + 1);
            __syncwarp();
        }
        // ---- substitution (hevcpred_template.c:250-286) in closed form ----
        int *ft = s_f[warp][0], *fleft = s_f[warp][1];
        {
            const int s = lf ? gl[n] /*left[n-1]*/ : ul ? gl[0] : up ? gt[1] : ur ? gt[n + 1] : (1 << (bd - 1));
            const int bl0 = bl ? gl[n + 1] : s;                 // final left[n]
            const int l0 = lf ? gl[1] : bl0;                    // final left[0]
            const int corner = ul ? gl[0] : l0;
            const int un1 = up ? gt[n] : corner;                // final top[n-1]
            for (int k = lane; k <= n2; k += 32) {
                const int t = k - 1;
                int tv, lv;
                if (t < 0) tv = lv = corner;
                else if (t < n) { tv = up ? gt[k] : corner; lv = lf ? gl[k] : bl0; }
                else { tv = ur ? gt[k] : un1; lv = bl ? gl[k] : s; }
                ft[k] = tv; fleft[k] = lv;
            }
        }
        __syncwarp();
        const int mode = r.mode;
        const int *top = ft + 1, *left = fleft + 1;
        // ---- smoothing (:288-327) ----
        if ((r.flags & B200_INF_FILTER) && mode != 1 && n != 4) {
            const int d26 = abs(mode - 26), d10 = abs(mode - 10), dist = min(d26, d10);
            const int thr = r.log2 == 3 ? 7 : r.log2 == 4 ? 1 : 0;
            if (dist > thr) {
                int *qt = s_ff[warp][0], *ql = s_ff[warp][1];
                const bool strong = (r.flags & B200_INF_STRONG) && r.plane == 0 && r.log2 == 5 &&
                                    abs(top[-1] + top[63] - 2 * top[31]) < (1 << (bd - 5)) &&
                                    abs(left[-1] + left[63] - 2 * left[31]) < (1 << (bd - 5));
                for (int k = lane; k <= n2; k += 32) {
                    const int t = k - 1;
                    int tv, lv;
                    if (strong) {
                        if (t < 0 || t == 63) { tv = top[t]; lv = left[t]; }
                        else { tv = ((63 - t) * top[-1] + (t + 1) * top[63] + 32) >> 6; lv = ((63 - t) * left[-1] + (t + 1) * left[63] + 32) >> 6; }
                    } else {
                        if (t < 0) tv = lv = (left[0] + 2 * left[-1] + top[0] + 2) >> 2;
                        else if (t == n2 - 1) { tv = top[t]; lv = left[t]; }
                        else { tv = (top[t + 1] + 2 * top[t] + top[t - 1] + 2) >> 2; lv = (left[t + 1] + 2 * left[t] + left[t - 1] + 2) >> 2; }
                    }
                    qt[k] = tv; ql[k] = lv;
                }
                __syncwarp();
                top = qt + 1; left = ql + 1;
            }
        }
        // ---- predictor ----
        int dc = 0;
        if (mode == 1) {
            int sum = 0;
            for (int i = lane; i < n; i += 32) sum += left[i] + top[i];
#pragma unroll
            for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
            dc = (sum + n) >> (r.log2 + 1);
        }
        const int angle = mode >= 2 ? c_intra_angle[mode - 2] : 0;
        const bool vertical = mode >= 18;
        const int *mainr = vertical ? top : left, *side = vertical ? left : top;
        const int inv = (mode >= 11 && mode <= 25) ? c_inv_angle[mode - 11] : 0;
        const bool edge = r.plane == 0 && n < 32;
        const int16_t *res = r.resid_off != B200_NO_RESID ? pool + r.resid_off : nullptr;
        __syncwarp();                                           // staging buffers are reused for the TU's own border below
        auto predict = [&](int x, int y) -> int {
            int v;
            if (mode == 0) {
                v = ((n - 1 - x) * left[y] + (x + 1) * top[n] + (n - 1 - y) * top[x] + (y + 1) * left[n] + n) >> (r.log2 + 1);
            } else if (mode == 1) {
                v = dc;
                if (edge) {
                    if (x == 0 && y == 0) v = (left[0] + 2 * dc + top[0] + 2) >> 2;
                    else if (y == 0) v = (top[x] + 3 * dc + 2) >> 2;
                    else if (x == 0) v = (left[y] + 3 * dc + 2) >> 2;
                }
            } else {
                const int a = vertical ? y : x, b = vertical ? x : y;     // a along the prediction direction
                const int pos = (a + 1) * angle, id = pos >> 5, fact = pos & 31;
                const int k0 = b + id + 1;                                 // ref[k] == main[k-1]; k < 0 -> projected side samples
                const int r0 = k0 >= 0 ? mainr[k0 - 1] : side[-1 + ((k0 * inv + 128) >> 8)];
                if (fact) {
                    const int k1 = k0 + 1;
                    const int r1 = k1 >= 0 ? mainr[k1 - 1] : side[-1 + ((k1 * inv + 128) >> 8)];
                    v = ((32 - fact) * r0 + fact * r1 + 16) >> 5;
                } else v = r0;
                if (edge) {
                    if (mode == 26 && x == 0) v = clip3i(top[0] + ((left[y] - left[-1]) >> 1), 0, maxv);
                    if (mode == 10 && y == 0) v = clip3i(left[0] + ((top[x] - top[-1]) >> 1), 0, maxv);
                }
            }
            if (res) v = clip3i(v + res[y * n + x], 0, maxv);
            return v;
        };
        // ---- the border first: the bottom row and right column are all a dependent TU ever reads, so they are
        //      predicted and published before the interior -- the interior is off the wavefront's critical path ----
        for (int i = lane; i < 2 * n - 1; i += 32) {
            const int x = i < n ? i : n - 1, y = i < n ? n - 1 : i - n;
            const int v = predict(x, y);
            if (i < n) stg_t[x] = (uint16_t)v; else stg_l[y] = (uint16_t)v;
            if (i == n - 1) stg_l[n - 1] = (uint16_t)v;
        }
        __syncwarp();
        publish_edges(e, fs, x0 >> 2, y0 >> 2, n >> 2, stg_t, stg_l, lane);
        // ---- then the whole block ----
        for (int i = lane; i < n * n; i += 32) {
            const int y = i >> r.log2, x = i & (n - 1);
            *px_ptr<PIX>(pd, x0 + x, y0 + y) = (PIX)predict(x, y);
        }
        __syncwarp();
    }
}

// --------------------------------------------------------------------------------------------
// K4: deblocking, both directions in ONE pass (k_deblock.cuh: one thread per 4-line edge segment).
// --------------------------------------------------------------------------------------------
#include "k_deblock.cuh"

template <typename PIX>
__global__ void __launch_bounds__(DBK_THREADS, 3) k_deblock(const uint16_t *__restrict__ grid, B200DbkLayout L, FrameDesc f, int bd)
{
    const int plane = blockIdx.z;
    const PlaneDesc pd = plane_of(f, plane);
    if (DBK_TW * (int)blockIdx.x - 4 >= pd.w || DBK_TH * (int)blockIdx.y - 4 >= pd.h) return;
    __shared__ __align__(16) uint16_t t[DBK_TH * DBK_PITCH];
    const int tid = threadIdx.x;
    dbk_load<PIX>(t, pd, blockIdx.x, blockIdx.y, tid);
    __syncthreads();
    dbk_vertical(t, grid, L, pd, plane, blockIdx.x, blockIdx.y, tid, bd);
    __syncthreads();
    dbk_horizontal(t, grid, L, pd, plane, blockIdx.x, blockIdx.y, tid, bd);
    __syncthreads();
    dbk_store<PIX>(t, pd, blockIdx.x, blockIdx.y, tid);
}

// --------------------------------------------------------------------------------------------
// K5: SAO.  Source = deblocked picture (never modified), destination = DPB slot, so the reference's
// sao_frame copy / SAO_APPLIED bookkeeping (hevc_filter.c:267-319) has no equivalent here.  CTBs
// without SAO are copied through.
//
// The stage is issue-bound, not bandwidth-bound, so the kernel is written around the instruction count:
//  * samples stay packed two per 32-bit register (16-bit halves; 8-bit pictures are widened on load) and are
//    classified with the 16x2 SIMD integer (DPX) instructions of sm_90a (VIADD.16x2, VIADDMNMX.S16x2.RELU):
//    sign(c - a) + 1 = relu(min(c + (1 - a), 2)) is ONE instruction for two samples;
//  * the offset is fetched with a byte permute (PRMT) from a 5-entry table held in two registers (offsets biased by
//    128: |offset| <= 124 for every legal stream up to 12 bits, hevc_cabac.c:684-692 / hevc.c:1178);
//  * one thread owns 8 samples x SAO_R rows, so rows are loaded once and reused as neighbours, and the CTB record is
//    decoded once per 8 x SAO_R samples; a warp never spans more than one CTB horizontally (no class divergence
//    inside a row of lanes).
// Picture-border rows / columns ("offset 0", hevcdsp_template.c:433-471) and the not-across-boundary restore of
// sao_edge_filter_1 (:533-566) touch only the outermost rows / columns of a CTB: those rows take sao_row_exact(),
// the scalar statement of the reference rules; everything else takes the packed path.
// --------------------------------------------------------------------------------------------
#include "k_sao.cuh"

#ifndef SAO_MINB
#define SAO_MINB 3
#endif
template <typename PIX>
__global__ void __launch_bounds__(256, SAO_MINB) k_sao(const B200SaoRec *__restrict__ grid, FrameDesc src, FrameDesc dst, int bd,
                                                int log2_ctb, int ctb_w, int ctb_h, int cfi, int4 tile_base, int3 tiles_x, TqbDesc tq)
{
    sao_thread<PIX>(grid, src, dst, bd, log2_ctb, ctb_w, ctb_h, cfi, tile_base, tiles_x, tq, blockIdx.x * 8 + (threadIdx.x >> 5), threadIdx.x & 31);
}

// --------------------------------------------------------------------------------------------
// K4a-c: deblocking parameters derived on the device (k_dbd.cuh)
// --------------------------------------------------------------------------------------------
#include "k_dbd.cuh"

template <typename PIX>
__global__ void k_fill(FrameDesc f, int value)
{
    const int plane = blockIdx.z;
    const PlaneDesc pd = plane_of(f, plane);
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x < pd.w && y < pd.h) *px_ptr<PIX>(pd, x, y) = (PIX)value;
}

// --------------------------------------------------------------------------------------------
// launchers
// --------------------------------------------------------------------------------------------
static int sm_count()                    // SMs of the current device: the persistent grid of K3 is sized per SM
{
    int dev = 0, n = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    return n > 0 ? n : 1;
}
int launch_mc(cudaStream_t st, const B200McRec *recs, int count, int n_big, const FrameDesc &cur, const FrameDesc *dpb_dev, const RefTable &rt, int bd, const uint32_t *gate)
{
    if (!count) return 0;
    int n = 0;
    const int n_small = count - n_big;
    if (n_big) {                        // one warp per tile
        const int grid = (n_big + 7) / 8;
        if (bd > 8) B200_LAUNCH(grid, 256, 0, st, k_mc<uint16_t, 32>)(recs, n_big, cur, dpb_dev, rt, bd, gate);
        else        B200_LAUNCH(grid, 256, 0, st, k_mc<uint8_t, 32>)(recs, n_big, cur, dpb_dev, rt, bd, gate);
        n++;
    }
    if (n_small) {                      // tiles of <= 8x8 samples: four per warp
        const int grid = (n_small + 31) / 32;
        if (bd > 8) B200_LAUNCH(grid, 256, 0, st, k_mc<uint16_t, 8>)(recs + n_big, n_small, cur, dpb_dev, rt, bd, gate);
        else        B200_LAUNCH(grid, 256, 0, st, k_mc<uint8_t, 8>)(recs + n_big, n_small, cur, dpb_dev, rt, bd, gate);
        n++;
    }
    return n;
}

template <typename PIX>
static int launch_residual_t(cudaStream_t st, const B200TuRec *const recs[4], const int counts[4], const int16_t *pool, int16_t *parked, const FrameDesc &cur, int bd, const uint32_t *gate)
{
    ResidualLists L;
    int total = 0;
    for (int k = 0; k < 4; k++) {
        const int per_cta = 4 * (32 >> (k + 2));         // 4 warps x (32 / N) TUs
        L.recs[k] = recs[k]; L.count[k] = counts[k]; L.nblk[k] = (counts[k] + per_cta - 1) / per_cta;
        total += L.nblk[k];
    }
    if (!total) return 0;
    B200_LAUNCH(total, 128, 0, st, k_residual<PIX>)(L, pool, parked, cur, bd, gate);
    return 1;
}
int launch_residual(cudaStream_t st, const B200TuRec *const recs[4], const int counts[4], const int16_t *pool, int16_t *parked, const FrameDesc &cur, int bd, const uint32_t *gate)
{
    return bd > 8 ? launch_residual_t<uint16_t>(st, recs, counts, pool, parked, cur, bd, gate) : launch_residual_t<uint8_t>(st, recs, counts, pool, parked, cur, bd, gate);
}

int launch_ccp(cudaStream_t st, const B200CcpRec *recs, int count, int16_t *parked, const FrameDesc &cur, int bd, uint32_t *gate, unsigned long long arena_bytes)
{
    if (!count) return 0;
    if (bd > 8) B200_LAUNCH(count, 128, 0, st, k_ccp<uint16_t>)(recs, count, parked, cur, bd, gate, arena_bytes);
    else        B200_LAUNCH(count, 128, 0, st, k_ccp<uint8_t>)(recs, count, parked, cur, bd, gate, arena_bytes);
    return 1;
}

int launch_intra(cudaStream_t st, const B200IntraRec *recs, int count, const int16_t *pool, const FrameDesc &cur, int bd,
                 uint2 *edges[3], const int edge_stride[3], uint32_t *counter, const uint32_t *cip_words, const B200CipHeader *cip_hdr, int cfi)
{
    if (!count) return 0;
    IntraEdges ed;
    for (int p = 0; p < 3; p++) { ed.e[p] = edges[p]; ed.stride[p] = edge_stride[p]; }
    // counter[0] (ticket) and counter[1] (gate) were cleared when the picture entered its lane (engine.cu)
    const dim3 gi((cur.p[0].w / 4 + 127) / 128, cur.p[0].h / 4, 3);
    if (bd > 8) B200_LAUNCH(gi, 128, 0, st, k_intra_edges_init<uint16_t>)(cur, ed);
    else        B200_LAUNCH(gi, 128, 0, st, k_intra_edges_init<uint8_t>)(cur, ed);
    B200_LAUNCH((count + 255) / 256, 256, 0, st, k_intra_prepass)(recs, count, ed, counter);
    int grid = (count + 3) / 4;
    // persistent warps.  The list is sorted by dependency level, so the TUs that can run together are adjacent and a
    // small window exposes all the parallelism there is; more waiting warps only take issue slots from the other pictures
    // in flight, while far fewer blocks than SMs lengthen the serial chain of an I picture.  One block per SM.
    static const int env_ctas = getenv("B200_INTRA_CTAS") ? atoi(getenv("B200_INTRA_CTAS")) : 0;
    const int max_ctas = env_ctas > 0 ? env_ctas : sm_count();
    if (grid > max_ctas) grid = max_ctas;
    CipDesc cd;
    memset(&cd, 0, sizeof(cd));
    if (cip_words && cip_hdr) {                        // device pointer to the blob's CIP section (B200CipHeader, then the bitmap) + host copy of the header
        const B200CipHeader &ch = *cip_hdr;
        cd.bits = cip_words + 4; cd.log2_pu = (int)ch.log2_min_pu_size; cd.pu_w = (int)ch.min_pu_width; cd.pu_h = (int)ch.min_pu_height;
        cd.pic_w = cur.p[0].w; cd.pic_h = cur.p[0].h; cd.hs_c = cfi != 3; cd.vs_c = cfi == 1;
    }
    if (bd > 8) B200_LAUNCH(grid, 128, 0, st, k_intra<uint16_t>)(recs, count, pool, cur, bd, ed, counter, cd);
    else        B200_LAUNCH(grid, 128, 0, st, k_intra<uint8_t>)(recs, count, pool, cur, bd, ed, counter, cd);
    return 3;
}

int launch_deblock(cudaStream_t st, const uint16_t *grid, const B200DbkLayout &L, const FrameDesc &cur, int bd)
{
    const dim3 g((cur.p[0].w + 4 + DBK_TW - 1) / DBK_TW, (cur.p[0].h + 4 + DBK_TH - 1) / DBK_TH, 3);
    if (bd > 8) B200_LAUNCH(g, DBK_THREADS, 0, st, k_deblock<uint16_t>)(grid, L, cur, bd);
    else        B200_LAUNCH(g, DBK_THREADS, 0, st, k_deblock<uint8_t>)(grid, L, cur, bd);
    return 1;
}

// Derives the picture's deblocking grids on the device into `maps.grid`; `check` (device pointer to the grid recorded from the
// reference's own calls, or null) compares the two.  `dbd` = device copy of the blob's DBD section, `hd` = host copy of its header.
int launch_dbd(cudaStream_t st, const uint8_t *blob_dev, const B200BlobHeader &h, const B200DbdHeader &hd, const uint8_t *dbd, const DbdMaps &maps, size_t maps_bytes,
               const B200DbkLayout &L, const RefTable &rt, int ctb_w, uint32_t *gate, const uint16_t *check)
{
    DbdArgs a;
    a.blob = blob_dev;
    a.mc = h.sec[B200_SEC_MC];
    for (int k = 0; k < 4; k++) a.tu[k] = h.sec[B200_SEC_TU4 + k];
    a.leaf = reinterpret_cast<const uint32_t *>(dbd + hd.off_leaf); a.n_leaf = (int)hd.n_leaf;
    a.qp = reinterpret_cast<const int8_t *>(dbd + hd.off_qp); a.log2_min_cb = (int)hd.log2_min_cb_size; a.min_cb_w = (int)hd.min_cb_width;
    a.ctb = reinterpret_cast<const int8_t *>(dbd + hd.off_ctb);
    a.pcm = (hd.flags & B200_DBDF_PCM) ? dbd + hd.off_pcm : nullptr;
    a.log2_min_pu = (int)hd.log2_min_pu_size; a.min_pu_w = (int)hd.min_pu_width; a.min_pu_h = (int)hd.min_pu_height;
    a.cb_qp_offset = hd.cb_qp_offset; a.cr_qp_offset = hd.cr_qp_offset;
    a.width = h.width; a.height = h.height; a.cfi = h.chroma_format_idc; a.log2_ctb = h.log2_ctb_size; a.ctb_w = ctb_w;
    a.rt = rt;
    cudaMemsetAsync(maps.mot, 0, maps_bytes, st);                    // one allocation: motion map (0 = intra), cbf, bs, grid
    int n = 0;
    uint32_t most = a.mc.count;
    for (int k = 0; k < 4; k++) if (a.tu[k].count > most) most = a.tu[k].count;
    if (most) { B200_LAUNCH((most + 255) / 256, 256, 0, st, k_dbd_raster)(a, maps, gate); n++; }
    if (a.n_leaf) { B200_LAUNCH((a.n_leaf + 7) / 8, 256, 0, st, k_dbd_bs)(a, maps, gate); n++; }
    const dim3 g((a.width / 8 + 255) / 256, a.height / 8, 4);
    B200_LAUNCH(g, 256, 0, st, k_dbd_params)(a, maps, L, gate); n++;
    if (check) { B200_LAUNCH((L.total + 255) / 256, 256, 0, st, k_dbd_compare)(maps.grid, check, L.total, gate); n++; }
    return n;
}

int launch_sao(cudaStream_t st, const B200SaoRec *grid, const FrameDesc &src, const FrameDesc &dst, int bd,
               int log2_ctb, int ctb_w, int ctb_h, int cfi, const uint32_t *tqb_words, const B200CipHeader *tqb_hdr)
{
    TqbDesc tq;
    tq.bits = nullptr; tq.log2_pu = 2; tq.pu_w = 0;
    if (tqb_words && tqb_hdr) { tq.bits = tqb_words + 4; tq.log2_pu = (int)tqb_hdr->log2_min_pu_size; tq.pu_w = (int)tqb_hdr->min_pu_width; }
    // warp tiles: (CTB width, at most 64) x (32 / strips x SAO_R) samples, all planes in one linear index
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
    if (bd > 8) B200_LAUNCH(blocks, 256, 0, st, k_sao<uint16_t>)(grid, src, dst, bd, log2_ctb, ctb_w, ctb_h, cfi, tb, tx, tq);
    else        B200_LAUNCH(blocks, 256, 0, st, k_sao<uint8_t>)(grid, src, dst, bd, log2_ctb, ctb_w, ctb_h, cfi, tb, tx, tq);
    return 1;
}

int launch_fill(cudaStream_t st, const FrameDesc &f, int bd, int value)
{
    const dim3 g((f.p[0].w + 255) / 256, f.p[0].h, 3);
    if (bd > 8) B200_LAUNCH(g, 256, 0, st, k_fill<uint16_t>)(f, value);
    else        B200_LAUNCH(g, 256, 0, st, k_fill<uint8_t>)(f, value);
    return 1;
}

// --------------------------------------------------------------------------------------------
// YUV -> planar RGB for consumers on the device (b200_yuv_to_rgb): one thread per 2x2 luma tile, a warp covers 64 consecutive
// samples of two rows, so loads and stores of a warp are contiguous runs
#include "k_yuv_rgb.cuh"

template <typename PIX, typename OUT>
__global__ void __launch_bounds__(256) k_yuv_rgb(YuvRgbJob j, int nx, int ny)
{
    const int tx = blockIdx.x * blockDim.x + threadIdx.x, ty = blockIdx.y * blockDim.y + threadIdx.y;
    if (tx >= nx || ty >= ny) return;
    yuv_rgb_tile<PIX, OUT>(j, j.tx0 + tx, j.ty0 + ty);
}

int launch_yuv_rgb(cudaStream_t st, const YuvRgbJob &j, int bd, int out_float)
{
    const int nx = ((j.x0 + j.w - 1) >> 1) - j.tx0 + 1, ny = ((j.y0 + j.h - 1) >> 1) - j.ty0 + 1;
    const dim3 g((nx + 31) / 32, (ny + 7) / 8), b(32, 8);
    if (bd > 8) { if (out_float) B200_LAUNCH(g, b, 0, st, k_yuv_rgb<uint16_t, float>)(j, nx, ny); else B200_LAUNCH(g, b, 0, st, k_yuv_rgb<uint16_t, uint8_t>)(j, nx, ny); }
    else        { if (out_float) B200_LAUNCH(g, b, 0, st, k_yuv_rgb<uint8_t, float>)(j, nx, ny);  else B200_LAUNCH(g, b, 0, st, k_yuv_rgb<uint8_t, uint8_t>)(j, nx, ny); }
    return 1;
}
