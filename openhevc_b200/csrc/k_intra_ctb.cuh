// k_intra_ctb.cuh — K3, CTB-granular: one thread block per CTB, the CTB's samples in shared memory.
//
// The TU-granular stage (k_intra, kernels.cu) pays one L2 round trip per dependent transform block, on each step of a
// ~3400-step chain on a 4K intra picture.  Most of those steps stay inside one CTB.  Here a block owns a CTB:
//   * the CTB's reconstruction (all three planes), its residuals and its records are staged in shared memory while the block
//     waits for its neighbour CTBs -- left, up-left, up, up-right: the wavefront of hevc.c:2751-2832 -- whose borders it then
//     reads from the picture (one row above, one column to the left);
//   * inside the CTB the records are ordered by dependency level (b200_intra_ctb_order, recorder.cpp): the block's warps take
//     the transform blocks of one level in parallel, one barrier per level, neighbours come from shared memory (~100 ns a step);
//   * a finished CTB publishes one flag (release); a waiting block polls the flags of its neighbours (acquire), not samples.
// Blocks are persistent and take CTBs in raster order from a ticket, so every CTB a block waits for has been taken by a block
// that is running: no dead lock, whatever the number of resident blocks.  No edge records, no initialisation pass over the
// picture.  constrained_intra_pred pictures keep the TU-granular stage (they need the picture's PU types per sample).
#pragma once

#define ICTB_WARPS 8
#define ICTB_MAXREC 768                 // 64x64 CTB of 4x4 blocks, 4:4:4: 3 x 256

struct IntraCtbArgs {
    const B200IntraRec *recs;
    const uint32_t *ctb_start;          // [n_ctb + 1]
    const int16_t *parked;
    uint32_t *counter;                  // lane counters: [0] ticket, [1] gate, [2] time-out latch
    uint32_t *done;                     // [n_ctb]: == gen once the CTB is reconstructed
    uint32_t gen;
    int n_ctb, ctb_w, log2_ctb, cfi, bd, count;
    unsigned long long parked_cap;      // int16 entries of the parked pool
    // shared-memory layout (bytes from the start of dynamic shared memory), computed by the launcher
    int tile_off[3], tile_stride[3];    // uint16 samples; column 0 = x0 - 1, row 0 = y0 - 1
    int rt_off[3], rt_stride[3];        // int16 residuals, origin = the CTB's origin
    int rec_off, scratch_off;           // uint4 records; per-warp int scratch for 16x16 / 32x32 blocks
};

__device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t *p)
{
#ifndef B200_EMUL
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
#else
    emu_yield();
    return __atomic_load_n(p, __ATOMIC_ACQUIRE);
#endif
}
__device__ __forceinline__ void st_release_u32(uint32_t *p, uint32_t v)
{
#ifndef B200_EMUL
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
#else
    __atomic_store_n(p, v, __ATOMIC_RELEASE);
#endif
}
template <typename PIX> __device__ __forceinline__ int ld_pix_cg(const PIX *p)      // bypass L1: written by another SM moments ago
{
#ifndef B200_EMUL
    return (int)__ldcg(p);
#else
    return (int)*p;
#endif
}

// One transform block, one warp.  tile: the plane's shared tile, S its stride, (tx, ty) the block's origin in tile coordinates
// (border included), res: the block's residual in the residual tile or null.  Arithmetic: hevcpred_template.c:250-538, as in k_intra.
template <typename PIX>
__device__ __forceinline__ void intra_tu_smem(const B200IntraRec &r, uint16_t *tile, int S, int rows, int tx, int ty, const int16_t *res, int RS,
                                              const PlaneDesc &pd, int bd, int lane, int *scr)
{
    // (indices a record could push beyond the tile -- a bottom-left block below the CTB, an up-right block beyond its row -- are
    // clamped: a legal list never asks for them, an illegal one must not read outside shared memory)
    const int cmax = S - 1 - tx, rmax = rows - 1 - ty;
    const unsigned FULL = 0xffffffffu;
    const int n = 1 << r.log2, n2 = 2 * n, maxv = (1 << bd) - 1, npx = n * n;
    const bool ul = r.flags & B200_INF_UP_LEFT, up = r.flags & B200_INF_UP, ur = r.flags & B200_INF_UP_RIGHT;
    const bool lf = r.flags & B200_INF_LEFT, bl = r.flags & B200_INF_BOTTOM_LEFT;
    const int trs = r.top_right_size, bls = r.bottom_left_size;
    const int mode = r.mode;
    const int angle = mode >= 2 ? c_intra_angle[mode - 2] : 0;
    const bool vertical = mode >= 18;
    const int inv = (mode >= 11 && mode <= 25) ? c_inv_angle[mode - 11] : 0;
    uint16_t *const t_top = tile + (ty - 1) * S + tx;          // [-1 .. 2n-1]: the row above, from the corner
    uint16_t *const t_org = tile + ty * S + tx;
    if (r.log2 <= 3) {
        // ---- 4x4 / 8x8: the <= 33 reference samples live one per lane (fT: lane k = top[k-1], fL: lane k = left[k]) ----
        int gT = 0, gL = 0;
        {
            const int t = lane - 1;
            const bool needT = lane == 0 ? ul : t < n ? up : (t < n2 && ur);
            const bool needL = lane < n ? lf : (lane < n2 && bl);
            if (needT) gT = t_top[lane == 0 ? -1 : min(min(t, n + trs - 1), cmax)];
            if (needL) gL = t_org[min(min(lane, n + bls - 1), rmax) * S - 1];
        }
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
        if ((r.flags & B200_INF_FILTER) && mode != 1 && n == 8) {
            const int d26 = abs(mode - 26), d10 = abs(mode - 10);
            if (min(d26, d10) > 7) {
                const int tm = __shfl_up_sync(FULL, fT, 1), tp = __shfl_down_sync(FULL, fT, 1);
                const int lm = __shfl_up_sync(FULL, fL, 1), lp = __shfl_down_sync(FULL, fL, 1);
                const int top0 = __shfl_sync(FULL, fT, 1), left0 = __shfl_sync(FULL, fL, 0);
                int qT, qL;
                if (lane == 0) qT = (left0 + 2 * corner + top0 + 2) >> 2;
                else if (lane == n2) qT = fT;
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
        const bool edge = r.plane == 0;
        const int topn_f = TOPS(n), leftn_f = LEFTS(n), top0_f = TOPS(0), left0_f = LEFTS(0);
#pragma unroll
        for (int it = 0; it < 2; it++) {
            const int i = lane + 32 * it;
            if (it * 32 >= npx) break;
            const int y = (i >> r.log2) & (n - 1), x = i & (n - 1);
            const int tyv = TOPS(x), lx = LEFTS(y);
            int v;
            if (mode == 0) {
                v = ((n - 1 - x) * lx + (x + 1) * topn_f + (n - 1 - y) * tyv + (y + 1) * leftn_f + n) >> (r.log2 + 1);
            } else if (mode == 1) {
                v = dc;
                if (edge) {
                    if (x == 0 && y == 0) v = (left0_f + 2 * dc + top0_f + 2) >> 2;
                    else if (y == 0) v = (tyv + 3 * dc + 2) >> 2;
                    else if (x == 0) v = (lx + 3 * dc + 2) >> 2;
                }
            } else {
                const int a = vertical ? y : x, b = vertical ? x : y;
                const int pos = (a + 1) * angle, id = pos >> 5, fact = pos & 31;
                const int k0 = b + id + 1, k1 = k0 + 1;
                const int j0 = k0 >= 0 ? k0 - 1 : -1 + ((k0 * inv + 128) >> 8), j1 = k1 >= 0 ? k1 - 1 : -1 + ((k1 * inv + 128) >> 8);
                const bool t0 = (k0 >= 0) == vertical, t1 = (k1 >= 0) == vertical;
                const int a0 = __shfl_sync(FULL, fT, (j0 + 1) & 31), b0 = __shfl_sync(FULL, fL, j0 & 31);
                const int a1 = __shfl_sync(FULL, fT, (j1 + 1) & 31), b1 = __shfl_sync(FULL, fL, j1 & 31);
                const int r0 = (t0 || j0 < 0) ? a0 : b0, r1 = (t1 || j1 < 0) ? a1 : b1;
                v = fact ? ((32 - fact) * r0 + fact * r1 + 16) >> 5 : r0;
                if (edge) {
                    if (mode == 26 && x == 0) v = clip3i(top0_f + ((lx - cornerf) >> 1), 0, maxv);
                    if (mode == 10 && y == 0) v = clip3i(left0_f + ((tyv - cornerf) >> 1), 0, maxv);
                }
            }
            if (i < npx) {
                if (res) v = clip3i(v + res[y * RS + x], 0, maxv);
                t_org[y * S + x] = (uint16_t)v;
                *px_ptr<PIX>(pd, r.x + x, r.y + y) = (PIX)v;
            }
        }
#undef TOPS
#undef LEFTS
        return;
    }
    // ---- 16x16 / 32x32: reference arrays in the warp's scratch ----
    int *gt = scr, *gl = scr + 66, *ft = scr + 132, *fleft = scr + 198, *qt = scr + 264, *ql = scr + 330;      // [k] holds index k - 1
    for (int k = lane; k <= n2; k += 32) {
        const int t = k - 1;
        int tv = 0, lv = 0;
        if (t < 0) { if (ul) tv = lv = t_top[-1]; }
        else {
            if (t < n ? up : ur) tv = t_top[min(t < n ? t : min(t, n + trs - 1), cmax)];
            if (t < n ? lf : bl) lv = t_org[min(t < n ? t : min(t, n + bls - 1), rmax) * S - 1];
        }
        gt[k] = tv; gl[k] = lv;
    }
    __syncwarp();
    {
        const int s = lf ? gl[n] : ul ? gl[0] : up ? gt[1] : ur ? gt[n + 1] : (1 << (bd - 1));
        const int bl0 = bl ? gl[n + 1] : s;
        const int l0 = lf ? gl[1] : bl0;
        const int corner = ul ? gl[0] : l0;
        const int un1 = up ? gt[n] : corner;
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
    const int *top = ft + 1, *left = fleft + 1;
    if ((r.flags & B200_INF_FILTER) && mode != 1) {
        const int d26 = abs(mode - 26), d10 = abs(mode - 10), dist = min(d26, d10);
        const int thr = r.log2 == 4 ? 1 : 0;
        if (dist > thr) {
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
    int dc = 0;
    if (mode == 1) {
        int sum = 0;
        for (int i = lane; i < n; i += 32) sum += left[i] + top[i];
#pragma unroll
        for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(FULL, sum, o);
        dc = (sum + n) >> (r.log2 + 1);
    }
    const int *mainr = vertical ? top : left, *side = vertical ? left : top;
    const bool edge = r.plane == 0 && n < 32;
    for (int i = lane; i < npx; i += 32) {
        const int y = i >> r.log2, x = i & (n - 1);
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
            const int a = vertical ? y : x, b = vertical ? x : y;
            const int pos = (a + 1) * angle, id = pos >> 5, fact = pos & 31;
            const int k0 = b + id + 1;
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
        if (res) v = clip3i(v + res[y * RS + x], 0, maxv);
        t_org[y * S + x] = (uint16_t)v;
        *px_ptr<PIX>(pd, r.x + x, r.y + y) = (PIX)v;
    }
    __syncwarp();
}

template <typename PIX>
__global__ void __launch_bounds__(ICTB_WARPS * 32) k_intra_ctb(IntraCtbArgs a, FrameDesc f)
{
    if (ld_relaxed(a.counter + 1)) return;               // the picture's work list failed validation
#ifdef B200_EMUL
    static __align__(16) uint8_t smem[160 * 1024];       // blocks run one after another in the emulation
#else
    extern __shared__ __align__(16) uint8_t smem[];
#endif
    __shared__ int s_ctb;
    __shared__ unsigned s_bad;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    uint4 *recs_s = reinterpret_cast<uint4 *>(smem + a.rec_off);
    int *scr = reinterpret_cast<int *>(smem + a.scratch_off) + warp * 400;
    const int ctb = 1 << a.log2_ctb;
    for (;;) {
        __syncthreads();                                  // everybody is done with the previous CTB's shared memory (and s_ctb)
        if (tid == 0) { s_ctb = (int)atomicAdd(a.counter, 1u); s_bad = 0; }
        __syncthreads();
        const int c = s_ctb;
        if (c >= a.n_ctb) break;
        const uint32_t start = __ldg(a.ctb_start + c), end = __ldg(a.ctb_start + c + 1);
        if (end <= start) continue;                       // no intra block in this CTB: complete after K1 / K2
        const int nrec = (int)(end - start);
        const int cxi = c % a.ctb_w, cyi = c / a.ctb_w;
        const int x0 = cxi << a.log2_ctb, y0 = cyi << a.log2_ctb;     // luma origin
        bool bad = nrec > ICTB_MAXREC || end > (uint32_t)a.count;
        // ---- stage: records, the CTB's samples as they stand after K1 / K2, the residuals (nothing here depends on the neighbours) ----
        if (!bad)
            for (int i = tid; i < nrec; i += ICTB_WARPS * 32) {
                const uint4 raw = __ldg(reinterpret_cast<const uint4 *>(a.recs + start) + i);
                recs_s[i] = raw;
                const int rx = raw.x & 0xffff, ry = raw.x >> 16, pl = raw.y & 0xff, lg = (raw.y >> 8) & 0xff;
                const int hs = pl && a.cfi != 3, vs = pl && a.cfi == 1;
                const int n = 1 << (lg & 7);
                if (pl > 2 || lg < 2 || lg > 5 || rx < (x0 >> hs) || ry < (y0 >> vs) || rx + n > ((x0 + ctb) >> hs) || ry + n > ((y0 + ctb) >> vs) ||
                    (raw.w != B200_NO_RESID && (unsigned long long)raw.w + n * n > a.parked_cap)) atomicOr(&s_bad, 1u);
            }
#pragma unroll
        for (int p = 0; p < 3; p++) {
            const int hs = p && a.cfi != 3, vs = p && a.cfi == 1;
            const PlaneDesc pd = plane_of(f, p);
            const int px0 = x0 >> hs, py0 = y0 >> vs, cw = min(ctb >> hs, pd.w - px0), chh = min(ctb >> vs, pd.h - py0);
            uint16_t *tile = reinterpret_cast<uint16_t *>(smem + a.tile_off[p]);
            const int S = a.tile_stride[p];
            for (int i = tid; i < cw * chh; i += ICTB_WARPS * 32) {
                const int y = i / cw, x = i - y * cw;
                tile[(y + 1) * S + x + 1] = *px_ptr<PIX>(pd, px0 + x, py0 + y);
            }
        }
        __syncthreads();
        bad = bad || s_bad != 0;
        if (!bad)
            for (int i = warp; i < nrec; i += ICTB_WARPS) {          // residuals: one warp per block, straight into the residual tile
                const uint4 raw = recs_s[i];
                if (raw.w == B200_NO_RESID) continue;
                const int rx = raw.x & 0xffff, ry = raw.x >> 16, pl = raw.y & 0xff, lg = (raw.y >> 8) & 0xff, n = 1 << lg;
                const int hs = pl && a.cfi != 3, vs = pl && a.cfi == 1;
                int16_t *rt = reinterpret_cast<int16_t *>(smem + (pl == 0 ? a.rt_off[0] : pl == 1 ? a.rt_off[1] : a.rt_off[2]));
                const int RS = pl == 0 ? a.rt_stride[0] : pl == 1 ? a.rt_stride[1] : a.rt_stride[2];
                const int16_t *src = a.parked + raw.w;
                int16_t *dst = rt + (ry - (y0 >> vs)) * RS + (rx - (x0 >> hs));
                for (int k = lane; k < n * n; k += 32) dst[(k >> lg) * RS + (k & (n - 1))] = src[k];
            }
        // ---- wait for the neighbour CTBs that reconstruct intra blocks themselves ----
        if (tid == 0 && !bad) {
            uint32_t spins = 0;
            const int nb[4] = { cxi > 0 ? c - 1 : -1, (cxi > 0 && cyi > 0) ? c - a.ctb_w - 1 : -1, cyi > 0 ? c - a.ctb_w : -1,
                                (cyi > 0 && cxi + 1 < a.ctb_w) ? c - a.ctb_w + 1 : -1 };
            for (int k = 0; k < 4; k++) {
                if (nb[k] < 0 || __ldg(a.ctb_start + nb[k]) == __ldg(a.ctb_start + nb[k] + 1)) continue;
                while (ld_acquire_u32(a.done + nb[k]) != a.gen) {
                    __nanosleep(40);
                    if ((++spins & 1023) == 0 && (spins > (1u << 21) || ld_relaxed(a.counter + 2) != 0)) { st_relaxed(a.counter + 2, 1u); latch_host(a.counter, 0x80000000u); break; }
                }
            }
        }
        __syncthreads();
        if (!bad) {
            // ---- borders: the row above (corner .. up-right) and the column to the left, from the picture ----
#pragma unroll
            for (int p = 0; p < 3; p++) {
                const int hs = p && a.cfi != 3, vs = p && a.cfi == 1;
                const PlaneDesc pd = plane_of(f, p);
                const int px0 = x0 >> hs, py0 = y0 >> vs, cw = ctb >> hs, chh = min(ctb >> vs, pd.h - py0);
                uint16_t *tile = reinterpret_cast<uint16_t *>(smem + a.tile_off[p]);
                const int S = a.tile_stride[p];
                const int ext = min(32, cw), wtop = 1 + cw + ext;
                if (py0 > 0)
                    for (int i = tid; i < wtop; i += ICTB_WARPS * 32) {
                        const int x = px0 - 1 + i;
                        if (x >= 0 && x < pd.w) tile[i] = (uint16_t)ld_pix_cg(px_ptr<PIX>(pd, x, py0 - 1));
                    }
                if (px0 > 0)
                    for (int i = tid; i < chh; i += ICTB_WARPS * 32) tile[(i + 1) * S] = (uint16_t)ld_pix_cg(px_ptr<PIX>(pd, px0 - 1, py0 + i));
            }
            __syncthreads();
            // ---- the CTB's transform blocks, level by level ----
            int pos = 0;
            while (pos < nrec) {
                const int lvl = (recs_s[pos].z >> 16) & 0xff;
                int cnt = 1;
                while (cnt < ICTB_WARPS && pos + cnt < nrec && (int)((recs_s[pos + cnt].z >> 16) & 0xff) == lvl) cnt++;
                if (warp < cnt) {
                    const uint4 raw = recs_s[pos + warp];
                    const B200IntraRec r = decode_intra(make_int4((int)raw.x, (int)raw.y, (int)raw.z, (int)raw.w));
                    const int pl = r.plane;
                    const int hs = pl && a.cfi != 3, vs = pl && a.cfi == 1;
                    uint16_t *tile = reinterpret_cast<uint16_t *>(smem + (pl == 0 ? a.tile_off[0] : pl == 1 ? a.tile_off[1] : a.tile_off[2]));
                    const int S = pl == 0 ? a.tile_stride[0] : pl == 1 ? a.tile_stride[1] : a.tile_stride[2];
                    const int RS = pl == 0 ? a.rt_stride[0] : pl == 1 ? a.rt_stride[1] : a.rt_stride[2];
                    const int16_t *rt = reinterpret_cast<const int16_t *>(smem + (pl == 0 ? a.rt_off[0] : pl == 1 ? a.rt_off[1] : a.rt_off[2]));
                    const int lx = r.x - (x0 >> hs), ly = r.y - (y0 >> vs);
                    intra_tu_smem<PIX>(r, tile, S, (ctb >> vs) + 1, lx + 1, ly + 1, r.resid_off != B200_NO_RESID ? rt + ly * RS + lx : nullptr, RS, plane_of(f, pl), a.bd, lane, scr);
                }
                pos += cnt;
                __syncthreads();
            }
        } else if (tid == 0) { a.counter[1] = 1u; atomicOr(a.counter + 3, 1u << B200_SEC_INTRA); latch_host(a.counter, 1u << B200_SEC_INTRA); }
        // ---- publish ----
        __threadfence();
        __syncthreads();
        if (tid == 0) st_release_u32(a.done + c, a.gen);
    }
}
