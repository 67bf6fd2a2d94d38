"""Synthetic per-picture work lists (SURVEY.md §8(d) "Synthetic inputs — kernel level").

No HEVC encoder or sample stream exists in the build environment, so the stimulus for parity
tests and for bench.py is generated here: a random but *syntax-consistent* coding structure
(CTB quadtrees in z-scan decode order, intra / inter CUs, residual quadtrees, PU partitions,
deblocking parameters from the reference's tc / beta tables, per-CTB SAO parameters), emitted
as exactly the records the recorder would produce for the same table calls.

Host-side test / benchmark input generation only; nothing here computes reconstructed pixels.
"""
import numpy as np

from . import worklist as W

# HEVC tables 8-12 (tc, beta) — the same constants as the reference's tctable / betatable (hevc_filter.c:50-60)
TC_TABLE = np.array([0] * 18 + [1] * 9 + [2] * 4 + [3] * 4 + [4] * 3 + [5, 5, 6, 6, 7, 8, 9, 10, 11, 13, 14, 16, 18, 20, 22, 24], np.int32)
BETA_TABLE = np.array([0] * 16 + list(range(6, 19)) + list(range(20, 66, 2)), np.int32)
QPC_TABLE = np.array([29, 30, 31, 32, 33, 33, 34, 34, 35, 35, 36, 36, 37, 37], np.int32)  # qp_c for 30..43 (ChromaArrayType 1)
assert len(TC_TABLE) == 54 and len(BETA_TABLE) == 52


def _morton(ux, uy, bits):
    z = 0
    for i in range(bits):
        z |= ((ux >> i) & 1) << (2 * i) | ((uy >> i) & 1) << (2 * i + 1)
    return z


class FrameSynth:
    """Generates one picture's work list.  `refs`: DPB slots usable as references (empty -> intra picture)."""

    def __init__(self, width, height, cfi=1, bit_depth=8, log2_ctb=6, seed=0, refs=(), cur_slot=0, poc=0,
                 p_intra=0.12, coded_frac=0.7, weighted=False, deblock=True, sao=True, sao_restore=False,
                 exotic=0.0, max_mv=64, split_bias=1.0, qp=32, bi_frac=0.6, cip=False):
        self.W, self.H, self.cfi, self.bd, self.log2_ctb = width, height, cfi, bit_depth, log2_ctb
        self.rng = np.random.default_rng(seed)
        self.refs, self.cur_slot, self.poc = list(refs), cur_slot, poc
        self.p_intra, self.coded_frac, self.weighted = p_intra, coded_frac, weighted
        self.deblock, self.sao, self.sao_restore, self.exotic = deblock, sao, sao_restore, exotic
        self.max_mv, self.split_bias, self.qp, self.bi_frac = max_mv, split_bias, qp, bi_frac
        self.cip = cip                                # constrained_intra_pred: the blob carries the intra bitmap of the min-PUs (4x4 luma)
        self.hs = 1 if cfi != 3 else 0
        self.vs = 1 if cfi == 1 else 0
        self.ctb = 1 << log2_ctb
        self.ctb_w = (width + self.ctb - 1) >> log2_ctb
        self.ctb_h = (height + self.ctb - 1) >> log2_ctb
        self.zbits = log2_ctb - 2
        n = 1 << self.zbits
        self.ztab = np.array([[_morton(x, y, self.zbits) for x in range(n)] for y in range(n)], np.int64)
        # per-4x4 luma maps used to derive deblocking parameters
        self.uw, self.uh = width // 4, height // 4
        self.bs_v = np.zeros((self.uh, self.uw), np.uint8)   # strength of the vertical edge on the LEFT of the unit
        self.bs_h = np.zeros((self.uh, self.uw), np.uint8)   # horizontal edge on TOP of the unit
        self.is_intra = np.zeros((self.uh, self.uw), bool)
        self.qp_map = np.full((height // 8, width // 8), qp, np.int32)
        self.tu = {2: [], 3: [], 4: [], 5: []}       # (plane, x, y, kind, flags, park, intra_index)
        self.intra = []                               # tuples
        self.mc = []
        self.stats = dict(mc_bytes=0, mc_samples=0, resid_samples=0, resid_parked=0, intra_samples=0, intra_bytes=0)

    # -- z-scan availability (6.4.1) ------------------------------------------------------------------
    def _z(self, x, y):
        cx, cy = x >> self.log2_ctb, y >> self.log2_ctb
        m = (1 << self.zbits) - 1
        return ((cy * self.ctb_w + cx) << (2 * self.zbits)) | int(self.ztab[(y >> 2) & m, (x >> 2) & m])

    def _avail(self, xl, yl, sl_h, sl_v):
        """neighbour flags + sizes for an intra block whose luma-coordinate footprint is (xl,yl,sl_h,sl_v)"""
        cur = self._z(xl, yl)
        up, left = yl > 0, xl > 0
        ur = up and xl + sl_h < self.W and self._z(xl + sl_h, yl - 1) < cur
        bl = left and yl + sl_v < self.H and self._z(xl - 1, yl + sl_v) < cur
        f = (W.INF_UP if up else 0) | (W.INF_LEFT if left else 0) | (W.INF_UP_LEFT if up and left else 0) | \
            (W.INF_UP_RIGHT if ur else 0) | (W.INF_BOTTOM_LEFT if bl else 0)
        trs = min(xl + 2 * sl_h, self.W) - (xl + sl_h)
        bls = min(yl + 2 * sl_v, self.H) - (yl + sl_v)
        return f, trs, bls

    # -- record emitters ---------------------------------------------------------------------------------
    def _emit_tu(self, plane, x, y, log2, intra_luma4, intra_idx):
        """one coded transform block (cbf = 1) at plane coordinates"""
        r = self.rng
        kind, flags = W.TU_IDCT, 0
        u = r.random()
        if intra_luma4 and plane == 0 and log2 == 2:
            kind = W.TU_DST
        if u < 0.15:
            kind = W.TU_DC if kind == W.TU_IDCT else kind
        elif u < 0.15 + 0.03 + self.exotic and log2 == 2:
            kind = W.TU_SKIP
            if r.random() < self.exotic:
                flags = W.TUF_RDPCM | (W.TUF_RDPCM_VERT if r.random() < 0.5 else 0)
        elif u > 1.0 - self.exotic:
            kind = W.TU_BYPASS
            if r.random() < 0.5:
                flags = W.TUF_RDPCM | (W.TUF_RDPCM_VERT if r.random() < 0.5 else 0)
        park = intra_idx is not None
        self.tu[log2].append((plane, x, y, kind, flags | (W.TUF_PARK if park else 0), intra_idx))
        n2 = 1 << (2 * log2)
        if park:
            self.stats["resid_parked"] += n2
        else:
            self.stats["resid_samples"] += n2

    def _emit_intra(self, plane, xl, yl, log2, mode):
        """intra_pred[log2-2](s, xl, yl, plane) with luma coordinates as in the reference (hevc.c:1215,1305)"""
        hs, vs = (self.hs, self.vs) if plane else (0, 0)
        n = 1 << log2
        f, trs, bls = self._avail(xl, yl, n << hs, n << vs)
        f |= W.INF_FILTER if (plane == 0 or self.cfi == 3) else 0
        f |= W.INF_STRONG
        self.intra.append([plane, xl >> hs, yl >> vs, log2, mode, f, trs >> hs, bls >> vs, W.NO_RESID])
        B = 2 if self.bd > 8 else 1
        self.stats["intra_samples"] += n * n
        self.stats["intra_bytes"] += B * (n * n + 4 * n + 1)
        return len(self.intra) - 1

    def _mark_edges(self, x, y, w, h, bs):
        """transform / prediction block boundary -> boundary strength on its left and top edges"""
        ux, uy, uw, uh = x >> 2, y >> 2, max(w >> 2, 1), max(h >> 2, 1)
        if x > 0:
            self.bs_v[uy:uy + uh, ux] = np.maximum(self.bs_v[uy:uy + uh, ux], bs)
        if y > 0:
            self.bs_h[uy, ux:ux + uw] = np.maximum(self.bs_h[uy, ux:ux + uw], bs)

    # -- coding tree ---------------------------------------------------------------------------------------
    def _chroma_tbs(self, xl, yl, log2_luma):
        """chroma transform blocks hanging off a luma TB of size log2_luma >= 3 (or the 8x8 parent of four 4x4s):
        list of (luma-coordinate x, y, log2_c)"""
        if self.cfi == 3:
            return [(xl, yl, log2_luma)]
        lc = log2_luma - 1
        if self.cfi == 2:
            return [(xl, yl, lc), (xl, yl + (1 << lc), lc)]
        return [(xl, yl, lc)]

    def _intra_tu(self, x, y, log2, modes, blk_parent=None, blk_idx=0):
        r = self.rng
        lmode, cmode = modes
        ii = self._emit_intra(0, x, y, log2, lmode)
        if r.random() < self.coded_frac:
            self._emit_tu(0, x, y, log2, True, ii)
            self.intra[ii][8] = -2          # resolved to the pool offset later
        self._mark_edges(x, y, 1 << log2, 1 << log2, 2)
        chroma = []
        if self.cfi == 3 or log2 > 2:
            chroma = self._chroma_tbs(x, y, log2)
        elif blk_idx == 3:
            chroma = self._chroma_tbs(blk_parent[0], blk_parent[1], 3)
        for plane in (1, 2):
            for (cx, cy, lc) in chroma:
                ii = self._emit_intra(plane, cx, cy, lc, cmode)
                if r.random() < self.coded_frac * 0.7:
                    self._emit_tu(plane, cx >> self.hs, cy >> self.vs, lc, True, ii)
                    self.intra[ii][8] = -2

    def _intra_tree(self, x, y, log2, modes, depth):
        if log2 > 5 or (log2 > 2 and depth < 2 and self.rng.random() < 0.25 * self.split_bias):
            h = 1 << (log2 - 1)
            for i, (dx, dy) in enumerate(((0, 0), (h, 0), (0, h), (h, h))):
                if log2 - 1 == 2:
                    self._intra_tu(x + dx, y + dy, 2, modes, (x, y), i)
                else:
                    self._intra_tree(x + dx, y + dy, log2 - 1, modes, depth + 1)
        else:
            self._intra_tu(x, y, log2, modes)

    def _inter_tree(self, x, y, log2, depth):
        r = self.rng
        if log2 > 5 or (log2 > 2 and depth < 2 and r.random() < 0.3 * self.split_bias):
            h = 1 << (log2 - 1)
            for dx, dy in ((0, 0), (h, 0), (0, h), (h, h)):
                self._inter_tree(x + dx, y + dy, log2 - 1, depth + 1)
            if log2 - 1 == 2 and self.cfi != 3:      # chroma of the four 4x4 luma blocks is coded once at the parent
                for plane in (1, 2):
                    for (cx, cy, lc) in self._chroma_tbs(x, y, 3):
                        if r.random() < self.coded_frac * 0.5:
                            self._emit_tu(plane, cx >> self.hs, cy >> self.vs, lc, False, None)
            return
        n = 1 << log2
        coded = False
        if r.random() < self.coded_frac:
            self._emit_tu(0, x, y, log2, False, None); coded = True
        if self.cfi == 3 or log2 > 2:
            for plane in (1, 2):
                for (cx, cy, lc) in self._chroma_tbs(x, y, log2):
                    if r.random() < self.coded_frac * 0.6:
                        self._emit_tu(plane, cx >> self.hs, cy >> self.vs, lc, False, None)
        self._mark_edges(x, y, n, n, 1 if coded else 0)

    def _pu(self, x, y, w, h):
        r = self.rng
        bi = r.random() < self.bi_frac and len(self.refs) > 0 and (w + h) != 12
        refs = [int(r.integers(0, len(self.refs))), int(r.integers(0, len(self.refs)))]     # indices into the reference table
        mvs = [(int(r.integers(-4 * self.max_mv, 4 * self.max_mv + 1)), int(r.integers(-4 * self.max_mv, 4 * self.max_mv + 1))) for _ in range(2)]
        if r.random() < 0.1:
            mvs[0] = (mvs[0][0] & ~3, mvs[0][1] & ~3)            # full-pel
        if r.random() < 0.1:
            mvs[1] = (mvs[1][0] & ~3, mvs[1][1])
        wts = [(int(r.integers(40, 89)), int(r.integers(-8, 9))) for _ in range(2)] if self.weighted else [(64, 0), (64, 0)]
        cwts = [(int(r.integers(40, 89)), int(r.integers(-8, 9))) for _ in range(2)] if self.weighted else [(64, 0), (64, 0)]
        B = 2 if self.bd > 8 else 1
        for plane in range(3):
            hs, vs = (self.hs, self.vs) if plane else (0, 0)
            pw_, ph_ = self.W >> hs, self.H >> vs
            bw, bh = w >> hs, h >> vs
            rec = dict(x=x >> hs, y=y >> vs, w=bw, h=bh, plane=plane,
                       flags=(W.MCF_BI if bi else 0) | (W.MCF_WEIGHTED if self.weighted else 0) | (W.MCF_CHROMA if plane else 0),
                       ref0=refs[0], ref1=refs[1], denom=6)
            nbytes = 0
            for l in range(2):
                mvx, mvy = mvs[l]
                if plane == 0:
                    fx, fy, ix, iy = mvx & 3, mvy & 3, mvx >> 2, mvy >> 2
                else:                                   # hevc.c:1807-1813: 1/8-pel index, units of the chroma grid
                    mx, my = mvx & ((1 << (2 + hs)) - 1), mvy & ((1 << (2 + vs)) - 1)
                    fx, fy = mx << (1 - hs), my << (1 - vs)
                    ix, iy = mvx >> (2 + hs), mvy >> (2 + vs)
                sx = min(max((x >> hs) + ix, -80), pw_ + 16)        # beyond that every sample clamps to the same border
                sy = min(max((y >> vs) + iy, -80), ph_ + 16)
                rec["sx%d" % l], rec["sy%d" % l], rec["frac%d" % l] = sx, sy, fx | (fy << 4)
                wt = wts[l] if plane == 0 else cwts[l]
                rec["w%d" % l], rec["o%d" % l] = wt
                if l == 0 or bi:
                    t = 3 if plane else 7
                    nbytes += B * (bw + (t if fx else 0)) * (bh + (t if fy else 0))
            self.mc.append(rec)
            self.stats["mc_bytes"] += nbytes + B * bw * bh
            self.stats["mc_samples"] += bw * bh
        self._mark_edges(x, y, w, h, 1 if r.random() < 0.5 else 0)

    def _cu(self, x, y, log2):
        r = self.rng
        n = 1 << log2
        intra = not self.refs or r.random() < self.p_intra
        qp = min(max(self.qp + int(r.integers(-4, 5)), 0), 51)
        self.qp_map[y >> 3:(y + n) >> 3, x >> 3:(x + n) >> 3] = qp
        self._mark_edges(x, y, n, n, 2 if intra else 1)
        if intra:
            self.is_intra[y >> 2:(y + n) >> 2, x >> 2:(x + n) >> 2] = True
            if 3 <= log2 <= 5 and r.random() < self.exotic * 0.5:
                # pcm_flag CU (hls_pcm_sample, hevc.c:1587-1623): raw samples for the three planes, no prediction, no residual
                self.tu[log2].append((0, x, y, W.TU_PCM, 0, None))
                for plane in (1, 2):
                    for (cx, cy, lc) in self._chroma_tbs(x, y, log2):
                        self.tu[lc].append((plane, cx >> self.hs, cy >> self.vs, W.TU_PCM, 0, None))
                self.stats["resid_samples"] += n * n * 3 // 2
                return
            lmode = int(r.integers(0, 35))
            cmode = int(r.choice([0, 1, 10, 26, 34, lmode]))
            if log2 == 3 and r.random() < 0.3:            # PART_NxN: four 4x4 luma blocks with their own modes
                for i, (dx, dy) in enumerate(((0, 0), (4, 0), (0, 4), (4, 4))):
                    self._intra_tu(x + dx, y + dy, 2, (int(r.integers(0, 35)), cmode), (x, y), i)
            else:
                self._intra_tree(x, y, log2, (lmode, cmode), 0)
            return
        # inter: prediction units (hevc.c:2103-2153), then the residual quadtree unless skipped
        u = r.random()
        if u < 0.65 or log2 == 3 and u < 0.8:
            parts = [(0, 0, n, n)]
        elif u < 0.8:
            parts = [(0, 0, n, n // 2), (0, n // 2, n, n // 2)]
        elif u < 0.92 or log2 == 3:
            parts = [(0, 0, n // 2, n), (n // 2, 0, n // 2, n)]
        else:                                               # AMP
            q = n // 4
            parts = [(0, 0, n, q), (0, q, n, n - q)] if r.random() < 0.5 else [(0, 0, q, n), (q, 0, n - q, n)]
        for (dx, dy, w, h) in parts:
            self._pu(x + dx, y + dy, w, h)
        if r.random() < 0.75:
            self._inter_tree(x, y, log2, 0)

    def _quadtree(self, x, y, log2):
        if x >= self.W or y >= self.H:
            return
        n = 1 << log2
        must = x + n > self.W or y + n > self.H
        p_split = {6: 0.85, 5: 0.6, 4: 0.35}.get(log2, 0.0) * self.split_bias
        if log2 > 3 and (must or self.rng.random() < p_split):
            h = n >> 1
            for dx, dy in ((0, 0), (h, 0), (0, h), (h, h)):
                self._quadtree(x + dx, y + dy, log2 - 1)
        else:
            self._cu(x, y, log2)

    # -- coefficient synthesis (vectorised per size) -----------------------------------------------------------
    def _coefficients(self):
        r = self.rng
        pool_parts, tu_arrays, off = [], {}, 0
        self._npark = 0
        for log2 in (2, 3, 4, 5):
            lst = self.tu[log2]
            m, n = len(lst), 1 << log2
            arr = np.zeros(m, W.tu_dt)
            if m:
                yy, xx = np.mgrid[0:n, 0:n]
                scale = r.uniform(0.6, 0.6 + n / 3.0, size=(m, 1, 1))
                prob = np.exp(-(xx + yy)[None] / scale)
                coef = (r.random((m, n, n)) < prob) * np.rint(r.laplace(0, 40, (m, n, n)))
                coef[:, 0, 0] += np.rint(r.laplace(0, 60, m))
                kinds = np.array([t[3] for t in lst])
                coef[kinds == W.TU_DC, :, :] *= (xx + yy == 0)
                big = r.random(m) < 0.02                   # a few saturating blocks
                coef[big] *= 40
                coef = np.clip(coef, -32768, 32767).astype(np.int16)
                pcm = kinds == W.TU_PCM
                if pcm.any():                                # PCM blocks carry final samples, already << (BD - pcm_bit_depth)
                    coef[pcm] = r.integers(0, 1 << self.bd, (int(pcm.sum()), n, n)).astype(np.int16)
                nz = coef != 0
                lx = np.where(nz.any(axis=1), np.arange(n)[None], 0).max(axis=1)
                ly = np.where(nz.any(axis=2), np.arange(n)[None], 0).max(axis=1)
                mxy = np.maximum(lx, ly)
                col_limit = lx + ly + 4                     # hevc_cabac.c:1927-1933
                col_limit = np.where(mxy < 4, np.minimum(4, col_limit), np.where(mxy < 8, np.minimum(8, col_limit), np.where(mxy < 12, np.minimum(24, col_limit), col_limit)))
                arr["plane"] = [t[0] for t in lst]; arr["x"] = [t[1] for t in lst]; arr["y"] = [t[2] for t in lst]
                arr["log2"] = log2; arr["kind"] = kinds; arr["flags"] = [t[4] for t in lst]
                arr["col_limit"] = np.minimum(col_limit, 255)
                # transport as the recorder does: sparse (position, value) pairs unless that is not smaller than the dense
                # block; PARK TUs carry their index in the parked-residual pool in front of their data
                flat = coef.reshape(m, n * n)
                cnt = (flat != 0).sum(axis=1)
                dense = pcm | (2 * cnt >= n * n)
                park = np.array([t[5] is not None for t in lst])
                size = np.where(dense, n * n, 2 * cnt) + 2 * park
                start = off + np.concatenate(([0], np.cumsum(size)[:-1]))
                part = np.zeros(int(size.sum()), np.int16)
                local = start - off
                if park.any():
                    po = self._npark + np.arange(int(park.sum())) * n * n
                    self._npark += int(park.sum()) * n * n
                    pidx = np.nonzero(park)[0]
                    part[local[pidx]] = (po & 0xffff).astype(np.uint16).view(np.int16)
                    part[local[pidx] + 1] = (po >> 16).astype(np.uint16).view(np.int16)
                    for k, o in zip(pidx, po):
                        self.intra[lst[k][5]][8] = int(o)
                data0 = local + 2 * park
                for k in np.nonzero(dense)[0]:
                    part[data0[k]:data0[k] + n * n] = flat[k]
                ti, pos = np.nonzero(np.where(dense[:, None], 0, flat))
                if len(ti):
                    rank = np.arange(len(ti)) - np.concatenate(([0], np.cumsum(np.bincount(ti, minlength=m))[:-1]))[ti]
                    part[data0[ti] + 2 * rank] = pos.astype(np.int16)
                    part[data0[ti] + 2 * rank + 1] = flat[ti, pos]
                arr["nnz"] = np.where(dense, W.TU_DENSE, cnt)
                arr["coeff_off"] = start
                pool_parts.append(part)
                off += int(size.sum())
            tu_arrays[log2] = arr
        pool = np.concatenate(pool_parts) if pool_parts else np.zeros(0, np.int16)
        return pool, tu_arrays

    # -- deblocking parameters from the block structure (hevc_filter.c:345-581) ---------------------------------
    def _deblock_grid(self, tc_offset=0, beta_offset=0):
        L = W.DbkLayout(self.W, self.H, self.cfi)
        grid = np.zeros(L.total, np.uint16)
        qp8 = self.qp_map
        # luma vertical edges: x = 8k, one entry per 4 rows
        for d in (0, 1):
            bs = self.bs_v if d == 0 else self.bs_h
            if d == 0:
                b = bs[:, 0::2]                                     # units on the 8-sample grid
                qa = np.repeat(qp8, 2, axis=0)                       # qp per 4-row segment
                q = (qa + np.roll(qa, 1, axis=1) + 1) >> 1           # (QpP + QpQ + 1) >> 1
                b = b.copy(); b[:, 0] = 0
            else:
                b = bs[0::2, :]
                qa = np.repeat(qp8, 2, axis=1)
                q = (qa + np.roll(qa, 1, axis=0) + 1) >> 1
                b = b.copy(); b[0, :] = 0
            tc = TC_TABLE[np.clip(q + 2 * (b.astype(np.int32) - 1) + tc_offset, 0, 53)]
            beta = BETA_TABLE[np.clip(q + beta_offset, 0, 51)]
            ent = np.where(b > 0, W.DBK_PRESENT | (tc & 63) | ((beta & 127) << 6), 0).astype(np.uint16)
            v = L.view(grid, 0, d)
            v[:ent.shape[0], :ent.shape[1]] = ent
            # chroma: only bs == 2, chroma grid of 8 samples (hevc_filter.c:424-478, 523-580)
            if self.cfi == 3:
                cb, cq = b, q
            elif d == 0:
                cb = b[::(2 if self.vs else 1), ::2]                  # every 2nd luma 8-column; one entry per 4 chroma rows
                cq = q[::(2 if self.vs else 1), ::2]
            else:
                cb = b[::(2 if self.vs else 1), ::(2 if self.hs else 1)] if self.vs else b[:, ::2]
                cq = q[::(2 if self.vs else 1), ::(2 if self.hs else 1)] if self.vs else q[:, ::2]
            qpc = np.where(cq < 30, cq, np.where(cq > 43, cq - 6, QPC_TABLE[np.clip(cq - 30, 0, 13)])) if self.cfi == 1 else np.minimum(cq, 51)
            ctc = TC_TABLE[np.clip(qpc + 2 + tc_offset, 0, 53)]
            cent = np.where(cb == 2, W.DBK_PRESENT | (ctc & 63), 0).astype(np.uint16)
            for plane in (1, 2):
                v = L.view(grid, plane, d)
                hh, ww = min(v.shape[0], cent.shape[0]), min(v.shape[1], cent.shape[1])
                v[:hh, :ww] = cent[:hh, :ww]
        return grid

    def _sao_grid(self):
        r = self.rng
        n = self.ctb_w * self.ctb_h
        g = np.zeros(3 * n, W.sao_dt)
        u = r.random(3 * n)
        g["type"] = np.where(u < 0.25, W.SAO_NONE, np.where(u < 0.5, W.SAO_BAND, W.SAO_EDGE))
        edge = g["type"] == W.SAO_EDGE
        g["param"] = np.where(edge, r.integers(0, 4, 3 * n), r.integers(0, 32, 3 * n))
        maxo = (1 << (min(self.bd, 10) - 5)) - 1
        mag = r.integers(0, maxo + 1, (3 * n, 4))
        sign = np.where(r.random((3 * n, 4)) < 0.5, -1, 1)
        sign[edge] = np.array([1, 1, -1, -1])            # edge offsets: first two positive, last two negative (hevc.c:1172-1177)
        g["offset_val"][:, 1:] = mag * sign
        cx = np.tile(np.arange(self.ctb_w), self.ctb_h); cy = np.repeat(np.arange(self.ctb_h), self.ctb_w)
        borders = (cx == 0) * 1 | (cy == 0) * 2 | (cx == self.ctb_w - 1) * 4 | (cy == self.ctb_h - 1) * 8
        g["borders"] = np.tile(borders, 3)
        if self.sao_restore:                                # slice / tile boundaries with filtering across disabled
            b = g["borders"]
            ve0 = ((b & 1) == 0) & (r.random(3 * n) < 0.3); ve1 = ((b & 4) == 0) & (r.random(3 * n) < 0.3)
            he0 = ((b & 2) == 0) & (r.random(3 * n) < 0.3); he1 = ((b & 8) == 0) & (r.random(3 * n) < 0.3)
            de0 = ((b & 3) == 0) & (r.random(3 * n) < 0.3); de1 = ((b & 6) == 0) & (r.random(3 * n) < 0.3)
            de2 = ((b & 12) == 0) & (r.random(3 * n) < 0.3); de3 = ((b & 9) == 0) & (r.random(3 * n) < 0.3)
            g["edges"] = ve0 | ve1 << 1 | he0 << 2 | he1 << 3 | de0 << 4 | de1 << 5 | de2 << 6 | de3 << 7
            g["variant"] = 1
        return g

    # -- public ---------------------------------------------------------------------------------------------------
    def generate(self, out=None):
        for cy in range(self.ctb_h):
            for cx in range(self.ctb_w):
                self._quadtree(cx << self.log2_ctb, cy << self.log2_ctb, self.log2_ctb)
        pool, tu = self._coefficients()
        intra = np.zeros(len(self.intra), W.intra_dt)
        if self.intra:
            a = np.array(self.intra, np.int64)
            for k, name in enumerate(("plane", "x", "y", "log2", "mode", "flags", "top_right_size", "bottom_left_size")):
                intra[name] = a[:, k]
            # sizes are only meaningful when the flag is set; keep the record canonical like the C recorder does
            intra["top_right_size"] = np.where(intra["flags"] & W.INF_UP_RIGHT, intra["top_right_size"], 0)
            intra["bottom_left_size"] = np.where(intra["flags"] & W.INF_BOTTOM_LEFT, intra["bottom_left_size"], 0)
            ro = a[:, 8]
            assert (ro != -2).all()
            intra["resid_off"] = np.where(ro < 0, W.NO_RESID, ro).astype(np.uint32)
            # picture-wide dependency-level order (the order k_intra takes the TUs in)
            perm, self.stats["intra_levels"] = W.level_order(intra, self.W, self.H, self.cfi)
            intra = intra[perm]
        mc = np.zeros(len(self.mc), W.mc_dt)
        if self.mc:
            for name in self.mc[0]:
                mc[name] = [rec[name] for rec in self.mc]
        mc = W.split_mc_tiles(mc)
        dbk = self._deblock_grid() if self.deblock else None
        sao = self._sao_grid() if self.sao else None
        blob = W.build_blob(self.W, self.H, self.cfi, self.bd, self.log2_ctb, self.cur_slot, self.poc, pool, tu, intra, mc, dbk, sao, out=out,
                            ref_slots=self.refs, cip=(2, self.is_intra) if self.cip else None)
        B = 2 if self.bd > 8 else 1
        S = sum(np.prod(W.plane_dims(self.W, self.H, self.cfi, p)) for p in range(3))
        st = self.stats
        st.update(samples=int(S), n_tu=sum(len(v) for v in tu.values()), n_intra=len(intra), n_mc_tiles=len(mc),
                  blob_bytes=int(blob.nbytes),
                  # algorithmic bytes per stage, SURVEY.md §8(d)
                  bytes_mc=int(st["mc_bytes"]),
                  # coefficient transport is sparse: the pool is read once; non-parked samples are read-modify-written,
                  # parked residuals are written (int16) for K3
                  bytes_residual=int(pool.nbytes + st["resid_samples"] * 2 * B + st["resid_parked"] * 2),
                  bytes_intra=int(st["intra_bytes"] + st["resid_parked"] * 2),
                  bytes_deblock=int(2 * B * S + (dbk.nbytes if dbk is not None else 0)) if self.deblock else 0,
                  bytes_sao=int(2 * B * S + (sao.nbytes if sao is not None else 0)) if self.sao else 0)
        st["bytes_total"] = st["bytes_mc"] + st["bytes_residual"] + st["bytes_intra"] + st["bytes_deblock"] + st["bytes_sao"]
        return blob, st


def smooth_frame(width, height, cfi, bit_depth, seed):
    """band-limited noise reference picture (sum of random 2-D cosines + small white noise), SURVEY.md §8(d)"""
    r = np.random.default_rng(seed)
    planes = []
    for p in range(3):
        pw, ph = W.plane_dims(width, height, cfi, p)
        yy, xx = np.mgrid[0:ph, 0:pw].astype(np.float32)
        v = np.zeros((ph, pw), np.float32)
        for _ in range(6):
            fx, fy, ph0 = r.uniform(-0.08, 0.08), r.uniform(-0.08, 0.08), r.uniform(0, 6.28)
            v += r.uniform(8, 28) * np.cos(fx * xx + fy * yy + ph0)
        v = 128 + v + r.integers(-4, 5, (ph, pw))
        v = np.clip(v, 16, 235) * (1 << (bit_depth - 8))
        planes.append(v.astype(np.uint16 if bit_depth > 8 else np.uint8))
    return planes
