"""GPU parity (-m gpu) of the residual (K2) and intra (K3) stages at the limits of their input space.

A systematic sweep rather than random structure.  Residual: every transform size on every plane, every kind (IDCT, DC,
DST, transform skip, transquant bypass, PCM), rdpcm off / horizontal / vertical on skip and bypass blocks, each block once
added in place and once parked for the intra stage, coefficients at +32767 / -32768, in the sign pattern of a DCT basis
vector (first-stage sums far beyond int16), as single impulses, as full-range noise; every col_limit from 1 to 2N+4 and 255;
destination samples at 0 and at the maximum.  Intra: all 35 modes at every size on every plane, every availability
combination the validation accepts, smoothing on and off, neighbours that are all 0, all max, alternating, exact linear
ramps on either side of the strong-smoothing threshold and corner / top / left values that push the mode-10 / mode-26
boundary filters past both ends; and a layout that tiles the planes densely in z-order, so that extreme values reach the
next TU through the edge records.  Blobs come from the C recorder (b200_rec_tu / b200_rec_intra / b200_rec_finish); the
device must equal the CPU oracle, and where the reference's own tables are built (oracle/_ref/libreplay_ref.so) the
oracle must equal them.  A numpy restatement counts how often each limit was really reached and fails if one never was."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib
from openhevc_b200 import FrameEngine, B200Error, _lib
from openhevc_b200 import worklist as W

pytestmark = pytest.mark.gpu

FORMATS = [(1, 8), (1, 10), (1, 12), (2, 10), (3, 8)]
# pictures whose planes are no multiple of the TU sizes: top_right_size / bottom_left_size below n at the borders
SMALL = [(72, 40, 1, 10), (40, 24, 3, 8), (24, 40, 2, 12)]
I16_MIN, I16_MAX = -32768, 32767
RDPCM_MODES = (0, W.TUF_RDPCM, W.TUF_RDPCM | W.TUF_RDPCM_VERT)
ALL_NEIGHBOURS = W.INF_UP_LEFT | W.INF_UP | W.INF_UP_RIGHT | W.INF_LEFT | W.INF_BOTTOM_LEFT

_COS = [64, 90, 90, 90, 89, 88, 87, 85, 83, 82, 80, 78, 75, 73, 70, 67, 64, 61, 57, 54, 50, 46, 43, 38, 36, 31, 25, 22, 18, 13, 9, 4, 0]


def _t32(k, n):
    m = ((2 * n + 1) * k) & 127
    return _COS[m] if m <= 32 else -_COS[64 - m] if m <= 64 else -_COS[m - 64] if m < 96 else _COS[128 - m]


T32 = np.array([[_t32(k, n) for n in range(32)] for k in range(32)], np.int64)     # HEVC core transform, T32[k][n]
DST4 = np.array([[29, 55, 74, 84], [74, 74, 0, -74], [84, -29, -74, 55], [55, -84, 74, -29]], np.int64)


def basis(kind, n):
    """B[j][r]: weight of input j in output r of the 1-D inverse transform"""
    return DST4 if kind == W.TU_DST else T32[::32 // n, :n]


def wrap16(v):
    return ((np.asarray(v, np.int64) + 32768) & 0xFFFF) - 32768


# ---------------------------------------------------------------------------------------------------------------------
# numpy restatement of the residual (hevcdsp_template.c:45-316), used to count the limits the sweep reaches
# ---------------------------------------------------------------------------------------------------------------------
def idct_keep(n, j, end):
    if n == 4:
        return True
    if n in (8, 16):
        return not (j & 1) or j < end
    if j & 1:
        return j < end
    if (j & 3) == 2:
        return (j >> 1) < end // 2
    return True


def residual(c, kind, flags, log2, col_limit, bd, count):
    """the residual of one TU as int64; `count` collects the limits it reached"""
    n = 1 << log2
    c = wrap16(c).reshape(n, n)
    if kind in (W.TU_IDCT, W.TU_DST):
        B = basis(kind, n)
        first = np.zeros((n, n), np.int64)
        lim2, lim = min(col_limit + 4, n), min(col_limit, n)
        for i in range(n):                                  # columns; the reference narrows the window every 4 columns
            keep = [j for j in range(n) if kind == W.TU_DST or idct_keep(n, j, lim2)]
            first[:, i] = (B[keep].T @ c[keep, i] + 64) >> 7
            if lim2 < n and (i & 3) == 0 and i:
                lim2 -= 4
        count["stage1_clip"] += int((first != np.clip(first, I16_MIN, I16_MAX)).any())
        first = np.clip(first, I16_MIN, I16_MAX)
        keep = [j for j in range(n) if kind == W.TU_DST or idct_keep(n, j, lim)]
        shift = 20 - bd
        second = (first[:, keep] @ B[keep] + (1 << (shift - 1))) >> shift
        count["stage2_clip"] += int((second != np.clip(second, I16_MIN, I16_MAX)).any())
        r = np.clip(second, I16_MIN, I16_MAX)
    elif kind == W.TU_DC:
        shift = 14 - bd
        r = np.full((n, n), wrap16((((c[0, 0] + 1) >> 1) + (1 << (shift - 1))) >> shift))
    elif kind == W.TU_SKIP:
        shift = 15 - bd - log2
        r = (c + (1 << (shift - 1))) >> shift if shift > 0 else c << -shift
        count["skip_shift_wrap"] += int((r != wrap16(r)).any())
        r = wrap16(r)
    else:
        r = c.copy()
    if flags & W.TUF_RDPCM:
        axis = 0 if flags & W.TUF_RDPCM_VERT else 1
        r = np.moveaxis(r, axis, 0).copy()
        wrapped = False
        for k in range(1, n):
            s = r[k] + r[k - 1]
            wrapped |= bool((s != wrap16(s)).any())
            r[k] = wrap16(s)
        count["rdpcm_wrap"] += int(wrapped)
        r = np.moveaxis(r, 0, axis)
    return r


# ---------------------------------------------------------------------------------------------------------------------
# blobs through the C recorder
# ---------------------------------------------------------------------------------------------------------------------
class Recorder:
    """one picture recorded the way the decoder's table calls arrive"""

    def __init__(self, geom, cur_slot=0):
        self.lib = _lib.load()
        w, h, cfi, bd = geom
        cfg = _lib.B200Config(0, w, h, cfi, bd, 6, 2, 2, 0, None, 0)
        self.r = C.c_void_p()
        assert self.lib.b200_rec_create(C.byref(cfg), C.byref(self.r)) == 0
        assert self.lib.b200_rec_begin(self.r, cur_slot, 0) == 0

    def tu(self, plane, x, y, log2, kind, flags, col_limit, coeffs, linked):
        c = np.ascontiguousarray(coeffs, np.int16)
        return self.lib.b200_rec_tu(self.r, plane, x, y, log2, kind, flags, col_limit, c.ctypes.data, linked)

    def pcm(self, plane, x, y, log2, samples):
        s = np.ascontiguousarray(samples, np.int16)
        assert self.lib.b200_rec_pcm(self.r, plane, x, y, log2, s.ctypes.data) == 0

    def intra(self, plane, x, y, log2, mode, flags, trs, bls):
        assert self.lib.b200_rec_intra(self.r, plane, x, y, log2, mode, flags, trs, bls) == 0

    def all_intra_cip(self, geom):
        """constrained_intra_pred with every min-PU intra: the general intra path, availability unchanged"""
        w, h = geom[0], geom[1]
        ones = np.ones((h >> 2) * (w >> 2), np.uint8)
        assert self.lib.b200_rec_set_cip(self.r, 2, w >> 2, h >> 2, ones.ctypes.data) == 0

    def finish(self):
        try:
            bp, nb = C.c_void_p(), C.c_uint64()
            assert self.lib.b200_rec_finish(self.r, C.byref(bp), C.byref(nb)) == 0
            return np.ctypeslib.as_array(C.cast(bp, C.POINTER(C.c_uint8)), (nb.value,)).copy()
        finally:
            self.lib.b200_rec_destroy(self.r)


def other_transport(blob, geom):
    """the same picture with every non-PCM TU in the other coefficient transport: dense blocks as (position, value) pairs of
    all their non-zero coefficients, pair lists as dense blocks (the recorder picks one form by density; both must agree)"""
    w, h, cfi, bd = geom
    hdr, secs = W.parse_blob(blob)
    pool, parts, o = secs[W.SEC_COEFF], [], 0
    tus = {}
    for k in range(4):
        recs = secs[W.SEC_TU4 + k].copy()
        for i in range(len(recs)):
            dense, park = W.tu_dense(recs[i], pool)
            head = [] if park is None else [park & 0xFFFF, park >> 16]
            if recs[i]["kind"] == W.TU_PCM or recs[i]["nnz"] != W.TU_DENSE:
                body, nnz = dense.astype(np.int64), W.TU_DENSE
            else:
                pos = np.flatnonzero(dense)
                body, nnz = np.stack([pos, dense[pos]], 1).reshape(-1), len(pos)
            words = wrap16(np.concatenate([np.array(head, np.int64), body]))
            recs["nnz"][i], recs["coeff_off"][i] = nnz, o
            pad = -len(words) % 8
            parts.append(np.concatenate([words, np.zeros(pad, np.int64)]).astype(np.int16))
            o += len(words) + pad
        tus[k + 2] = recs
    coeff = np.concatenate(parts) if parts else np.zeros(0, np.int16)
    return W.build_blob(w, h, cfi, bd, int(hdr["log2_ctb_size"]), int(hdr["cur_slot"]), coeff=coeff, tu=tus, intra=secs[W.SEC_INTRA].copy())


def assert_same(got, want, what):
    for p in range(3):
        bad = np.argwhere(np.asarray(got[p]) != np.asarray(want[p]))
        assert len(bad) == 0, f"{what} plane {p}: {len(bad)} samples differ, first at (y,x)={tuple(bad[0])} got {got[p][tuple(bad[0])]} want {want[p][tuple(bad[0])]}"


def check_picture(eng, blob, cur, what):
    """device == oracle (== reference tables), reconstruction in place in slot 0 from the uploaded planes `cur`"""
    oracle_lib.check_decode_order(blob)
    want = oracle_lib.execute(blob, [cur])
    if oracle_lib.ref_lib() is not None:
        assert_same(oracle_lib.ref_execute(blob, [cur]), want, what + " reference tables")
    eng.upload_slot(0, cur)
    assert_same(eng.decode(blob), want, what)
    return want


def noise_planes(geom, rng):
    w, h, cfi, bd = geom
    dt = np.uint16 if bd > 8 else np.uint8
    return [rng.integers(0, 1 << bd, W.plane_dims(w, h, cfi, p)[::-1]).astype(dt) for p in range(3)]


# ---------------------------------------------------------------------------------------------------------------------
# residual sweep
# ---------------------------------------------------------------------------------------------------------------------
def coefficient_sets(kind, log2, plane, rng, impulse_step):
    """(name, NxN int64) contents for one kind and size"""
    n = 1 << log2
    out = [("max", np.full((n, n), I16_MAX)), ("min", np.full((n, n), I16_MIN))]
    if kind in (W.TU_IDCT, W.TU_DST):
        B = basis(kind, n)
        for r in sorted({0, n // 2 - 1, n - 1, (plane * 5 + log2) % n}):        # output row / column whose basis the signs follow
            s = np.where(B[:, r] >= 0, 1, -1)
            out.append(("basis", np.outer(s, s) * I16_MAX))
            out.append(("basis-", np.outer(s, -s) * 32768))
        for k in range(0, n * n, impulse_step):
            c = np.zeros(n * n, np.int64)
            c[k] = (I16_MAX, I16_MIN, int(rng.integers(-4096, 4096)))[k % 3]
            out.append(("impulse", c.reshape(n, n)))
    out.append(("noise", rng.integers(I16_MIN, I16_MAX + 1, (n, n))))
    if kind in (W.TU_SKIP, W.TU_BYPASS):            # runs whose rdpcm running sums wrap
        run = np.full((n, n), 20000 if kind == W.TU_BYPASS else I16_MAX)
        run[:, ::3] = -run[:, ::3] // 2
        out.append(("runs", run))
        out.append(("runs-", -run))
    return out


def residual_blocks(geom, rng, impulse_step):
    """every (plane, log2, kind, flags, col_limit, coefficients, parked) of the sweep"""
    w, h, cfi, bd = geom
    blocks = []
    for plane in range(3):
        pw, ph = W.plane_dims(w, h, cfi, plane)
        for log2 in (2, 3, 4, 5):
            n = 1 << log2
            if n > min(pw, ph):
                continue
            limits = list(range(1, 2 * n + 5)) + [255]
            kinds = [W.TU_IDCT, W.TU_DC, W.TU_SKIP, W.TU_BYPASS, W.TU_PCM] + ([W.TU_DST] if plane == 0 and log2 == 2 else [])
            for kind in kinds:
                if kind == W.TU_PCM:
                    maxv = (1 << bd) - 1
                    for c in (np.zeros((n, n)), np.full((n, n), maxv), rng.integers(0, 2, (n, n)) * maxv):
                        blocks.append((plane, log2, kind, 0, 0, c, False))
                    continue
                for k, (name, c) in enumerate(coefficient_sets(kind, log2, plane, rng, impulse_step)):
                    for parked in (False, True):
                        flags = RDPCM_MODES[(k + parked) % 3] if kind in (W.TU_SKIP, W.TU_BYPASS) else 0
                        col_limit = limits[(3 * k + 7 * log2 + plane + parked) % len(limits)] if kind == W.TU_IDCT else n
                        blocks.append((plane, log2, kind, flags, col_limit, c, parked))
                        if kind in (W.TU_SKIP, W.TU_BYPASS) and name in ("runs", "runs-", "max"):
                            for f in RDPCM_MODES:                # every rdpcm direction over the wrapping content
                                if f != flags:
                                    blocks.append((plane, log2, kind, f, col_limit, c, parked))
    return blocks


def grid_places(pw, ph, n):
    return [(x, y) for y in range(0, ph - n + 1, n) for x in range(0, pw - n + 1, n)]


def run_residual_sweep(geom, seed, impulse_step=1):
    w, h, cfi, bd = geom
    maxv = (1 << bd) - 1
    rng = np.random.default_rng(seed)
    blocks = residual_blocks(geom, rng, impulse_step)
    count = dict(stage1_clip=0, stage2_clip=0, skip_shift_wrap=0, rdpcm_wrap=0, add_clip_lo=0, add_clip_hi=0, parked=0, pcm=0)
    # pictures: per plane, each size on its own grid of TU places; a picture takes as many blocks of each (plane, size)
    # as it has places for them, so the picture count is set by the fullest list
    queues = {}
    for b in blocks:
        queues.setdefault((b[0], b[1]), []).append(b)
    eng = FrameEngine(*geom, n_slots=2)
    try:
        pic = 0
        while any(queues.values()):
            cur = noise_planes(geom, rng)
            rec = Recorder(geom)
            direct = []
            for plane in range(3):
                pw, ph = W.plane_dims(w, h, cfi, plane)
                free = np.ones((ph, pw), bool)
                for log2 in (5, 4, 3, 2):
                    n = 1 << log2
                    q = queues.get((plane, log2), [])
                    for (x, y) in grid_places(pw, ph, n):
                        if not q:
                            break
                        if not free[y:y + n, x:x + n].all():
                            continue
                        free[y:y + n, x:x + n] = False
                        _, _, kind, flags, col_limit, c, parked = q.pop(0)
                        k = len(direct) + pic
                        if kind == W.TU_PCM:
                            rec.pcm(plane, x, y, log2, c)
                            count["pcm"] += 1
                            continue
                        if parked:
                            rec.intra(plane, x, y, log2, k % 35, 0, 0, 0)
                            assert rec.tu(plane, x, y, log2, kind, flags, col_limit, wrap16(c), 1) == 0
                            residual(c, kind, flags, log2, col_limit, bd, count)
                            count["parked"] += 1
                            continue
                        cur[plane][y:y + n, x:x + n] = (0, maxv, cur[plane][y:y + n, x:x + n])[k % 3]
                        assert rec.tu(plane, x, y, log2, kind, flags, col_limit, wrap16(c), 0) == 0
                        direct.append((plane, x, y, n, residual(c, kind, flags, log2, col_limit, bd, count)))
            blob = rec.finish()
            what = f"{geom} residual picture {pic}"
            want = check_picture(eng, blob, cur, what)
            eng.upload_slot(0, cur)
            assert_same(eng.decode(other_transport(blob, geom)), want, what + " other transport")
            for (plane, x, y, n, r) in direct:
                before = cur[plane][y:y + n, x:x + n].astype(np.int64) + r
                count["add_clip_lo"] += int((before < 0).any())
                count["add_clip_hi"] += int((before > maxv).any())
                # the restatement is the oracle's arithmetic: otherwise the counts above would prove nothing
                assert (np.clip(before, 0, maxv) == want[plane][y:y + n, x:x + n]).all(), f"{what}: numpy restatement differs at plane {plane} ({x},{y}) {n}x{n}"
            pic += 1
    finally:
        eng.close()
    for key in ("stage1_clip", "rdpcm_wrap", "add_clip_lo", "add_clip_hi", "parked", "pcm") + (("stage2_clip",) if bd > 8 else ()) + (("skip_shift_wrap",) if bd == 12 else ()):
        assert count[key] > 0, f"{geom}: the sweep never reached {key} ({count})"
    return count


@pytest.mark.parametrize("cfi,bd", FORMATS)
def test_residual_sweep(cfi, bd):
    """every kind, size, plane, rdpcm direction and coefficient content above, direct and parked, recorder transport and the
    other one; impulses at every coefficient position"""
    run_residual_sweep((256, 128, cfi, bd), seed=10 * cfi + bd)


@pytest.mark.parametrize("w,h,cfi,bd", SMALL)
def test_residual_sweep_small_pictures(w, h, cfi, bd):
    run_residual_sweep((w, h, cfi, bd), seed=w + h + bd, impulse_step=7)


# ---------------------------------------------------------------------------------------------------------------------
# intra sweep: isolated TUs whose neighbours come from the uploaded picture
# ---------------------------------------------------------------------------------------------------------------------
CONTENTS = ("zero", "max", "alt", "ramp", "top_thr-1", "top_thr", "left_thr-1", "left_thr", "filter_hi", "filter_lo", "noise")
RESIDS = (None, I16_MAX, I16_MIN, "noise")


def neighbour_span(x, y, n, pw, ph):
    """(columns of the top row incl. the corner, rows of the left column incl. the corner) inside the plane"""
    return np.arange(x - 1, min(x + 2 * n, pw)), np.arange(y - 1, min(y + 2 * n, ph))


def fill_neighbours(plane, x, y, n, content, bd, rng):
    ph, pw = plane.shape
    maxv, thr = (1 << bd) - 1, 1 << (bd - 5)
    cols, rows = neighbour_span(x, y, n, pw, ph)
    k_top, k_left = np.arange(len(cols)), np.arange(len(rows))          # index + 1 into top[-1..2n-1] / left[-1..2n-1]
    if content in ("zero", "max"):
        top = left = np.full(max(len(cols), len(rows)), 0 if content == "zero" else maxv)
    elif content == "alt":
        top = left = (np.arange(max(len(cols), len(rows))) & 1) * maxv
    elif content.startswith(("ramp", "top_", "left_")):
        st, sl = (int(rng.integers(0, maxv // 70 + 1)) for _ in range(2))
        base = int(rng.integers(thr + 1, maxv - 65 * max(st, sl) - thr))
        top, left = base + st * np.arange(2 * n + 1), base + sl * np.arange(2 * n + 1)
        if content != "ramp":                                        # second difference at index 31 is exactly thr-1 or thr
            d = thr - 1 if content.endswith("-1") else thr
            (top if content.startswith("top") else left)[2 * n] += d
    elif content == "filter_hi":                                     # corner 0, top / left max: top[0] + (left[y] - corner) / 2 > max
        top = left = np.r_[0, np.full(2 * n, maxv)]
    elif content == "filter_lo":
        top = left = np.r_[maxv, np.zeros(2 * n, np.int64)]
    else:
        top, left = rng.integers(0, maxv + 1, 2 * n + 1), rng.integers(0, maxv + 1, 2 * n + 1)
    plane[y - 1, cols] = np.asarray(top)[k_top]
    plane[rows, x - 1] = np.asarray(left)[k_left]


def intra_specs(geom, plane, log2, start):
    """modes, availability, smoothing flags, neighbour content and parked residual of the TUs of one (plane, size)"""
    w, h, cfi, bd = geom
    filt = plane == 0 or cfi == 3                                    # where the reference can smooth (hevcpred_template.c:288)
    specs = []
    for i in range(70):
        j = start + i
        avail = (7 * i + j // 70) % 32                              # every availability combination, twice over the list
        flags = avail | (W.INF_FILTER if filt and (i // 35 + j) % 2 == 0 else 0) | (W.INF_STRONG if (i // 2) % 2 else 0)
        specs.append((i % 35, flags, CONTENTS[j % len(CONTENTS)], RESIDS[(j // 3) % len(RESIDS)]))
    if plane == 0 and log2 == 5:         # strong smoothing: exact ramps on both sides of the threshold, all neighbours present
        for k, content in enumerate(("ramp", "top_thr-1", "top_thr", "left_thr-1", "left_thr") * 2):
            specs.append(((0, 2, 18, 34, 7)[k % 5], ALL_NEIGHBOURS | W.INF_FILTER | W.INF_STRONG, content, None))
    if plane == 0 and log2 < 5:          # the boundary filters of modes 10 and 26 past 0 and past max
        for k, content in enumerate(("filter_hi", "filter_lo") * 2):
            specs.append(((10, 26)[k // 2], W.INF_UP_LEFT | W.INF_UP | W.INF_LEFT | (W.INF_FILTER if k & 1 else 0), content, None))
    return specs


def box_places(pw, ph, n):
    """TU origins 4 samples into boxes of (2n + 4)^2: the neighbours one TU reads are no other TU's and no other TU's
    neighbours; boxes at the right / bottom border may be cut, so the up-right / bottom-left sizes drop below n there"""
    return [(x + 4, y + 4) for y in range(0, ph - n - 3, 2 * n + 4) for x in range(0, pw - n - 3, 2 * n + 4)]


def intra_count(plane, x, y, n, log2, p, mode, flags, bd, count):
    """strong smoothing and boundary-filter clips, restated for TUs whose neighbours are all raw picture samples"""
    if flags & (W.INF_UP_LEFT | W.INF_UP | W.INF_LEFT) != (W.INF_UP_LEFT | W.INF_UP | W.INF_LEFT):
        return
    ph, pw = plane.shape
    maxv, thr = (1 << bd) - 1, 1 << (bd - 5)
    pl = plane.astype(np.int64)
    trs, bls = min(2 * n, pw - x) - n, min(2 * n, ph - y) - n
    top = np.r_[pl[y - 1, x - 1:x + n], pl[y - 1, x + n + np.minimum(np.arange(n), trs - 1)] if flags & W.INF_UP_RIGHT and trs > 0 else np.full(n, pl[y - 1, x + n - 1])]
    left = np.r_[pl[y - 1:y + n, x - 1], pl[y + n + np.minimum(np.arange(n), bls - 1), x - 1] if flags & W.INF_BOTTOM_LEFT and bls > 0 else np.full(n, pl[y + n - 1, x - 1])]
    if p == 0 and n < 32 and mode in (10, 26):
        v = top[1] + ((left[1:n + 1] - left[0]) >> 1) if mode == 26 else left[1] + ((top[1:n + 1] - top[0]) >> 1)
        count["filter_clip_lo"] += int((v < 0).any())
        count["filter_clip_hi"] += int((v > maxv).any())
    if p == 0 and log2 == 5 and flags & W.INF_FILTER and flags & W.INF_STRONG and mode != 1 and min(abs(mode - 26), abs(mode - 10)) > 0:
        d = max(abs(top[0] + top[64] - 2 * top[32]), abs(left[0] + left[64] - 2 * left[32]))
        count["strong"] += int(d < thr)
        count["strong_thr-1"] += int(d == thr - 1)
        count["strong_thr"] += int(d == thr)


def border_pictures(geom, sizes):
    """for every size and every up-right / bottom-left size t below n (multiples of 4): a TU at (pw - n - t, ph - n - t) on
    each plane that has room, so that the reference's own top_right_size / bottom_left_size is t on both sides"""
    w, h, cfi, bd = geom
    out = []
    for log2 in sizes:
        n = 1 << log2
        for t in range(4, n, 4):
            specs = []
            for plane in range(3):
                pw, ph = W.plane_dims(w, h, cfi, plane)
                if pw >= n + t + 4 and ph >= n + t + 4:
                    filt = W.INF_FILTER if plane == 0 or cfi == 3 else 0
                    k = t // 4 + log2 + plane
                    specs.append((plane, pw - n - t, ph - n - t, (k * 11) % 35, ALL_NEIGHBOURS | filt | W.INF_STRONG, CONTENTS[k % len(CONTENTS)], RESIDS[k % len(RESIDS)]))
            if specs:
                out.append((log2, specs))
    return out


def run_intra_sweep(geom, seed, sizes=(2, 3, 4, 5)):
    w, h, cfi, bd = geom
    rng = np.random.default_rng(seed)
    count = dict(strong=0, **{"strong_thr-1": 0, "strong_thr": 0}, filter_clip_lo=0, filter_clip_hi=0, resid_hi=0, resid_lo=0, cip=0)
    sides = set()                                                   # (n, "trs" / "bls", size below n) the sweep ran
    queues = {}
    for plane in range(3):
        pw, ph = W.plane_dims(w, h, cfi, plane)
        for log2 in sizes:
            if box_places(pw, ph, 1 << log2):
                queues[plane, log2] = intra_specs(geom, plane, log2, 5 * plane + log2)
    pictures = []                                                   # (log2, [(plane, x, y, mode, flags, content, resid)])
    while any(queues.values()):
        for log2 in sizes:                                           # one size per picture
            if not any(queues.get((p, log2)) for p in range(3)):
                continue
            specs = []
            for plane in range(3):
                pw, ph = W.plane_dims(w, h, cfi, plane)
                q = queues.get((plane, log2), [])
                for (x, y) in box_places(pw, ph, 1 << log2):
                    if not q:
                        break
                    specs.append((plane, x, y) + q.pop(0))
            pictures.append((log2, specs))
    pictures += border_pictures(geom, sizes)
    eng = FrameEngine(*geom, n_slots=2)
    try:
        for pic, (log2, specs) in enumerate(pictures):
            n = 1 << log2
            cur = noise_planes(geom, rng)
            placed = []
            for (plane, x, y, mode, flags, content, resid) in specs:
                pw, ph = W.plane_dims(w, h, cfi, plane)
                trs, bls = min(2 * n, pw - x) - n, min(2 * n, ph - y) - n
                if trs <= 0:
                    flags &= ~W.INF_UP_RIGHT
                if bls <= 0:
                    flags &= ~W.INF_BOTTOM_LEFT
                if flags & W.INF_UP_RIGHT and trs < n:
                    sides.add((n, "trs", trs))
                if flags & W.INF_BOTTOM_LEFT and bls < n:
                    sides.add((n, "bls", bls))
                fill_neighbours(cur[plane], x, y, n, content, bd, rng)
                placed.append((plane, x, y, log2, mode, flags, trs, bls, resid))
                intra_count(cur[plane], x, y, n, log2, plane, mode, flags, bd, count)
            for cip in ((False, True) if log2 <= 3 else (False,)):
                rec = Recorder(geom)
                for (plane, x, y, lg, mode, flags, trs, bls, resid) in placed:
                    rec.intra(plane, x, y, lg, mode, flags, trs, bls)
                    if resid is not None:
                        c = rng.integers(I16_MIN, I16_MAX + 1, (n, n)) if resid == "noise" else np.full((n, n), resid)
                        assert rec.tu(plane, x, y, lg, W.TU_BYPASS, 0, n, c, 1) == 0
                        if not cip:
                            count["resid_hi"] += int(resid == I16_MAX)
                            count["resid_lo"] += int(resid == I16_MIN)
                if cip:
                    rec.all_intra_cip(geom)
                    count["cip"] += 1
                check_picture(eng, rec.finish(), cur, f"{geom} intra {n}x{n} picture {pic}{' cip' if cip else ''}")
    finally:
        eng.close()
    for log2 in sizes:                  # every partial up-right / bottom-left size that fits the luma plane was run
        n = 1 << log2
        missing = [(n, side, t) for side in ("trs", "bls") for t in range(4, n, 4) if min(w, h) >= n + t + 4 and (n, side, t) not in sides]
        assert not missing, f"{geom}: no TU with {missing}"
    return count


@pytest.mark.parametrize("cfi,bd", FORMATS)
def test_intra_sweep(cfi, bd):
    """all 35 modes at every size on every plane, every availability combination, every up-right / bottom-left size below n,
    smoothing on and off, neighbour content at the limits; 4x4 / 8x8 pictures once more through the general path
    (constrained intra prediction, every PU intra)"""
    count = run_intra_sweep((256, 128, cfi, bd), seed=20 * cfi + bd)
    for key, v in count.items():
        assert v > 0, f"the sweep never reached {key} ({count})"


@pytest.mark.parametrize("w,h,cfi,bd", SMALL)
def test_intra_sweep_small_pictures(w, h, cfi, bd):
    run_intra_sweep((w, h, cfi, bd), seed=w * h + bd, sizes=(2, 3, 4))


# ---------------------------------------------------------------------------------------------------------------------
# dense z-order layout: every neighbour is an intra TU of the same picture, read through the edge records
# ---------------------------------------------------------------------------------------------------------------------
def _morton(ux, uy):
    z = 0
    for i in range(3):
        z |= ((ux >> i) & 1) << (2 * i) | ((uy >> i) & 1) << (2 * i + 1)
    return z


def zorder_leaves(pw, ph, rng):
    """quadtree leaves of 4..32 samples covering the plane, in z-scan order within 32x32 blocks taken in raster order, with
    the availability a z-scan decode gives (6.4.1): (x, y, log2, flags, top_right_size, bottom_left_size)"""
    bw = (pw + 31) >> 5

    def z(x, y):
        return (((y >> 5) * bw + (x >> 5)) << 6) | _morton((x & 31) >> 2, (y & 31) >> 2)

    leaves = []

    def quad(x, y, log2):
        n = 1 << log2
        if x >= pw or y >= ph:
            return
        if log2 > 2 and (x + n > pw or y + n > ph or rng.random() < 0.6):
            for dy in (0, n // 2):
                for dx in (0, n // 2):
                    quad(x + dx, y + dy, log2 - 1)
            return
        cur = z(x, y)
        trs, bls = min(2 * n, pw - x) - n, min(2 * n, ph - y) - n
        f = (W.INF_UP if y else 0) | (W.INF_LEFT if x else 0) | (W.INF_UP_LEFT if x and y else 0)
        f |= W.INF_UP_RIGHT if y and trs > 0 and z(x + n, y - 1) < cur else 0
        f |= W.INF_BOTTOM_LEFT if x and bls > 0 and z(x - 1, y + n) < cur else 0
        f &= ~(rng.integers(0, 32) if rng.random() < 0.2 else 0)     # now and then a neighbour the decoder would not use
        leaves.append((x, y, log2, int(f), trs, bls))

    for by in range(0, ph, 32):
        for bx in range(0, pw, 32):
            quad(bx, by, 5)
    return leaves


def run_dense_intra(geom, seed):
    w, h, cfi, bd = geom
    rng = np.random.default_rng(seed)
    eng = FrameEngine(*geom, n_slots=2)
    try:
        for k in range(2):
            cur = noise_planes(geom, rng)
            plan = []
            for plane in range(3):
                pw, ph = W.plane_dims(w, h, cfi, plane)
                filt = plane == 0 or cfi == 3
                for i, (x, y, log2, f, trs, bls) in enumerate(zorder_leaves(pw, ph, rng)):
                    f |= (W.INF_FILTER if filt and rng.random() < 0.7 else 0) | (W.INF_STRONG if rng.random() < 0.7 else 0)
                    mode = int(rng.choice([0, 1, 10, 26, 2, 18, 34])) if rng.random() < 0.5 else int(rng.integers(0, 35))
                    resid = (I16_MAX, I16_MIN, None, "noise")[(i + k) % 4] if rng.random() < 0.8 else None
                    plan.append((plane, x, y, log2, mode, f, trs, bls, resid))
            for cip in (False, True):
                rec = Recorder(geom)
                for (plane, x, y, log2, mode, f, trs, bls, resid) in plan:
                    rec.intra(plane, x, y, log2, mode, f, trs, bls)
                    if resid is not None:
                        n = 1 << log2
                        c = np.random.default_rng(x * 7 + y).integers(I16_MIN, I16_MAX + 1, (n, n)) if resid == "noise" else np.full((n, n), resid)
                        assert rec.tu(plane, x, y, log2, W.TU_BYPASS if resid != "noise" else W.TU_IDCT, 0, n, c, 1) == 0
                if cip:
                    rec.all_intra_cip(geom)
                blob = rec.finish()
                hdr, secs = W.parse_blob(blob)
                intra = secs[W.SEC_INTRA]
                perm, levels = W.level_order(intra, w, h, cfi)
                assert (perm == np.arange(len(intra))).all() and levels > 1      # the recorder's list is in dependency order
                want = check_picture(eng, blob, cur, f"{geom} dense intra picture {k}{' cip' if cip else ''}")
                maxv = (1 << bd) - 1
                assert all((want[p] == maxv).any() and (want[p] == 0).any() for p in range(3))   # the extremes travel
    finally:
        eng.close()


@pytest.mark.parametrize("w,h,cfi,bd", [(256, 128, 1, 12), (256, 128, 3, 8), (72, 40, 2, 10)])
def test_intra_dense_zorder(w, h, cfi, bd):
    """extreme values (12-bit maxima through the 15-bit edge records) reach the next TU through the wavefront's edge records"""
    run_dense_intra((w, h, cfi, bd), seed=w + bd)


# ---------------------------------------------------------------------------------------------------------------------
# constrained intra prediction in inter pictures
# ---------------------------------------------------------------------------------------------------------------------
def all_intra_cip(blob):
    """the same picture with every min-PU of its constrained_intra_pred bitmap intra"""
    out = blob.copy()
    hdr = W.parse_blob(out)[0]
    off, count = int(hdr["cip"]["off"]), int(hdr["cip"]["count"])
    out[off + 16:off + 4 * count] = 0xff
    return out


CIP_CASES = [(1, 8, 0.12, 1.0), (1, 10, 0.45, 1.0), (2, 10, 0.3, 2.0), (3, 8, 0.6, 0.5), (1, 12, 0.8, 2.0)]     # cfi, bd, p_intra, split_bias


@pytest.mark.late
@pytest.mark.parametrize("cfi,bd,p_intra,split", CIP_CASES)
def test_constrained_intra_rules(cfi, bd, p_intra, split):
    """cip_flags() / cip_substitute() (k_intra_cip.cuh, run by lane 0 of k_intra) against the oracle's restatement of
    hevcpred_template.c:116-249, for every intra TU of synthetic inter pictures over noise references.  A picture shows only
    the reference entries its modes read, so each one runs with every intra TU at mode 2, at 18 and at 34, strong smoothing
    off: between them these read every entry [-1 .. 2N-1] of both arrays, and a wrong entry or flag changes a sample."""
    from openhevc_b200.synth import FrameSynth
    w, h = 320, 192
    geom = (w, h, cfi, bd)
    blob, st = FrameSynth(w, h, cfi=cfi, bit_depth=bd, seed=500 + cfi + bd, refs=[1], cur_slot=0, cip=True, p_intra=p_intra, split_bias=split).generate()
    assert int(W.parse_blob(blob)[0]["flags"]) & W.FRAME_CIP
    rng = np.random.default_rng(9)
    dpb = [noise_planes(geom, rng) for _ in range(2)]                 # noise: any mix-up of two samples shows
    eng = FrameEngine(*geom, n_slots=2)
    try:
        eng.upload_slot(1, dpb[1])
        for mode in (2, 18, 34):
            b = blob.copy()
            intra = W.parse_blob(b)[1][W.SEC_INTRA]
            intra["mode"] = mode
            intra["flags"] &= 0xff ^ W.INF_STRONG
            want = oracle_lib.execute(b, dpb)
            every = oracle_lib.execute(all_intra_cip(b), dpb)
            changed = sum(bool((want[p][y:y + n, x:x + n] != every[p][y:y + n, x:x + n]).any())
                          for p, x, y, n in zip(intra["plane"], intra["x"], intra["y"], 1 << intra["log2"].astype(int)))
            assert changed > 10, "the constrained-intra rule never removed a candidate: the test picture does not exercise it"
            eng.upload_slot(0, dpb[0])
            assert_same(eng.decode(b), want, f"{geom} mode {mode}")
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# rdpcm on blocks the device transforms in another order
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.late
def test_rdpcm_on_transformed_or_pcm_blocks_is_rejected():
    """rdpcm follows transform skip or transquant bypass only (hevc_cabac.c:1873,1892).  The device applies the vertical
    running sum between its two transform stages and would apply it to PCM samples too, where the reference transforms
    first and never touches PCM: a record with rdpcm on an IDCT, DST or PCM block must be rejected, not executed, and the
    recorder must refuse to write one."""
    geom = (64, 32, 1, 8)
    rng = np.random.default_rng(3)
    coeffs8, coeffs4, pcm8 = rng.integers(-200, 200, (8, 8)), rng.integers(-200, 200, (4, 4)), rng.integers(0, 256, (8, 8))
    # the good picture: an IDCT 8x8, a DC 8x8, a DST 4x4 and a PCM 8x8 block, and skip / bypass blocks with rdpcm
    rec = Recorder(geom)
    assert rec.tu(0, 0, 0, 3, W.TU_IDCT, 0, 8, coeffs8, 0) == 0
    assert rec.tu(0, 0, 8, 3, W.TU_DC, 0, 8, coeffs8, 0) == 0
    assert rec.tu(0, 8, 0, 2, W.TU_DST, 0, 4, coeffs4, 0) == 0
    rec.pcm(0, 16, 0, 3, pcm8)
    assert rec.tu(0, 24, 0, 2, W.TU_SKIP, W.TUF_RDPCM | W.TUF_RDPCM_VERT, 4, coeffs4, 0) == 0
    assert rec.tu(0, 32, 0, 3, W.TU_BYPASS, W.TUF_RDPCM, 8, coeffs8, 0) == 0
    good = rec.finish()
    cur = noise_planes(geom, rng)
    eng = FrameEngine(*geom, n_slots=2, n_lanes=1)
    try:
        first = check_picture(eng, good, cur, "good picture")
        for sec, kind, flags in ((W.SEC_TU8, W.TU_IDCT, W.TUF_RDPCM | W.TUF_RDPCM_VERT), (W.SEC_TU4, W.TU_DST, W.TUF_RDPCM | W.TUF_RDPCM_VERT),
                                 (W.SEC_TU8, W.TU_PCM, W.TUF_RDPCM), (W.SEC_TU8, W.TU_PCM, W.TUF_RDPCM | W.TUF_RDPCM_VERT),
                                 (W.SEC_TU8, W.TU_DC, W.TUF_RDPCM)):
            bad = good.copy()
            tus = W.parse_blob(bad)[1][sec]
            tus["flags"][tus["kind"] == kind] |= flags
            eng.upload_slot(0, cur)
            with pytest.raises(B200Error, match="rejected on the device"):
                eng.decode(bad)
            eng.upload_slot(0, cur)
            assert_same(eng.decode(good), first, f"good picture after rdpcm on kind {kind}")
    finally:
        eng.close()
    rec = Recorder(geom)
    for kind, log2, c in ((W.TU_IDCT, 3, coeffs8), (W.TU_DST, 2, coeffs4), (W.TU_DC, 3, coeffs8), (W.TU_PCM, 3, pcm8)):
        for flags in (W.TUF_RDPCM, W.TUF_RDPCM | W.TUF_RDPCM_VERT):
            assert rec.tu(0, 0, 0, log2, kind, flags, 1 << log2, c, 0) == -1, (kind, flags)      # B200_EINVAL
    rec.finish()
