"""GPU parity (-m gpu) of inter prediction (K1) at the limits of its input space.

A systematic sweep rather than random structure: every legal luma prediction-block shape with the chroma shapes each format
derives from it, all 16 luma and 64 chroma fraction pairs on each list, the four prediction modes, the whole legal range of
explicit weighted prediction (denominators 0..7, weights 2^denom + [-128, 127], offsets -128..127), reference content that
drives the 14-bit intermediate to its extremes, and source windows at every phase of the pair loads and at, over and far
beyond every picture border.  Each picture runs twice on the device: as a list of tiles (the numpy builder) and as a list of
whole prediction blocks that the device cuts into tiles (k_mc_expand; recorded through the C recorder, b200_rec_mc).  Both
must equal the CPU oracle, and where the reference's own tables are built (oracle/_ref/libreplay_ref.so) the oracle must equal
them as well.  Destination rectangles within a picture never overlap, so the order in which tiles run cannot matter."""
import numpy as np
import pytest

import oracle_lib
from oracle_lib import assert_same, padded_engine
from openhevc_b200 import FrameEngine, B200Error
from openhevc_b200 import worklist as W
from openhevc_b200.synth import FrameSynth, smooth_frame

pytestmark = pytest.mark.gpu

QPEL = np.array([[0, 0, 0, 64, 0, 0, 0, 0], [-1, 4, -10, 58, 17, -5, 1, 0], [-1, 4, -11, 40, 40, -11, 4, -1], [0, 1, -5, 17, 58, -10, 4, -1]], np.int64)
EPEL = np.array([[0, 64, 0, 0], [-2, 58, 10, -2], [-4, 54, 16, -2], [-6, 46, 28, -4], [-4, 36, 36, -4], [-4, 28, 46, -6], [-2, 16, 54, -4], [-2, 10, 58, -2]], np.int64)
FORMATS = [(1, 8), (1, 10), (1, 12), (2, 10), (3, 8)]
# pictures smaller than a CTB or no multiple of it, with chroma planes whose width is no multiple of 8
SMALL = [(16, 16, 1, 8), (72, 40, 1, 10), (24, 40, 2, 10), (40, 24, 3, 8)]
MODES = (0, W.MCF_BI, W.MCF_WEIGHTED, W.MCF_BI | W.MCF_WEIGHTED)
WEIGHT_DELTA = (-128, -1, 0, 127)         # weight = 2^denom + delta (luma_weight_l0_delta range, hevc.c:251)
OFFSETS = (-128, 0, 127)
# where the source window of one list lies: inside at a given phase, exactly touching a border (left / right / top / bottom),
# hanging over a side or a corner by 1..taps samples, or entirely outside by a few hundred samples
PLACES = ("inside", "touch_l", "touch_r", "touch_t", "touch_b", "over_l", "over_r", "over_t", "over_b", "over_tl", "over_tr", "over_bl", "over_br", "far")
REF_SLOTS = [1, 2]


def luma_shapes():
    """the 24 luma prediction-block shapes: 2Nx2N, 2NxN, Nx2N and the four AMP partitions of 64..16 CUs (hevc.c:2103-2153),
    and 8x8, 8x4, 4x8 of 8x8 CUs"""
    out = []
    for n in (64, 32, 16, 8):
        out += [(n, n), (n, n // 2), (n // 2, n)]
        if n > 8:
            q = n // 4
            out += [(n, q), (n, n - q), (q, n), (n - q, n)]
    return out


def pack(shapes, width, height):
    """shelf packing of luma rectangles into pictures of width x height: one list of disjoint (x, y, w, h) per picture"""
    pics, cur, x, y, shelf = [], [], 0, 0, 0
    for (w, h) in sorted(shapes, key=lambda s: (-s[1], -s[0])):
        if x + w > width:
            x, y, shelf = 0, y + shelf, 0
        if y + h > height:
            pics.append(cur)
            cur, x, y, shelf = [], 0, 0, 0
        cur.append((x, y, w, h))
        x, shelf = x + w, max(shelf, h)
    return pics + [cur]


def _origin(place, axis, k, n, size, pair):
    """window origin on one axis (x: axis 0, y: axis 1) for a window of `size` samples in a plane of `n`"""
    d = 1 + k % 4 if pair == 4 else 1 + k % 8                  # overhang of 1..taps samples
    side = {0: ("l", "r"), 1: ("t", "b")}[axis]
    if place == "touch_" + side[0]:
        return 0
    if place == "touch_" + side[1]:
        if axis == 1:
            return n - size
        par = k & 1                                          # both skews of the even-aligned pair loads (kernels.cu: mc_win)
        return n - 2 * ((size + par + 1) >> 1) + par         # ax + Ws == n
    if place.startswith("over_") and side[0] in place[5:]:
        return -d
    if place.startswith("over_") and side[1] in place[5:]:
        return n - size + d
    if place == "far":
        return (-300, n + 190, -230, n + 260)[(k + 2 * axis) % 4] if (k + axis) % 2 == 0 else None
    return None


def source(place, k, j, w, h, pw, ph, mx, my, chroma):
    """(sx, sy) of list j of a w x h record: the window the filter reads starts `before` samples ahead of it"""
    taps, before = (4, 1) if chroma else (8, 3)
    bx, by = (before if mx else 0), (before if my else 0)
    cw, ch = w + (taps - 1 if mx else 0), h + (taps - 1 if my else 0)
    out = []
    for axis, n, size, b, phase in ((0, pw, cw, bx, (k + 3 * j) % 8), (1, ph, ch, by, (k // 8 + 5 * j) % 8)):
        o = _origin(place, axis, k, n, size, taps)
        if o is None:                                        # inside, source at phase `phase` of 8 (sx mod 8)
            first = (phase - b) % 8
            cands = list(range(first, n - size + 1, 8))
            o = cands[(k // 3) % len(cands)] if cands else first - 8
        out.append(o + b)
    return out


def sweep_records(rects, geom, k, content):
    """one record per plane for every luma rectangle; k = (luma, chroma) running record index of the sweep (advanced in place)"""
    width, height, cfi, bd = geom
    hs, vs = (1 if cfi != 3 else 0), (1 if cfi == 1 else 0)
    recs = []
    for (x, y, w, h) in rects:
        for plane in range(3):
            chroma = plane > 0
            s, t = (hs, vs) if chroma else (0, 0)
            pw, ph = W.plane_dims(width, height, cfi, plane)
            n_frac, bits = (64, 3) if chroma else (16, 2)
            i = k[1 if chroma else 0]
            k[1 if chroma else 0] += 1
            f0 = i % n_frac
            f1 = ((9 if chroma else 5) * f0 + 3 + i // n_frac) % n_frac
            flags = MODES[(i // n_frac + i) % 4] | (W.MCF_CHROMA if chroma else 0)
            bi = flags & W.MCF_BI
            place0, place1 = PLACES[i % len(PLACES)], PLACES[(3 * i + 5) % len(PLACES)]
            if content == "sign" and bi and not chroma:
                f0, place0 = 2 | (2 << bits), "inside"          # list 0 at (2, 2) over the sign pattern: the int16 wrap
            denom = (i + i // 8) % 8
            r = dict(x=x >> s, y=y >> t, w=w >> s, h=h >> t, plane=plane, flags=flags, denom=denom,
                     ref0=0 if content == "sign" else i % 2, ref1=(i // 2) % 2,
                     w0=(1 << denom) + WEIGHT_DELTA[i % 4], w1=(1 << denom) + WEIGHT_DELTA[(i // 4 + 1) % 4],
                     o0=OFFSETS[i % 3], o1=OFFSETS[(i // 3 + 1) % 3])
            for j, (f, place) in enumerate(((f0, place0), (f1, place1))):
                mx, my = f & ((1 << bits) - 1), f >> bits
                r["frac%d" % j] = mx | (my << 4)
                r["sx%d" % j], r["sy%d" % j] = source(place, i, j, r["w"], r["h"], pw, ph, mx, my, chroma)
            recs.append(r)
    out = np.zeros(len(recs), W.mc_dt)
    for name in recs[0]:
        out[name] = [r[name] for r in recs]
    return out


def sign_pattern(shape, taps, frac, maxv, complement=False):
    """maxv where the 2-D filter tap product at (x mod taps, y mod taps) is positive (negative for the complement), else 0: the
    content that drives the 2-D intermediate of that fraction to its maximum (minimum) at every taps-th sample"""
    f = (QPEL if taps == 8 else EPEL)[frac]
    prod = np.outer(f, f)[np.arange(shape[0])[:, None] % taps, np.arange(shape[1])[None, :] % taps]
    return np.where(prod < 0 if complement else prod > 0, maxv, 0)


def references(geom, content, seed):
    """DPB of three slots: 0 the picture's background, 1 and 2 the references (list 0 of the sign content reads slot 1)"""
    width, height, cfi, bd = geom
    rng = np.random.default_rng(seed)
    maxv = (1 << bd) - 1
    dt = np.uint16 if bd > 8 else np.uint8
    dpb = []
    for slot in range(3):
        planes = []
        for p in range(3):
            pw, ph = W.plane_dims(width, height, cfi, p)
            if slot == 0 or content == "noise":
                v = rng.integers(0, maxv + 1, (ph, pw))
            elif content == "zero":
                v = np.zeros((ph, pw))
            elif content == "max":
                v = np.full((ph, pw), maxv)
            else:
                v = sign_pattern((ph, pw), 4 if p else 8, 4 if p else 2, maxv, complement=slot == 2)
            planes.append(v.astype(dt))
        dpb.append(planes)
    return dpb


def qpel_22_intermediate(ref, sx, sy, w, h, bd):
    """the 14-bit intermediate of luma fraction (2, 2) of a w x h block whose source is (sx, sy): put_hevc_qpel_hv
    (hevcdsp_template.c:763-790) with clamped addressing, computed without the int16 store of list 0"""
    f = QPEL[2]
    ys = np.clip(np.arange(sy - 3, sy + h + 4), 0, ref.shape[0] - 1)
    xs = np.clip(np.arange(sx - 3, sx + w + 4), 0, ref.shape[1] - 1)
    win = ref[np.ix_(ys, xs)].astype(np.int64)
    tmp = sum(f[i] * win[:, i:i + w] for i in range(8)) >> (bd - 8)
    assert np.abs(tmp).max() < 1 << 15                      # the first stage always fits the reference's int16 tmp[]
    return sum(f[j] * tmp[j:j + h] for j in range(8)) >> 6


def assert_list0_wraps(pictures, bd):
    """coverage guard: the bi-predicted luma records of the sign content really take list 0 beyond int16, up to the peak the
    filter table allows (33150 / 33247 / 33271 at 8 / 10 / 12 bits).  Without this the sweep could lose its reason to exist."""
    f, maxv = QPEL[2], (1 << bd) - 1
    pos, neg = int(f[f > 0].sum()), int(f[f < 0].sum())
    peak = (pos * ((pos * maxv) >> (bd - 8)) + neg * ((neg * maxv) >> (bd - 8))) >> 6
    assert peak > 32767
    hits = [qpel_22_intermediate(dpb[REF_SLOTS[m["ref0"]]][0], int(m["sx0"]), int(m["sy0"]), int(m["w"]), int(m["h"]), bd)
            for recs, dpb in pictures for m in recs if m["plane"] == 0 and m["flags"] & W.MCF_BI and m["frac0"] == 0x22]
    assert hits and max(int(v.max()) for v in hits) == peak
    assert sum(int((v > 32767).sum()) for v in hits) >= 8


def block_blob(geom, recs, cur_slot=0, poc=0):
    """the records as whole prediction blocks through the C recorder, the way the decoder's table calls arrive (b200_rec_mc):
    the blob carries B200BlobHeader.mc_tile_count and the device cuts the blocks into tiles itself (k_mc_expand)"""
    rec = W.Recorder(geom, cur_slot, poc)
    for block in recs:
        rec.mc(block)
    rec.set_refs(REF_SLOTS)
    return rec.finish()


def tile_blob(geom, recs):
    width, height, cfi, bd = geom
    return W.build_blob(width, height, cfi, bd, 6, 0, mc=W.split_mc_tiles(recs), ref_slots=REF_SLOTS)


def assert_disjoint(geom, recs):
    width, height, cfi, _ = geom
    for p in range(3):
        pw, ph = W.plane_dims(width, height, cfi, p)
        cover = np.zeros((ph, pw), np.int32)
        for m in recs[recs["plane"] == p]:
            cover[m["y"]:m["y"] + m["h"], m["x"]:m["x"] + m["w"]] += 1
        assert cover.max() <= 1, f"plane {p}: destinations overlap"


def check_picture(eng, geom, recs, dpb, what, reference_tables=True, blobs=None):
    """tile form and block form on the device, against the oracle (and the oracle against the reference's tables)"""
    assert_disjoint(geom, recs)
    tiles, blocks = blobs or (tile_blob(geom, recs), block_blob(geom, recs))
    want = oracle_lib.execute(tiles, dpb)
    assert_same(oracle_lib.execute(blocks, dpb), want, what + " oracle, block form")
    if reference_tables and oracle_lib.ref_lib() is not None:
        assert_same(oracle_lib.ref_execute(tiles, dpb), want, what + " reference tables")
    for slot in (1, 2):
        eng.upload_slot(slot, dpb[slot])
    for blob, form in ((tiles, "tile form"), (blocks, "block form")):
        eng.upload_slot(0, dpb[0])
        assert_same(eng.decode(blob), want, f"{what} {form}")


def run_sweep(geom, contents, rects_per_picture, seed, wrap_guard=True):
    eng = FrameEngine(*geom, n_slots=3)
    k, signed = [0, 0], []
    try:
        for c, content in enumerate(contents):
            for n, rects in enumerate(rects_per_picture):
                dpb = references(geom, content, seed + 10 * c + n)
                recs = sweep_records(rects, geom, k, content)
                if content == "sign":
                    signed.append((recs, dpb))
                check_picture(eng, geom, recs, dpb, f"{geom} {content} picture {n}")
    finally:
        eng.close()
    if wrap_guard:
        assert_list0_wraps(signed, geom[3])
    return k


@pytest.mark.parametrize("cfi,bd", FORMATS)
def test_mc_sweep(cfi, bd):
    """all 24 shapes in one 256x128 picture, once per reference content: the sign pattern (list 0 of every bi-predicted luma
    block at (2, 2): the intermediate exceeds int16 and the reference's int16 tmp[] wraps it) and its complement, all-zero,
    all-max and full-range noise.  Over the four pictures each list takes every luma and every chroma fraction pair."""
    geom = (256, 128, cfi, bd)
    pics = pack(luma_shapes(), 256, 128)
    assert len(pics) == 1 and len(pics[0]) == 24
    k = run_sweep(geom, ("sign", "zero", "max", "noise"), pics, seed=100 * cfi + bd)
    assert k[0] >= 64 and k[1] >= 128                       # every fraction pair on both lists, all four modes per pair


@pytest.mark.parametrize("w,h,cfi,bd", SMALL)
def test_mc_sweep_small_pictures(w, h, cfi, bd):
    """pictures of one partial CTB: every block is near a border, many windows hang over two of them"""
    pics = pack([s for s in luma_shapes() if s[0] <= w and s[1] <= h], w, h)
    run_sweep((w, h, cfi, bd), ("sign", "noise"), pics, seed=w + h + bd, wrap_guard=False)     # windows too large to lie inside


MC_CASES = [  # w, h, cfi, bd, FrameSynth arguments
    (256, 128, 1, 8, {}),
    (256, 128, 1, 10, dict(weighted=True)),
    (320, 192, 1, 10, dict(max_mv=150)),               # windows far outside the picture: clamped loads
    (192, 128, 2, 10, {}),
    (192, 128, 3, 8, dict(weighted=True)),
    (320, 192, 1, 12, dict(split_bias=2.5)),           # many small blocks
    (256, 192, 1, 10, dict(split_bias=0.3, bi_frac=0.2)),
]


@pytest.mark.late
@pytest.mark.parametrize("w,h,cfi,bd,kw", MC_CASES)
def test_mc_synthetic_pictures(w, h, cfi, bd, kw):
    """pure inter pictures of the synthetic quadtrees: every PU shape they produce, all 16 / 64 phases, uni / bi / weighted,
    windows over the picture border, tiles of one warp and of 8-lane groups; garbage in the row padding of the references and
    of the current picture"""
    eng = padded_engine((w, h, cfi, bd), n_slots=3)
    try:
        for seed in range(2):
            blob, st = FrameSynth(w, h, cfi=cfi, bit_depth=bd, seed=800 + 10 * seed + bd + cfi, refs=[1, 2], cur_slot=0, p_intra=0.0, coded_frac=0.0,
                                  deblock=False, sao=False, **kw).generate()
            hdr, secs = W.parse_blob(blob)
            assert len(secs[W.SEC_INTRA]) == 0 and sum(len(secs[k]) for k in (W.SEC_TU4, W.SEC_TU8, W.SEC_TU16, W.SEC_TU32)) == 0
            dpb = [smooth_frame(w, h, cfi, bd, 300 + k) for k in range(3)]
            for slot in (1, 2):
                eng.upload_slot(slot, dpb[slot])
            assert_same(eng.decode(blob), oracle_lib.execute(blob, dpb), f"seed {seed}")
    finally:
        eng.close()


def test_mc_block_with_tiles_in_two_buckets():
    """a 40x8 block cuts into a 32x8 and an 8x8 tile, which belong to different lists of the wire format: the recorder sends it
    as one block per tile (recorder.cpp b200_rec_mc).  40 is no width of the reference's tables: oracle only."""
    for geom in ((128, 64, 1, 10), (128, 64, 3, 8)):
        rects = [(x, y, 40, 8) for y in range(0, 64, 16) for x in (0, 48)]
        eng = FrameEngine(*geom, n_slots=3)
        try:
            k = [5, 7]
            for content in ("sign", "noise"):
                dpb = references(geom, content, 7)
                recs = sweep_records(rects, geom, k, content)
                blocks = block_blob(geom, recs)
                hdr, secs = W.parse_blob(blocks)
                assert len(secs[W.SEC_MC]) > len(recs)          # the luma blocks travel as tiles
                check_picture(eng, geom, recs, dpb, f"{geom} 40x8 {content}", reference_tables=False, blobs=(tile_blob(geom, recs), blocks))
        finally:
            eng.close()


def test_small_tile_region_need_not_be_bucket_ordered():
    """k_validate accepts a tile list whose <= 8x8 tiles are not grouped by (chroma, bi), so the eight-lane groups of one warp
    take different branches; every barrier of k_mc is group-local, so the picture must still be right"""
    geom = (256, 128, 1, 8)
    rects = pack(luma_shapes(), 256, 128)[0]
    eng = FrameEngine(*geom, n_slots=3)
    try:
        dpb = references(geom, "noise", 3)
        recs = sweep_records(rects, geom, [16, 32], "noise")
        tiles = tile_blob(geom, recs)
        hdr, secs = W.parse_blob(tiles)
        small = secs[W.SEC_MC][int(hdr["mc_big_count"]):]
        small[:] = small[np.random.default_rng(1).permutation(len(small))]
        key = 2 * ((small["flags"] & W.MCF_CHROMA) != 0) + ((small["flags"] & W.MCF_BI) != 0)
        quads = key[:len(key) // 4 * 4].reshape(-1, 4)                 # the four tiles of one warp
        assert (quads != quads[:, :1]).any(axis=1).sum() >= len(quads) // 2
        check_picture(eng, geom, recs, dpb, "unordered small tiles", blobs=(tiles, block_blob(geom, recs)))
    finally:
        eng.close()


@pytest.mark.late
def test_block_lists_whose_tile_counts_or_places_disagree_are_rejected():
    """A block-form list says where each block's tiles go in the lane's tile list (B200McRec.pad, per bucket; the header's
    mc_tile_count sizes the buckets).  A header that claims more tiles than its blocks cut into, or two blocks that claim the
    same place, leave places unwritten -- and on a lane that ran a picture of the same geometry before, those places still hold
    that picture's tiles, which are well-formed.  Such lists must be rejected, not executed, and leave the context usable."""
    geom = (128, 64, 1, 8)
    # bucket 0: A (16x32, two tiles, places 0-1), B (32x8, place 2), C (16x16, place 3); small tiles: D (8x8 uni), E (8x8 bi)
    rects = [(0, 0, 16, 32), (16, 0, 32, 8), (48, 0, 16, 16), (64, 0, 8, 8), (72, 0, 8, 8)]
    dpb = references(geom, "noise", 11)
    recs = sweep_records(rects, geom, [0, 0], "noise")
    recs = recs[recs["plane"] == 0]
    recs["flags"] = [0, 0, 0, 0, W.MCF_BI]
    eng = FrameEngine(*geom, n_slots=3, n_lanes=1)
    try:
        for slot in (1, 2):
            eng.upload_slot(slot, dpb[slot])
        good = block_blob(geom, recs)
        hdr, secs = W.parse_blob(good)
        assert list(hdr["mc_tile_count"]) == [4, 1, 1, 0, 0] and list(secs[W.SEC_MC]["pad"][:3, 0]) == [0, 2, 3]
        eng.upload_slot(0, dpb[0])
        first = eng.decode(good)
        assert_same(first, oracle_lib.execute(good, dpb), "good block list")
        # 1. C left out, the header still counts its tile: place 3 keeps C's tile from the picture before
        bad = block_blob(geom, recs[[0, 1, 3, 4]])
        W.header(bad)["mc_tile_count"][0] += 1
        # 2. C claims B's place: place 3 is not written
        bad2 = good.copy()
        W.parse_blob(bad2)[1][W.SEC_MC]["pad"][2] = W.parse_blob(bad2)[1][W.SEC_MC]["pad"][1]
        # 3. the same, with the header counting only the places the blocks cover: every place is written, one of them twice
        bad3 = bad2.copy()
        W.header(bad3)["mc_tile_count"][0] -= 1
        for k, blob in enumerate((bad, bad2, bad3)):
            eng.upload_slot(0, dpb[0])
            with pytest.raises(B200Error, match="rejected on the device"):
                eng.decode(blob)
            eng.upload_slot(0, dpb[0])
            assert_same(eng.decode(good), first, f"good block list after malformed list {k + 1}")
    finally:
        eng.close()
