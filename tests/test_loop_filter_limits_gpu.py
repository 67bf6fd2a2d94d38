"""GPU parity (-m gpu) of deblocking (K4) and SAO (K5) at the limits of their input space.

Grids no synthetic stream produces: SAO offsets beyond the packed 16x2 table (up to +-600), a non-zero offset_val[0] (legal
in the wire format, never written by the parser), border bits set away from the picture edge, random `edges` in the
variant that restores transquant-bypass PUs, 16x16 CTBs; deblocking grids at three densities with random no_p / no_q, on
pictures whose small steps at the block edges take all three filter decisions.  Widths and heights end inside a CTB and
inside an 8-sample strip.  The test picture enters through the residual stage as PCM blocks (b200_rec_pcm), then the blob
carries the grid; the device must equal the CPU oracle on every sample.  The DPB is caller-owned memory filled with 0x5a
beforehand, so garbage in the row padding of the filtered picture must stay unread."""
import numpy as np
import pytest

import oracle_lib
from oracle_lib import assert_same, padded_engine
from openhevc_b200 import worklist as W
from openhevc_b200.synth import smooth_frame

pytestmark = pytest.mark.gpu


def pcm_picture(geom, planes):
    """coeff / tu sections of a blob whose residual stage writes `planes` as PCM blocks (the largest that fit, up to 32x32)"""
    w, h, cfi, bd = geom
    rec = W.Recorder(geom)

    def quad(p, x, y, log2):
        pw, ph = W.plane_dims(w, h, cfi, p)
        n = 1 << log2
        if x >= pw or y >= ph:
            return
        if x + n <= pw and y + n <= ph:
            rec.pcm(p, x, y, log2, planes[p][y:y + n, x:x + n])
        else:
            for k in range(4):
                quad(p, x + (k & 1) * n // 2, y + (k >> 1) * n // 2, log2 - 1)

    for p in range(3):
        pw, ph = W.plane_dims(w, h, cfi, p)
        for y in range(0, ph, 32):
            for x in range(0, pw, 32):
                quad(p, x, y, 5)
    hdr, secs = W.parse_blob(rec.finish())
    sections = dict(coeff=secs[W.SEC_COEFF], tu={k + 2: secs[W.SEC_TU4 + k] for k in range(4)})
    assert_same(oracle_lib.execute(W.build_blob(w, h, cfi, bd, 6, 0, **sections), [[np.zeros_like(p) for p in planes]]), planes, "PCM picture")
    return sections


def noisy_planes(w, h, cfi, bd, rng, flat):
    """small-amplitude noise on a ramp: plenty of equal neighbours (edge index 0) and of both signs"""
    planes = []
    for p in range(3):
        pw, ph = W.plane_dims(w, h, cfi, p)
        yy, xx = np.mgrid[0:ph, 0:pw]
        base = ((xx * 3 + yy * 5) % (1 << bd)) if not flat else np.full((ph, pw), (1 << bd) - 3)
        v = np.clip(base + rng.integers(-3, 4, (ph, pw)), 0, (1 << bd) - 1)
        planes.append(v.astype(np.uint16))
    return planes


def random_sao_grid(w, h, bd, log2_ctb, rng, restore, big_offsets):
    ctb = 1 << log2_ctb
    cw, ch = (w + ctb - 1) // ctb, (h + ctb - 1) // ctb
    n = 3 * cw * ch
    g = np.zeros(n, W.sao_dt)
    u = rng.random(n)
    g["type"] = np.where(u < 0.15, W.SAO_NONE, np.where(u < 0.4, W.SAO_BAND, W.SAO_EDGE))
    edge = g["type"] == W.SAO_EDGE
    g["param"] = np.where(edge, rng.integers(0, 4, n), rng.integers(0, 32, n))
    maxo = 31 << max(0, bd - 10)
    off = rng.integers(-maxo, maxo + 1, (n, 5))
    off[:, 0] = 0
    if big_offsets:
        big = rng.random(n) < 0.3
        off[big] = rng.integers(-600, 601, (int(big.sum()), 5))
        off[rng.random(n) < 0.1, 0] = 5          # a non-zero entry 0: never produced by the parser, legal in the wire format
    g["offset_val"] = off
    cx = np.tile(np.arange(cw), ch); cy = np.repeat(np.arange(ch), cw)
    at_edge = (cx == 0) * 1 | (cy == 0) * 2 | (cx == cw - 1) * 4 | (cy == ch - 1) * 8     # hevc_filter.c:207-253: always set there
    g["borders"] = np.tile(at_edge, 3) | rng.integers(0, 16, n) * (rng.random(n) < 0.2)    # ... and the kernels must obey any other
    if restore:
        g["variant"] = rng.random(n) < 0.6
        g["edges"] = rng.integers(0, 256, n) * g["variant"]
    return g


SAO_CASES = [
    # w, h, cfi, bd, log2_ctb, restore, big
    (256, 128, 1, 8, 6, False, False),
    (256, 128, 1, 10, 6, True, False),
    (200, 104, 1, 10, 6, True, False),      # widths / heights that end inside a CTB and inside an 8-sample strip
    (136, 72, 1, 8, 4, True, False),        # 16x16 CTBs: 8-sample chroma CTBs
    (192, 128, 2, 10, 5, True, False),      # 4:2:2
    (192, 128, 3, 8, 6, True, False),       # 4:4:4
    (320, 192, 1, 12, 6, True, True),       # 12 bit, offsets beyond the packed table
    (72, 40, 1, 10, 5, True, True),
]


@pytest.mark.late
@pytest.mark.parametrize("w,h,cfi,bd,log2_ctb,restore,big", SAO_CASES)
def test_sao_limits(w, h, cfi, bd, log2_ctb, restore, big):
    geom = (w, h, cfi, bd)
    eng = padded_engine(geom, n_slots=1, log2_ctb_size=log2_ctb)
    try:
        for seed in range(3):
            rng = np.random.default_rng(1000 * seed + w + bd)
            grid = random_sao_grid(w, h, bd, log2_ctb, rng, restore, big)
            src = noisy_planes(w, h, cfi, bd, rng, flat=(seed == 2))
            blob = W.build_blob(w, h, cfi, bd, log2_ctb, 0, **pcm_picture(geom, src), sao=grid)
            assert_same(eng.decode(blob), oracle_lib.execute(blob, [src]), f"{geom} seed {seed}")
    finally:
        eng.close()


def random_dbk_grid(w, h, cfi, rng, density):
    L = W.DbkLayout(w, h, cfi)
    g = np.zeros(L.total, np.uint16)
    for p in range(3):
        for d in range(2):
            v = L.view(g, p, d)
            n = v.shape
            tc = rng.integers(0, 25, n); beta = rng.integers(0, 65, n)
            nop = rng.random(n) < 0.1; noq = rng.random(n) < 0.1
            e = W.DBK_PRESENT | tc | (beta << 6) | (nop.astype(np.int64) << 13) | (noq.astype(np.int64) << 14)
            v[...] = np.where(rng.random(n) < density, e, 0).astype(np.uint16)
    return g


DBK_CASES = [(256, 128, 1, 8), (256, 128, 1, 10), (200, 104, 1, 10), (136, 72, 1, 8), (192, 128, 2, 10), (192, 136, 3, 8), (320, 192, 1, 12), (520, 264, 1, 10)]


@pytest.mark.late
@pytest.mark.parametrize("w,h,cfi,bd", DBK_CASES)
def test_deblock_limits(w, h, cfi, bd):
    geom = (w, h, cfi, bd)
    eng = padded_engine(geom, n_slots=1)
    try:
        for seed in range(3):
            rng = np.random.default_rng(77 * seed + w + bd)
            grid = random_dbk_grid(w, h, cfi, rng, density=(0.9, 0.5, 0.1)[seed])
            # smooth pictures with small steps at the block edges: all three branches (none / normal / strong) are taken
            src = [np.clip(p.astype(np.int64) + rng.integers(-2, 3, p.shape) + 6 * ((np.indices(p.shape)[0] // 8 + np.indices(p.shape)[1] // 8) % 2),
                           0, (1 << bd) - 1).astype(np.uint16) for p in smooth_frame(w, h, cfi, bd, seed)]
            blob = W.build_blob(w, h, cfi, bd, 6, 0, **pcm_picture(geom, src), dbk=grid)
            want = oracle_lib.execute(blob, [src])
            assert any((want[p] != src[p]).any() for p in range(3)), "the test picture was not filtered at all"
            assert_same(eng.decode(blob), want, f"{geom} seed {seed}")
    finally:
        eng.close()


RESTORE_CASES = [(256, 128, 1, 8, 6), (256, 128, 1, 10, 6), (200, 104, 1, 10, 5), (192, 128, 2, 10, 6), (192, 128, 3, 12, 4)]


@pytest.mark.late
@pytest.mark.parametrize("w,h,cfi,bd,log2_ctb", RESTORE_CASES)
def test_sao_restore_limits(w, h, cfi, bd, log2_ctb):
    """restore_tqb_pixels (hevc_filter.c:163-193) with random `edges`, against the oracle's restatement with the reference's two
    quirks: chroma visits the PUs of half a CTB only, and above 8 bits half of each PU row comes back"""
    geom = (w, h, cfi, bd)
    eng = padded_engine(geom, n_slots=1, log2_ctb_size=log2_ctb)
    try:
        for seed in range(2):
            rng = np.random.default_rng(4000 + 10 * seed + w + bd)
            grid = random_sao_grid(w, h, bd, log2_ctb, rng, restore=True, big_offsets=False)
            pu = rng.random((h // 4, w // 4)) < (0.15 if seed else 0.6)
            pu[:, : (1 << log2_ctb) // 4] = False                         # a column of CTBs without any such PU
            src = noisy_planes(w, h, cfi, bd, rng, flat=False)
            pic = pcm_picture(geom, src)
            blob = W.build_blob(w, h, cfi, bd, log2_ctb, 0, **pic, sao=grid, tqb=(2, pu))
            hdr, secs = W.parse_blob(blob)
            assert int(hdr["flags"]) & W.FRAME_TQB and secs[W.SEC_SAO]["tqb"].any() and not secs[W.SEC_SAO]["tqb"].all()
            want = oracle_lib.execute(blob, [src])
            plain = oracle_lib.execute(W.build_blob(w, h, cfi, bd, log2_ctb, 0, **pic, sao=grid), [src])
            assert any((a != b).any() for a, b in zip(want, plain)), "the restore changed nothing"
            assert_same(eng.decode(blob), want, f"{geom} seed {seed}")
    finally:
        eng.close()
