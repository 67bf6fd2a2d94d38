"""CPU suite: the per-thread code of the CUDA kernels (openhevc_b200/csrc/k_*.cuh, compiled for the host by
tests/emul/kernel_emul.cu) against the oracle.  This is the same source the GPU runs, executed thread by thread, so the
packed 16x2 arithmetic, the tile / lane geometry and the border rules are checked without a GPU.  TEST INFRASTRUCTURE:
the product library never runs this code on the host."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_lib
from openhevc_b200 import worklist as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_SO = os.path.join(ROOT, "oracle", "_ref", "libkernel_emul.so")
EMUL_SRC = os.path.join(ROOT, "tests", "emul", "kernel_emul.cu")


@pytest.fixture(scope="module")
def emul():
    if not os.path.exists(EMUL_SO):
        if not os.path.exists("/usr/local/cuda/bin/nvcc"):
            pytest.skip("kernel emulation library not built and nvcc not available")
        subprocess.run(["make", "-C", os.path.join(ROOT, "tests", "emul")], check=True, capture_output=True)
    lib = C.CDLL(EMUL_SO)
    lib.emul_sao.restype = C.c_int
    return lib


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


CASES = [
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


@pytest.mark.parametrize("w,h,cfi,bd,log2_ctb,restore,big", CASES)
def test_sao_thread_code_equals_oracle(emul, w, h, cfi, bd, log2_ctb, restore, big):
    for seed in range(3):
        rng = np.random.default_rng(1000 * seed + w + bd)
        grid = random_sao_grid(w, h, bd, log2_ctb, rng, restore, big)
        src = noisy_planes(w, h, cfi, bd, rng, flat=(seed == 2))
        blob = W.build_blob(w, h, cfi, bd, log2_ctb, 0, sao=grid)
        want = oracle_lib.execute(blob, [src])
        dt = np.uint16 if bd > 8 else np.uint8
        B = np.dtype(dt).itemsize
        pitches, s_bufs, d_bufs = [], [], []
        for p in range(3):
            pw, ph = W.plane_dims(w, h, cfi, p)
            pitch = (pw * B + 255) // 256 * 256
            sb = np.full((ph, pitch // B), 0x5a5a if bd > 8 else 0x5a, dt)     # garbage in the row padding, as on the device
            sb[:, :pw] = src[p]
            db = np.zeros_like(sb)
            pitches.append(pitch); s_bufs.append(sb); d_bufs.append(db)
        sp = (C.c_void_p * 3)(*[b.ctypes.data for b in s_bufs])
        dp = (C.c_void_p * 3)(*[b.ctypes.data for b in d_bufs])
        rc = emul.emul_sao(grid.ctypes.data_as(C.c_void_p), sp, dp, (C.c_int * 3)(*pitches), w, h, cfi, bd, log2_ctb, None)
        assert rc == 0
        for p in range(3):
            pw, ph = W.plane_dims(w, h, cfi, p)
            got = d_bufs[p][:, :pw].astype(np.uint16)
            bad = np.argwhere(got != want[p])
            assert len(bad) == 0, (f"seed {seed} plane {p}: {len(bad)} samples differ, first at (y,x)={tuple(bad[0])} "
                                   f"got {got[tuple(bad[0])]} want {want[p][tuple(bad[0])]}")


def run_emul_planes(fn, planes, w, h, cfi, bd, *args):
    """copies the planes into pitched native-type buffers (garbage in the padding), runs fn in place, returns uint16 planes"""
    dt = np.uint16 if bd > 8 else np.uint8
    B = np.dtype(dt).itemsize
    pitches, bufs = [], []
    for p in range(3):
        pw, ph = W.plane_dims(w, h, cfi, p)
        pitch = (pw * B + 255) // 256 * 256
        b = np.full((ph, pitch // B), 0x5a5a if bd > 8 else 0x5a, dt)
        b[:, :pw] = planes[p]
        pitches.append(pitch); bufs.append(b)
    ptrs = (C.c_void_p * 3)(*[b.ctypes.data for b in bufs])
    assert fn(*args, ptrs, (C.c_int * 3)(*pitches), w, h, cfi, bd) == 0
    return [bufs[p][:, :W.plane_dims(w, h, cfi, p)[0]].astype(np.uint16) for p in range(3)]


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


@pytest.mark.parametrize("w,h,cfi,bd", DBK_CASES)
def test_deblock_thread_code_equals_oracle(emul, w, h, cfi, bd):
    from openhevc_b200.synth import smooth_frame
    for seed in range(3):
        rng = np.random.default_rng(77 * seed + w + bd)
        grid = random_dbk_grid(w, h, cfi, rng, density=(0.9, 0.5, 0.1)[seed])
        # smooth pictures with small steps at the block edges: all three branches (none / normal / strong) are taken
        src = [np.clip(p.astype(np.int64) + rng.integers(-2, 3, p.shape) + 6 * ((np.indices(p.shape)[0] // 8 + np.indices(p.shape)[1] // 8) % 2),
                       0, (1 << bd) - 1).astype(np.uint16) for p in smooth_frame(w, h, cfi, bd, seed)]
        blob = W.build_blob(w, h, cfi, bd, 6, 0, dbk=grid)
        want = oracle_lib.execute(blob, [src])
        assert any((want[p] != src[p]).any() for p in range(3)), "the test picture was not filtered at all"
        got = run_emul_planes(emul.emul_deblock, src, w, h, cfi, bd, grid.ctypes.data_as(C.c_void_p))
        for p in range(3):
            bad = np.argwhere(got[p] != want[p])
            assert len(bad) == 0, (f"seed {seed} plane {p}: {len(bad)} samples differ, first at (y,x)={tuple(bad[0])} "
                                   f"got {got[p][tuple(bad[0])]} want {want[p][tuple(bad[0])]}")


@pytest.mark.parametrize("cfi,bd,p_intra,split", [(1, 8, 0.12, 1.0), (1, 10, 0.45, 1.0), (2, 10, 0.3, 2.0), (3, 8, 0.6, 0.5), (1, 12, 0.8, 2.0)])
def test_constrained_intra_rules_equal_oracle(emul, cfi, bd, p_intra, split):
    """cip_flags() / cip_substitute() (k_intra_cip.cuh, run by lane 0 of k_intra) against the oracle's restatement of
    hevcpred_template.c:116-249, for every intra TU of synthetic inter pictures"""
    from openhevc_b200.synth import FrameSynth, smooth_frame
    w, h = 320, 192
    blob, st = FrameSynth(w, h, cfi=cfi, bit_depth=bd, seed=500 + cfi + bd, refs=[1], cur_slot=0, cip=True, p_intra=p_intra, split_bias=split).generate()
    hdr, secs = W.parse_blob(blob)
    assert int(hdr["flags"]) & W.FRAME_CIP
    rng = np.random.default_rng(9)
    planes = [rng.integers(0, 1 << bd, W.plane_dims(w, h, cfi, p)[::-1]).astype(np.uint16) for p in range(3)]     # noise: any mix-up of two samples shows
    cip_words = np.ascontiguousarray(blob[int(hdr["cip"]["off"]):int(hdr["cip"]["off"]) + 4 * int(hdr["cip"]["count"])]).view("<u4")
    o = oracle_lib.lib()
    pp = (C.c_void_p * 3)(*[p.ctypes.data for p in planes])
    recs = secs[W.SEC_INTRA]
    changed = 0
    for i in range(len(recs)):
        ot, ol, of = (C.c_int * 65)(), (C.c_int * 65)(), C.c_int()
        et, el, ef = (C.c_int * 65)(), (C.c_int * 65)(), C.c_int()
        assert o.orc_debug_cip_refs(np.ascontiguousarray(blob).ctypes.data_as(C.c_void_p), pp, i, ot, ol, C.byref(of)) == 0
        r = recs[i:i + 1]
        pl = int(r["plane"][0])
        assert emul.emul_cip_refs(cip_words.ctypes.data_as(C.c_void_p), r.ctypes.data_as(C.c_void_p), planes[pl].ctypes.data_as(C.c_void_p),
                                  planes[pl].shape[1], w, h, cfi, bd, et, el, C.byref(ef)) == 0
        n2 = 2 << int(r["log2"][0])
        assert of.value == ef.value, f"record {i}: flags {ef.value:#x} != oracle {of.value:#x}"
        assert list(ot)[:n2 + 1] == list(et)[:n2 + 1] and list(ol)[:n2 + 1] == list(el)[:n2 + 1], f"record {i}: reference arrays differ"
        changed += of.value != (int(r["flags"][0]) & 31)
    assert changed > 10, "the constrained-intra rule never removed a candidate: the test picture does not exercise it"


MC_CASES = [  # w, h, cfi, bd, kw
    (256, 128, 1, 8, {}),
    (256, 128, 1, 10, dict(weighted=True)),
    (320, 192, 1, 10, dict(max_mv=150)),               # windows far outside the picture: clamped loads
    (192, 128, 2, 10, {}),
    (192, 128, 3, 8, dict(weighted=True)),
    (320, 192, 1, 12, dict(split_bias=2.5)),           # many small blocks
    (256, 192, 1, 10, dict(split_bias=0.3, bi_frac=0.2)),
]


@pytest.mark.parametrize("w,h,cfi,bd,kw", MC_CASES)
def test_mc_phase_code_equals_oracle(emul, w, h, cfi, bd, kw):
    """K1 (k_mc in kernels.cu, run by the warp-lockstep emulation with its group-local barriers: tests/emul/mc_emul.cpp) against
    the oracle on pure inter pictures (every PU shape of the synthetic quadtrees, all 16 / 64 phases, uni / bi / weighted, luma
    and chroma, windows hanging over the picture border, tiles of one warp and of 8-lane groups)"""
    from openhevc_b200.synth import FrameSynth, smooth_frame
    for seed in range(2):
        blob, st = FrameSynth(w, h, cfi=cfi, bit_depth=bd, seed=800 + 10 * seed + bd + cfi, refs=[1, 2], cur_slot=0, p_intra=0.0, coded_frac=0.0,
                              deblock=False, sao=False, **kw).generate()
        hdr, secs = W.parse_blob(blob)
        assert len(secs[W.SEC_INTRA]) == 0 and sum(len(secs[k]) for k in (W.SEC_TU4, W.SEC_TU8, W.SEC_TU16, W.SEC_TU32)) == 0
        dpb = [smooth_frame(w, h, cfi, bd, 300 + k) for k in range(3)]
        want = oracle_lib.execute(blob, dpb)
        dt = np.uint16 if bd > 8 else np.uint8
        B = np.dtype(dt).itemsize
        pitches, bufs = [], []
        for slot in range(3):
            for p in range(3):
                pw, ph = W.plane_dims(w, h, cfi, p)
                pitch = (pw * B + 255) // 256 * 256
                b = np.full((ph, pitch // B), 0x5a5a if bd > 8 else 0x5a, dt)
                b[:, :pw] = dpb[slot][p] if slot else 0
                bufs.append(b)
                if slot == 0:
                    pitches.append(pitch)
        ptrs = (C.c_void_p * 9)(*[b.ctypes.data for b in bufs])
        cur = (C.c_void_p * 3)(*[b.ctypes.data for b in bufs[:3]])
        mc = np.ascontiguousarray(secs[W.SEC_MC])
        ref_slot = np.ascontiguousarray(hdr["ref_slot"])
        rc = emul.emul_mc(mc.ctypes.data_as(C.c_void_p), len(mc), int(hdr["mc_big_count"]), cur, ptrs, 3, (C.c_int * 3)(*pitches), w, h, cfi, bd,
                          ref_slot.ctypes.data_as(C.c_void_p))
        assert rc == 0
        for p in range(3):
            pw, ph = W.plane_dims(w, h, cfi, p)
            got = bufs[p][:, :pw].astype(np.uint16)
            bad = np.argwhere(got != want[p])
            assert len(bad) == 0, (f"seed {seed} plane {p}: {len(bad)} samples differ, first at (y,x)={tuple(bad[0])} "
                                   f"got {got[tuple(bad[0])]} want {want[p][tuple(bad[0])]}")


@pytest.mark.parametrize("w,h,cfi,bd,log2_ctb", [(256, 128, 1, 8, 6), (256, 128, 1, 10, 6), (200, 104, 1, 10, 5), (192, 128, 2, 10, 6), (192, 128, 3, 12, 4)])
def test_sao_restore_of_bypass_pus_equals_oracle(emul, w, h, cfi, bd, log2_ctb):
    """restore_tqb_pixels (hevc_filter.c:163-193) as the SAO kernel does it (sao_restore_row) against the oracle's restatement,
    with the reference's two quirks: chroma visits the PUs of half a CTB only, and above 8 bits half of each PU row comes back"""
    for seed in range(2):
        rng = np.random.default_rng(4000 + 10 * seed + w + bd)
        grid = random_sao_grid(w, h, bd, log2_ctb, rng, restore=True, big_offsets=False)
        pu = rng.random((h // 4, w // 4)) < (0.15 if seed else 0.6)
        pu[:, : (1 << log2_ctb) // 4] = False                         # a column of CTBs without any such PU
        src = noisy_planes(w, h, cfi, bd, rng, flat=False)
        blob = W.build_blob(w, h, cfi, bd, log2_ctb, 0, sao=grid, tqb=(2, pu))
        hdr, secs = W.parse_blob(blob)
        assert int(hdr["flags"]) & W.FRAME_TQB and secs[W.SEC_SAO]["tqb"].any() and not secs[W.SEC_SAO]["tqb"].all()
        want = oracle_lib.execute(blob, [src])
        plain = oracle_lib.execute(W.build_blob(w, h, cfi, bd, log2_ctb, 0, sao=grid), [src])
        assert any((a != b).any() for a, b in zip(want, plain)), "the restore changed nothing"
        tqb_words = np.ascontiguousarray(blob[int(hdr["tqb"]["off"]):int(hdr["tqb"]["off"]) + 4 * int(hdr["tqb"]["count"])]).view("<u4")
        g2 = np.ascontiguousarray(secs[W.SEC_SAO])
        dt = np.uint16 if bd > 8 else np.uint8
        B = np.dtype(dt).itemsize
        pitches, s_bufs, d_bufs = [], [], []
        for p in range(3):
            pw, ph = W.plane_dims(w, h, cfi, p)
            pitch = (pw * B + 255) // 256 * 256
            sb = np.full((ph, pitch // B), 0x5a5a if bd > 8 else 0x5a, dt)
            sb[:, :pw] = src[p]
            pitches.append(pitch); s_bufs.append(sb); d_bufs.append(np.zeros_like(sb))
        sp = (C.c_void_p * 3)(*[b.ctypes.data for b in s_bufs])
        dp = (C.c_void_p * 3)(*[b.ctypes.data for b in d_bufs])
        assert emul.emul_sao(g2.ctypes.data_as(C.c_void_p), sp, dp, (C.c_int * 3)(*pitches), w, h, cfi, bd, log2_ctb, tqb_words.ctypes.data_as(C.c_void_p)) == 0
        for p in range(3):
            pw, ph = W.plane_dims(w, h, cfi, p)
            got = d_bufs[p][:, :pw].astype(np.uint16)
            bad = np.argwhere(got != want[p])
            assert len(bad) == 0, f"seed {seed} plane {p}: {len(bad)} samples differ, first at (y,x)={tuple(bad[0])} got {got[tuple(bad[0])]} want {want[p][tuple(bad[0])]}"
