"""GPU parity (-m gpu): the CUDA path, called through the C ABI (libb200hevc.so), against the CPU oracle
on the same seeded work lists.  Bit-exact or fail."""
import os

import numpy as np
import pytest

import oracle_lib
from openhevc_b200 import FrameEngine, B200Error
from openhevc_b200 import worklist as W
from openhevc_b200.synth import FrameSynth, smooth_frame

pytestmark = pytest.mark.gpu


def run_sequence(w, h, cfi, bd, seeds, n_slots=4, check_order=True, **kw):
    """I picture -> slot 0, then pictures predicted from everything decoded so far; every picture compared."""
    eng = FrameEngine(w, h, cfi, bd, n_slots=n_slots)
    dpb = [[np.zeros_like(p) for p in smooth_frame(w, h, cfi, bd, 0)] for _ in range(n_slots)]
    try:
        for k, seed in enumerate(seeds):
            refs = list(range(k))
            blob, st = FrameSynth(w, h, cfi, bd, seed=seed, refs=refs, cur_slot=k, poc=k, **kw).generate()
            if check_order:
                oracle_lib.check_decode_order(blob)
            got = eng.decode(blob)
            want = oracle_lib.execute(blob, dpb)
            for p in range(3):
                bad = np.argwhere(got[p] != want[p])
                assert len(bad) == 0, f"picture {k} plane {p}: {len(bad)} samples differ, first at (y,x)={tuple(bad[0])} got {got[p][tuple(bad[0])]} want {want[p][tuple(bad[0])]}"
            dpb[k] = [p.copy() for p in want]
    finally:
        eng.close()


@pytest.mark.parametrize("w,h,cfi,bd", [(256, 128, 1, 8), (256, 128, 1, 10), (192, 128, 2, 10), (192, 128, 3, 8), (320, 192, 1, 12)])
def test_sequence_all_stages(w, h, cfi, bd):
    run_sequence(w, h, cfi, bd, seeds=[11, 12, 13], exotic=0.04)


def test_weighted_prediction_and_sao_restore():
    run_sequence(256, 192, 1, 10, seeds=[21, 22, 23], weighted=True, sao_restore=True)


def test_constrained_intra_pred():
    """pps->constrained_intra_pred_flag: inter pictures whose intra TUs may only use intra-coded neighbours; the device
    applies hevcpred_template.c:116-249 itself from the picture's intra bitmap (B200BlobHeader.cip)"""
    run_sequence(256, 192, 1, 10, seeds=[61, 62, 63], cip=True, p_intra=0.4)
    run_sequence(256, 128, 1, 8, seeds=[64, 65], cip=True, p_intra=0.15, split_bias=2.0)
    run_sequence(192, 128, 2, 10, seeds=[66, 67], cip=True, p_intra=0.5)
    run_sequence(192, 128, 3, 8, seeds=[68, 69], cip=True, p_intra=0.7, split_bias=0.4)


@pytest.mark.late
def test_sao_restore_of_bypass_pus():
    """transquant-bypass / PCM-without-loop-filter PUs get their deblocked samples back after SAO (restore_tqb_pixels,
    hevc_filter.c:163-193, with the reference's two quirks): blob with a TQB bitmap, SAO kernel vs oracle"""
    for (w, h, cfi, bd) in ((256, 128, 1, 8), (256, 128, 1, 10), (192, 128, 2, 10), (192, 128, 3, 8)):
        eng = FrameEngine(w, h, cfi, bd, n_slots=2)
        try:
            for seed in (71, 72):
                syn = FrameSynth(w, h, cfi, bd, seed=seed + bd, cur_slot=0, sao_restore=True)
                blob, _ = syn.generate()
                hdr, secs = W.parse_blob(blob)
                rng = np.random.default_rng(seed)
                pu = rng.random((h // 4, w // 4)) < 0.3
                pu[:, :16] = False
                blob2 = W.build_blob(w, h, cfi, bd, 6, 0, coeff=secs[W.SEC_COEFF], tu={k + 2: secs[W.SEC_TU4 + k] for k in range(4)}, intra=secs[W.SEC_INTRA],
                                     dbk=secs[W.SEC_DBK], sao=secs[W.SEC_SAO], tqb=(2, pu))
                got = eng.decode(blob2)
                dpb = [[np.zeros_like(p) for p in smooth_frame(w, h, cfi, bd, 0)] for _ in range(2)]
                want = oracle_lib.execute(blob2, dpb)
                plain = oracle_lib.execute(blob, dpb)
                assert any((a != b).any() for a, b in zip(want, plain)), "the restore changed nothing"
                for p in range(3):
                    assert (got[p] == want[p]).all(), f"{w}x{h} cfi {cfi} bd {bd} seed {seed} plane {p}"
        finally:
            eng.close()


def test_intra_only_small_blocks():
    """all-intra with a deep quadtree: the TU-granular wavefront and every predictor / smoothing branch"""
    run_sequence(256, 256, 1, 8, seeds=[31], split_bias=2.0)
    run_sequence(256, 256, 1, 10, seeds=[32], split_bias=0.3)


def test_stages_individually():
    """deblock off / SAO off / no residual: each stage alone must still match"""
    run_sequence(256, 128, 1, 8, seeds=[41, 42], deblock=False, sao=False)
    run_sequence(256, 128, 1, 8, seeds=[43, 44], deblock=True, sao=False)
    run_sequence(256, 128, 1, 10, seeds=[45, 46], deblock=False, sao=True, coded_frac=0.0)


def test_far_out_of_picture_motion():
    """motion vectors pointing far outside: emulated_edge_mc == clamped addressing (videodsp_template.c:26-100)"""
    run_sequence(128, 128, 1, 8, seeds=[51, 52], max_mv=200)


def test_config_c1_832x480_intra():
    """BASELINE config 1 geometry: 832x480 8-bit, I pictures only"""
    run_sequence(832, 480, 1, 8, seeds=[61])


def test_config_c2_1080p_random_access():
    run_sequence(1920, 1080, 1, 8, seeds=[71, 72], n_slots=3)


def test_config_c3_4k_main10_b_picture():
    """BASELINE config 3 at full size: one bi-predicted 3840x2160 Main10 picture, all stages, bit-exact"""
    w, h, cfi, bd = 3840, 2160, 1, 10
    eng = FrameEngine(w, h, cfi, bd, n_slots=3)
    try:
        dpb = [smooth_frame(w, h, cfi, bd, 80 + k) for k in range(3)]
        for s in (1, 2):
            eng.upload_slot(s, dpb[s])
        blob, st = FrameSynth(w, h, cfi, bd, seed=81, refs=[1, 2], cur_slot=0).generate()
        got = eng.decode(blob)
        want = oracle_lib.execute(blob, dpb)
        for p in range(3):
            assert (got[p] == want[p]).all()
        # size-independent properties: determinism of the whole pipeline and independence from arena / slot reuse
        again = eng.decode(blob)
        for p in range(3):
            assert (again[p] == got[p]).all()
    finally:
        eng.close()


def test_config_c5_8k_422_main10():
    """BASELINE config 5 geometry: 7680x4320 4:2:2 10-bit (RExt chroma format), inter picture with deblock + SAO"""
    w, h, cfi, bd = 7680, 4320, 2, 10
    eng = FrameEngine(w, h, cfi, bd, n_slots=2)
    try:
        dpb = [smooth_frame(w, h, cfi, bd, 90 + k) for k in range(2)]
        eng.upload_slot(1, dpb[1])
        blob, st = FrameSynth(w, h, cfi, bd, seed=91, refs=[1], cur_slot=0, split_bias=0.4, coded_frac=0.3).generate()
        got = eng.decode(blob)
        want = oracle_lib.execute(blob, dpb)
        for p in range(3):
            assert (got[p] == want[p]).all()
    finally:
        eng.close()


def test_pcm_and_exotic_transform_paths():
    """pcm CUs (put_pcm), transform-skip, rdpcm, transquant-bypass TUs in one sequence"""
    run_sequence(256, 128, 1, 8, seeds=[95, 96], exotic=0.3)
    run_sequence(192, 128, 2, 10, seeds=[97, 98], exotic=0.3)


def test_malformed_blobs_are_rejected_not_executed():
    eng = FrameEngine(128, 64, 1, 8, n_slots=2)
    try:
        blob, _ = FrameSynth(128, 64, 1, 8, seed=5, cur_slot=0).generate()
        bad = blob.copy(); bad[0] ^= 0xFF
        with pytest.raises(B200Error):
            eng.submit(bad)
        bad = blob.copy(); bad[23] = 9                         # cur_slot out of range
        with pytest.raises(B200Error):
            eng.submit(bad)
        with pytest.raises(B200Error):
            eng.submit(blob[:1000])
        bad = blob.copy(); bad[:256].view(W.header_dt)["reserved_section"]["count"] = 1     # reserved header field in use
        with pytest.raises(B200Error, match="reserved"):
            eng.submit(bad)
        eng.decode(blob)                                        # context still usable
        # a record that points outside the picture / the coefficient pool / the reference table: caught by the
        # validation kernel in front of the picture's kernels (k_validate); the picture is not executed
        hdr, secs = W.parse_blob(blob)
        for sec, field, value in ((W.SEC_TU8, "x", 124), (W.SEC_TU4, "coeff_off", 0x7fffffff), (W.SEC_INTRA, "mode", 77), (W.SEC_INTRA, "y", 62)):
            bad = blob.copy()
            _, bsecs = W.parse_blob(bad)
            if len(bsecs[sec]) == 0:
                continue
            bsecs[sec][field][len(bsecs[sec]) // 2] = value
            before = eng.decode(blob)
            with pytest.raises(B200Error, match="rejected on the device"):
                eng.decode(bad)
            after = eng.decode(blob)                            # context still usable, and the good picture unchanged
            assert all((a == b).all() for a, b in zip(before, after))
    finally:
        eng.close()


@pytest.mark.late
def test_malformed_inter_records_are_rejected_on_the_device():
    w, h = 128, 64
    eng = FrameEngine(w, h, 1, 8, n_slots=3)
    try:
        eng.upload_slot(1, smooth_frame(w, h, 1, 8, 3))
        blob, _ = FrameSynth(w, h, 1, 8, seed=6, refs=[1], cur_slot=0).generate()
        good = eng.decode(blob)
        for field, value in (("ref0", 9), ("w", 40), ("x", 127), ("frac0", 0x7f)):
            bad = blob.copy()
            _, bsecs = W.parse_blob(bad)
            bsecs[W.SEC_MC][field][3] = value
            with pytest.raises(B200Error, match="rejected on the device"):
                eng.decode(bad)
        again = eng.decode(blob)
        assert all((a == b).all() for a, b in zip(good, again))
    finally:
        eng.close()


@pytest.mark.late
@pytest.mark.parametrize("cfi,bd", [(1, 8), (2, 10)])
def test_grey_reference_fill(cfi, bd):
    """generate_missing_ref (hevc_refs.c:538): a reference the stream lost is a picture of 1 << (bit_depth - 1); the
    drop-in fills the slot on the device (b200_slot_fill) and the next picture predicts from it"""
    w, h, grey = 192, 128, 1 << (bd - 1)
    eng = FrameEngine(w, h, cfi, bd, n_slots=3)
    try:
        eng.upload_slot(1, smooth_frame(w, h, cfi, bd, 5))       # something else first: the fill must overwrite every sample
        eng.fill_slot(1, grey)
        got = eng.readback(1)
        dpb = [[np.zeros_like(p) for p in got] for _ in range(3)]
        for p in range(3):
            assert got[p].shape == eng.plane_shape(p) and (got[p] == grey).all()
            dpb[1][p][:] = grey
        blob, _ = FrameSynth(w, h, cfi, bd, seed=41, refs=[1], cur_slot=0, poc=1).generate()
        pic, want = eng.decode(blob), oracle_lib.execute(blob, dpb)
        for p in range(3):
            assert np.array_equal(pic[p], want[p])
    finally:
        eng.close()


@pytest.mark.late
def test_empty_work_list_and_smallest_pictures():
    """a work list without a single record leaves the picture as it was (and says so through the same path as any other); the
    smallest geometry the context accepts (16x16) and sizes that are no multiple of any CTB size; smaller ones are refused"""
    w, h, cfi, bd = 64, 48, 1, 10
    eng = FrameEngine(w, h, cfi, bd, n_slots=2)
    try:
        before = smooth_frame(w, h, cfi, bd, 9)
        eng.upload_slot(0, before)
        blob = W.build_blob(w, h, cfi, bd, 6, 0)
        got = eng.decode(blob)
        want = oracle_lib.execute(blob, [[p.copy() for p in before], [np.zeros_like(p) for p in before]])
        for p in range(3):
            assert np.array_equal(got[p], want[p]) and np.array_equal(got[p], before[p])
    finally:
        eng.close()
    for (w, h, cfi, bd) in ((16, 16, 1, 8), (16, 16, 3, 10), (24, 40, 2, 10), (72, 24, 1, 12)):
        run_sequence(w, h, cfi, bd, seeds=[5, 6, 7], exotic=0.1)
    with pytest.raises(B200Error):
        FrameEngine(8, 8, 1, 8)
    with pytest.raises(B200Error):
        FrameEngine(20, 16, 1, 8)                         # not a multiple of the minimum coding block


def ccp_blob(w, h, bd, seed, corrupt=False):
    """a 4:4:4 picture of cross-component-prediction blocks built through the recorder API the way the shim does it
    (hevcdsp_init_b200.c: rec_cross_component): luma block, the same luma block parked, the chroma block's own residual parked
    (or none), and the record that combines them -- half of the blocks intra predicted (result parked for the intra stage)"""
    import ctypes as C
    from openhevc_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(seed)
    cfg = _lib.B200Config(0, w, h, 3, bd, 6, 2, 2, 0, None, 0)
    r = C.c_void_p()
    assert lib.b200_rec_create(C.byref(cfg), C.byref(r)) == 0
    assert lib.b200_rec_begin(r, 0, 0) == 0
    for y in range(0, h, 16):
        for x in range(0, w, 16):
            log2 = int(rng.choice([2, 3, 4]))
            n = 1 << log2
            intra = bool(rng.integers(2))

            def coeffs():
                c = np.zeros((n, n), np.int16)
                k = int(rng.integers(1, 6))
                c[rng.integers(0, min(n, 4), k), rng.integers(0, min(n, 4), k)] = rng.integers(-300, 300, k)
                return np.ascontiguousarray(c)
            cy = coeffs()
            if intra:
                assert lib.b200_rec_intra(r, 0, x, y, log2, 1, 0, 0, 0) == 0
            assert lib.b200_rec_tu(r, 0, x, y, log2, W.TU_IDCT, 0, n, cy.ctypes.data, -1) == 0
            off_y = C.c_uint32()
            assert lib.b200_rec_tu_parked(r, 0, x, y, log2, W.TU_IDCT, 0, n, cy.ctypes.data, C.byref(off_y)) == 0
            for plane in (1, 2):
                if intra:
                    assert lib.b200_rec_intra(r, plane, x, y, log2, 1, 0, 0, 0) == 0
                has_c = bool(rng.integers(2))
                off_c = C.c_uint32()
                if has_c:
                    cc = coeffs()
                    assert lib.b200_rec_tu_parked(r, plane, x, y, log2, W.TU_IDCT, 0, n, cc.ctypes.data, C.byref(off_c)) == 0
                scale = int(rng.choice([1, 2, 4, 8])) * int(rng.choice([-1, 1]))
                assert lib.b200_rec_ccp(r, plane, x, y, log2, scale, off_y.value, int(has_c), off_c.value) == 0
    blob_p, nbytes = C.c_void_p(), C.c_uint64()
    assert lib.b200_rec_finish(r, C.byref(blob_p), C.byref(nbytes)) == 0
    blob = np.ctypeslib.as_array(C.cast(blob_p, C.POINTER(C.c_uint8)), (nbytes.value,)).copy()
    lib.b200_rec_destroy(r)
    if corrupt:
        hdr, _ = W.parse_blob(blob)
        off = int(hdr["ccp"]["off"])
        blob[off + 8:off + 12] = np.frombuffer(np.uint32(0x7fffff00).tobytes(), np.uint8)      # off_y of the first record far outside the pool
    return blob


@pytest.mark.late
@pytest.mark.parametrize("bd", [8, 10])
def test_cross_component_prediction(bd):
    """range-extension cross-component prediction (hevc.c:1295-1360): chroma residual += (res_scale_val * luma residual) >> 3"""
    w, h = 96, 64
    eng = FrameEngine(w, h, 3, bd, n_slots=2)
    try:
        before = smooth_frame(w, h, 3, bd, 4)
        for seed in (1, 2):
            eng.upload_slot(0, before)
            blob = ccp_blob(w, h, bd, seed)
            got = eng.decode(blob)
            want = oracle_lib.execute(blob, [[p.copy() for p in before], [np.zeros_like(p) for p in before]])
            for p in range(3):
                assert np.array_equal(got[p], want[p]), f"plane {p} differs (seed {seed})"
        with pytest.raises(B200Error, match="rejected on the device"):
            eng.decode(ccp_blob(w, h, bd, 3, corrupt=True))
        eng.upload_slot(0, before)
        blob = ccp_blob(w, h, bd, 1)
        again = eng.decode(blob)
        want = oracle_lib.execute(blob, [[p.copy() for p in before], [np.zeros_like(p) for p in before]])
        assert all(np.array_equal(a, b) for a, b in zip(again, want))
    finally:
        eng.close()


def test_cyclic_intra_dependencies_time_out_instead_of_hanging():
    """a work list whose intra TUs wait on each other (cannot come from a real decode order) must not hang the device"""
    w, h = 128, 64
    intra = np.zeros(2, W.intra_dt)
    # A at (0,8) claims its up-right block B=(8,0) is available, B claims its bottom-left block A is available
    intra[0] = (0, 8, 0, 3, 1, W.INF_UP | W.INF_UP_RIGHT, 8, 0, (0, 0), W.NO_RESID)
    intra[1] = (8, 0, 0, 3, 1, W.INF_LEFT | W.INF_BOTTOM_LEFT, 0, 8, (0, 0), W.NO_RESID)
    blob = W.build_blob(w, h, 1, 8, 6, 0, intra=intra)
    eng = FrameEngine(w, h, 1, 8, n_slots=2)
    try:
        with pytest.raises(B200Error, match="decode order"):
            eng.decode(blob)
    finally:
        eng.close()


@pytest.mark.parametrize("lanes", [1, 4])
def test_out_of_order_lanes_keep_slot_hazards(lanes):
    """18 pictures submitted back to back (no host sync) on `lanes` compute lanes, 6 DPB slots recycled: every picture
    must see its references complete (RAW), must not overwrite a slot that an earlier picture or a read-back still
    reads (WAR), and slot rewrites stay ordered (WAW).  Hierarchical references make neighbours independent."""
    w, h, cfi, bd, n_slots = 832, 480, 1, 10, 6
    eng = FrameEngine(w, h, cfi, bd, n_slots=n_slots, n_arenas=8, n_lanes=lanes)
    dpb = [[np.zeros_like(p) for p in smooth_frame(w, h, cfi, bd, 0)] for _ in range(n_slots)]
    rng = np.random.default_rng(7)
    try:
        outs, wants, recent = [], [], []
        for k in range(18):
            cur = k % n_slots
            cand = [s for s in recent if s != cur]
            refs = [] if k % 9 == 0 else sorted(set(int(x) for x in rng.choice(cand, size=min(2, len(cand)), replace=False)))
            blob, _ = FrameSynth(w, h, cfi, bd, seed=700 + k, refs=refs, cur_slot=cur, poc=k, p_intra=0.1 if refs else 1.0).generate()
            eng.submit(blob)
            outs.append(eng.readback(cur, eng.new_host_frame(pinned=True), sync=False))
            want = oracle_lib.execute(blob, dpb)
            dpb[cur] = [p.copy() for p in want]
            wants.append(want)
            recent = ([cur] + [s for s in recent if s != cur])[:4]
        eng.sync()
        for k, (got, want) in enumerate(zip(outs, wants)):
            for p in range(3):
                assert np.array_equal(got[p], want[p]), f"picture {k} plane {p} differs ({lanes} lanes)"
    finally:
        eng.close()


@pytest.mark.gpu
def test_frame_parallel_over_two_gpus_equals_sequential_decode():
    """tools/verify_multi_gpu.py under torchrun, 2 ranks: the product schedule (ownership by intra period, the one anchor per
    period sent to the next GPU with NCCL send / recv inside the engine's slot-hazard protocol, 8 lanes) -- every picture of
    every rank against the sequential decode by the CPU oracle.  Needs two visible GPUs (the driver's multi-GPU tier)."""
    import subprocess
    import sys
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU visible")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", "29517",
                        os.path.join(root, "tools", "verify_multi_gpu.py"), "--gops", "8"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and '"verify_multi_gpu": "ok"' in r.stdout, (r.stdout[-2000:], r.stderr[-2000:])
