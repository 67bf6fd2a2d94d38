"""The drop-in itself (-m gpu): the reference's own call sequence -- table slots of HEVCDSPContext / HEVCPredContext /
VideoDSPContext invoked exactly as hevc.c / hevc_cabac.c / hevc_filter.c invoke them (oracle/replay_ref.c) -- once with the
reference's C functions installed, once with ff_hevcdsp_init_b200 / ff_hevcpred_init_b200 / ff_videodsp_init_b200
(libb200hevc_shim.so: pointer -> record -> GPU -> b200_frame_readback).  Pictures must be identical."""
import os

import numpy as np
import pytest

import oracle_lib
from openhevc_b200.synth import FrameSynth, smooth_frame

pytestmark = pytest.mark.gpu


REFERENCE_MD5 = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dropin_reference.md5")
CASES = [
    (256, 128, 1, 8, [], {}),
    (256, 128, 1, 10, [1, 2], dict(weighted=True)),
    (320, 192, 1, 8, [1, 2], dict(max_mv=150, exotic=0.3)),
    (192, 128, 2, 10, [2], {}),
    (192, 128, 3, 8, [1, 2], dict(sao_restore=True)),
    (832, 480, 1, 8, [], {}),
    (256, 128, 1, 10, [1, 2], dict(cip=True, p_intra=0.4)),       # constrained_intra_pred: the shim hands the PU types over at frame end
    (192, 128, 2, 8, [1], dict(cip=True, p_intra=0.6)),
]


def case(w, h, cfi, bd, refs, kw):
    blob, _ = FrameSynth(w, h, cfi, bd, seed=300 + w + bd + cfi, refs=refs, cur_slot=0, **kw).generate()
    return blob, [smooth_frame(w, h, cfi, bd, 30 + k) for k in range(3)]


@pytest.mark.parametrize("w,h,cfi,bd,refs,kw", CASES)
def test_tables_through_shim_equal_reference_tables(w, h, cfi, bd, refs, kw):
    blob, dpb = case(w, h, cfi, bd, refs, kw)
    if oracle_lib.ref_lib() is None or not os.path.exists(oracle_lib.SHIM_SO):
        # without the reference build: the CUDA path against MD5s of the reference tables' picture (golden/make_golden.py)
        from openhevc_b200 import FrameEngine
        from openhevc_b200 import worklist as W
        want = open(REFERENCE_MD5).read().splitlines()[CASES.index((w, h, cfi, bd, refs, kw))]
        eng = FrameEngine(w, h, cfi, bd, n_slots=3)
        try:
            for s in range(3):
                eng.upload_slot(s, dpb[s])
            got = oracle_lib.md5_line(0, W.parse_blob(blob)[0], eng.decode(blob))
        finally:
            eng.close()
        assert got == want
        return
    want = oracle_lib.ref_execute(blob, dpb)
    got = oracle_lib.ref_execute_b200(blob, dpb)
    for p in range(3):
        bad = np.argwhere(got[p] != want[p])
        assert len(bad) == 0, f"plane {p}: {len(bad)} samples differ, first at {tuple(bad[0])}"
