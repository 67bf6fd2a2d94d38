"""Committed golden fixtures (tests/golden/*.npz, produced by the reference's own C functions, see make_golden.py):
the oracle on the CPU, the CUDA path on the GPU."""
import glob
import os

import numpy as np
import pytest

import oracle_lib
from openhevc_b200.synth import smooth_frame

FIXTURES = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "*.npz")))


def load(path):
    z = np.load(path)
    w, h, cfi, bd = [int(v) for v in z["geom"]]
    dpb = [smooth_frame(w, h, cfi, bd, int(s)) for s in z["dpb_seeds"]]
    return z["blob"], (w, h, cfi, bd), dpb, [z["y"], z["cb"], z["cr"]]


def test_fixtures_exist():
    assert len(FIXTURES) >= 5


@pytest.mark.parametrize("path", FIXTURES, ids=[os.path.basename(p) for p in FIXTURES])
def test_oracle_reproduces_reference_golden(path):
    blob, geom, dpb, want = load(path)
    oracle_lib.assert_same(oracle_lib.execute(blob, dpb), want, os.path.basename(path))


@pytest.mark.gpu
@pytest.mark.parametrize("path", FIXTURES, ids=[os.path.basename(p) for p in FIXTURES])
def test_cuda_reproduces_reference_golden(path):
    from openhevc_b200 import FrameEngine
    blob, (w, h, cfi, bd), dpb, want = load(path)
    eng = FrameEngine(w, h, cfi, bd, n_slots=3)
    try:
        for s in (1, 2):
            eng.upload_slot(s, dpb[s])
        oracle_lib.assert_same(eng.decode(blob), want, os.path.basename(path))
    finally:
        eng.close()
