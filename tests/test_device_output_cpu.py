"""CPU suite for device-resident output: b200_yuv_to_rgb (k_yuv_rgb) and b200_slot_export_async, run on the warp-lockstep
emulated library (oracle/_ref/libb200hevc_emul.so: kernels.cu + engine.cu compiled unchanged for the CPU).

oracle_lib.yuv_rgb_reference() restates the fixed-point definition of openhevc_b200/csrc/k_yuv_rgb.cuh in numpy; the kernel must
equal it bit for bit, for uint8 and for float32 output."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle_lib import CROPPED, random_planes, yuv_rgb_reference

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REFDIR = os.path.join(ROOT, "oracle", "_ref")
EMUL = os.path.join(REFDIR, "libb200hevc_emul.so")
needs_emul = pytest.mark.skipif(not os.path.exists(EMUL), reason="oracle/_ref/libb200hevc_emul.so not built (make -C tests/emul)")


def run_yuv_rgb(lib, planes, cfi, bd, matrix, full_range, out_float, crop):
    from openhevc_b200 import _lib
    a = _lib.B200RgbArgs()
    for p in range(3):
        a.planes[p] = planes[p].ctypes.data
        a.pitches[p] = planes[p].strides[0]
    a.height, a.width = planes[0].shape
    a.chroma_format_idc, a.bit_depth, a.matrix, a.full_range, a.out_float = cfi, bd, matrix, full_range, out_float
    a.crop_x, a.crop_y, a.crop_w, a.crop_h = crop
    ow, oh = (crop[2], crop[3]) if crop[2] or crop[3] else (a.width, a.height)
    out = np.full((3, oh, ow), 77, np.float32 if out_float else np.uint8)
    a.out = out.ctypes.data
    rc = lib.b200_yuv_to_rgb(C.byref(a), None)
    return rc, out


def _emul_lib():
    from openhevc_b200 import _lib
    saved = _lib.LIB_PATH
    _lib.LIB_PATH = os.environ.get("B200_TEST_EMUL_LIB", EMUL)
    try:
        return _lib.load()
    finally:
        _lib.LIB_PATH = saved


# odd offsets and sizes that are not multiples of 8, the whole picture, one sample
CROPS = [(0, 0, 0, 0), (3, 5, 37, 19), (1, 2, 13, 7), (46, 30, 1, 1)]


def check_yuv_rgb(cfi, bd, w=48, h=32):
    lib = _emul_lib()
    planes = random_planes(w, h, cfi, bd, seed=100 * cfi + bd)
    n = 0
    for matrix in (1, 6, 9):
        for full_range in (0, 1):
            for out_float in (0, 1):
                for crop in CROPS:
                    c = (0, 0, w, h) if crop == (0, 0, 0, 0) else crop
                    rc, got = run_yuv_rgb(lib, planes, cfi, bd, matrix, full_range, out_float, crop)
                    assert rc == 0, (matrix, full_range, out_float, crop)
                    want = yuv_rgb_reference(planes, cfi, bd, matrix, full_range, out_float, c)
                    assert got.dtype == want.dtype and np.array_equal(got.view(np.uint8), want.view(np.uint8)), \
                        (cfi, bd, matrix, full_range, out_float, crop)
                    n += 1
    return n


@needs_emul
@pytest.mark.parametrize("bd", [8, 10, 12])
@pytest.mark.parametrize("cfi", [1, 2, 3])
def test_yuv_to_rgb_equals_the_fixed_point_definition(cfi, bd):
    assert check_yuv_rgb(cfi, bd) == 3 * 2 * 2 * len(CROPS)


@needs_emul
def test_yuv_to_rgb_float_output_spans_zero_to_one():
    lib = _emul_lib()
    bd = 10
    y = np.array([[0, 1023], [64, 940]], np.uint16)          # full-range black / white, limited-range black / white
    c = np.full((1, 1), 512, np.uint16)
    for full_range, black, white in ((1, (0, 0), (0, 1)), (0, (1, 0), (1, 1))):
        rc, out = run_yuv_rgb(lib, [y, c, c], 1, bd, 1, full_range, 1, (0, 0, 2, 2))
        assert rc == 0
        assert (out[:, black[0], black[1]] == 0).all() and (out[:, white[0], white[1]] == 1).all(), out


@needs_emul
def test_yuv_to_rgb_rejects_what_it_does_not_implement():
    lib = _emul_lib()
    planes = random_planes(16, 16, 1, 8, 1)
    assert run_yuv_rgb(lib, planes, 1, 8, 2, 0, 0, (0, 0, 0, 0))[0] == -5        # matrix_coefficients 2: unspecified
    assert run_yuv_rgb(lib, planes, 1, 8, 0, 0, 0, (0, 0, 0, 0))[0] == -5        # identity (GBR) is not a YUV matrix here
    assert run_yuv_rgb(lib, planes, 0, 8, 1, 0, 0, (0, 0, 0, 0))[0] == -5        # monochrome
    assert run_yuv_rgb(lib, planes, 1, 14, 1, 0, 0, (0, 0, 0, 0))[0] == -5       # 14 bit
    assert run_yuv_rgb(lib, planes, 1, 8, 1, 0, 0, (8, 8, 9, 4))[0] == -1        # crop window outside the picture


VARIANT_CODE = ("import sys; sys.path[:0] = [%r, %r]\n"
                "import test_device_output_cpu as T\n"
                "for cfi in (1, 2, 3):\n"
                "    for bd in (8, 10, 12): T.check_yuv_rgb(cfi, bd)\n"
                "T.check_export(1, 10); T.check_export(2, 8)\n")


@needs_emul
def test_yuv_to_rgb_and_export_in_reverse_lane_order():
    r = subprocess.run([sys.executable, "-c", VARIANT_CODE % (ROOT, HERE)], capture_output=True, text=True, timeout=900,
                       env=dict(os.environ, B200_EMUL_ORDER="reverse"))
    assert r.returncode == 0, r.stderr[-3000:]


@needs_emul
def test_yuv_to_rgb_and_export_under_the_address_sanitizer():
    asan_lib = os.path.join(REFDIR, "libb200hevc_emul_asan.so")
    rt = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.exists(asan_lib) or not os.path.isabs(rt) or not os.path.exists(rt):
        pytest.skip("no address sanitizer build / runtime")
    r = subprocess.run([sys.executable, "-c", VARIANT_CODE % (ROOT, HERE)], capture_output=True, text=True, timeout=1800,
                       env=dict(os.environ, B200_TEST_EMUL_LIB=asan_lib, LD_PRELOAD=rt,
                                ASAN_OPTIONS="detect_leaks=0:detect_stack_use_after_return=0"))
    assert r.returncode == 0 and "ERROR: AddressSanitizer" not in r.stderr, r.stderr[-4000:]


def check_export(cfi, bd, w=64, h=48):
    """b200_slot_export_async of a slot equals b200_slot_readback of the same slot, cropped"""
    from openhevc_b200 import FrameEngine, _lib
    saved = _lib.LIB_PATH
    _lib.LIB_PATH = os.environ.get("B200_TEST_EMUL_LIB", EMUL)
    try:
        eng = FrameEngine(w, h, cfi, bd, n_slots=3)
    finally:
        _lib.LIB_PATH = saved
    try:
        sx, sy = int(cfi != 3), int(cfi == 1)
        pics = [random_planes(w, h, cfi, bd, seed=7 + s) for s in range(3)]
        for s in range(3):
            eng.upload_slot(s, pics[s])
        for slot, (x, y, cw, ch) in ((0, (0, 0, 0, 0)), (1, (6, 4, 40, 36)), (2, (2, 2, 58, 38))):
            cw, ch = (cw, ch) if cw else (w, h)
            full = eng.readback(slot)
            dst, e = [], _lib.B200Export()
            for p in range(3):
                hs, vs = (sx, sy) if p else (0, 0)
                pitch = (cw >> hs) + 24                            # rows padded: the pitch is the destination's own
                buf = np.full((ch >> vs, pitch), 0xAB, eng.dtype)
                dst.append(buf)
                e.planes[p], e.pitches[p] = buf.ctypes.data, buf.strides[0]
            e.crop_x, e.crop_y, e.crop_w, e.crop_h = (x, y, cw, ch) if (x, y) != (0, 0) or cw != w else (0, 0, 0, 0)
            tok = C.c_uint32()
            eng._chk(eng.lib.b200_slot_export_async(eng.h, slot, C.byref(e), C.byref(tok)))
            eng._chk(eng.lib.b200_export_wait(eng.h, tok.value))
            assert eng.lib.b200_export_event(eng.h, tok.value)
            for p in range(3):
                hs, vs = (sx, sy) if p else (0, 0)
                want = full[p][y >> vs:(y + ch) >> vs, x >> hs:(x + cw) >> hs]
                assert np.array_equal(dst[p][:, :cw >> hs], want), (cfi, bd, slot, p)
                assert (dst[p][:, cw >> hs:] == 0xAB).all()           # nothing written past the row
    finally:
        eng.close()


@needs_emul
@pytest.mark.parametrize("cfi,bd", [(1, 8), (1, 10), (2, 12), (3, 8)])
def test_export_equals_readback_cropped(cfi, bd):
    check_export(cfi, bd)


@needs_emul
def test_export_rejects_crop_windows_off_the_chroma_grid():
    from openhevc_b200 import FrameEngine, _lib
    saved = _lib.LIB_PATH
    _lib.LIB_PATH = EMUL
    try:
        eng = FrameEngine(32, 32, 1, 8, n_slots=1)
    finally:
        _lib.LIB_PATH = saved
    try:
        buf = np.zeros((32, 32), np.uint8)
        for crop in ((1, 0, 8, 8), (0, 1, 8, 8), (0, 0, 7, 8), (0, 0, 8, 7), (24, 0, 10, 8), (-2, 0, 8, 8)):
            e = _lib.B200Export()
            for p in range(3):
                e.planes[p], e.pitches[p] = buf.ctypes.data, 32
            e.crop_x, e.crop_y, e.crop_w, e.crop_h = crop
            assert eng.lib.b200_slot_export_async(eng.h, 0, C.byref(e), None) == -1, crop
        e.crop_x, e.crop_y, e.crop_w, e.crop_h = 0, 0, 16, 8
        e.pitches[1] = 7                                                          # chroma rows of 8 samples need 8 bytes
        assert eng.lib.b200_slot_export_async(eng.h, 0, C.byref(e), None) == -1
        e.pitches[1] = 32
        assert eng.lib.b200_export_event(eng.h, 64) is None
        e.crop_x, e.crop_y, e.crop_w, e.crop_h = 0, 0, 0, 0
        assert eng.lib.b200_slot_export_async(eng.h, 0, C.byref(e), None) == 0      # the rejected calls left the context usable
    finally:
        eng.close()


@needs_emul
@pytest.mark.parametrize("threads", ["1", "4"])
def test_cropped_stream_through_the_host_path_on_the_emulated_device(threads):
    decoder = os.path.join(REFDIR, "decode_b200")
    if not os.path.exists(decoder):
        pytest.skip("oracle/_ref/decode_b200 not built (needs the reference sources)")
    out = subprocess.run([decoder, CROPPED, threads], capture_output=True, text=True, timeout=900, env=dict(os.environ, LD_PRELOAD=EMUL))
    assert out.returncode == 0, out.stderr[-2000:]
    assert [ln for ln in out.stdout.splitlines() if ln.startswith("frame ")] == open(CROPPED[:-5] + ".md5").read().splitlines()


def test_cropped_stream_has_a_conformance_window():
    want = open(CROPPED[:-5] + ".md5").read().splitlines()
    assert len(want) == 4 and all(" 416x240 bd10 " in ln for ln in want)
    ref = os.path.join(REFDIR, "decode_ref")
    if os.path.exists(ref):
        out = subprocess.run([ref, CROPPED, "1"], capture_output=True, text=True, timeout=120)
        assert [ln for ln in out.stdout.splitlines() if ln.startswith("frame ")] == want
