"""Device-resident output on the GPU: FrameEngine.export (b200_slot_export_async) ordered as a slot reader, and yuv_to_rgb
(k_yuv_rgb) against the numpy restatement of its fixed-point definition (test_device_output_cpu.yuv_rgb_reference)."""
import os

import numpy as np
import pytest

import oracle_lib
from test_device_output_cpu import random_planes, yuv_rgb_reference

pytestmark = pytest.mark.gpu
STREAMS = oracle_lib.recorded_streams()


def _planes_np(planes):
    return [p.cpu().numpy().view(np.uint16) if p.dtype.itemsize == 2 else p.cpu().numpy() for p in planes]


@pytest.mark.parametrize("stream", STREAMS, ids=os.path.basename)
def test_export_of_every_picture_equals_the_reference_decoder(stream):
    """every picture is exported right after its submission, without any host synchronisation, and writers of the same DPB
    slot are queued behind it (the later pictures, grey fills of the slot right behind the export where no later picture reads
    it, and of every slot at the end): the exports must still hold the picture (the export is a reader of the slot, so its
    next writer waits for it) and equal the MD5s of the reference decoder (which b200_slot_readback reproduces,
    tests/test_recorded_worklists.py)"""
    import torch
    from openhevc_b200 import FrameEngine
    from openhevc_b200 import worklist as W
    rec = oracle_lib.recorded_worklists(stream)
    want = open(stream[:-5] + ".md5").read().splitlines()
    hdr0, _ = W.parse_blob(rec["blobs"][0])
    w, h, cfi, bd = int(hdr0["width"]), int(hdr0["height"]), int(hdr0["chroma_format_idc"]), int(hdr0["bit_depth"])
    eng = FrameEngine(w, h, cfi, bd, log2_ctb_size=int(hdr0["log2_ctb_size"]), n_slots=32)
    try:
        hdrs = [W.parse_blob(b)[0] for b in rec["blobs"]]
        later_refs = [set() for _ in hdrs]                 # slots a later picture still reads (or refills / rewrites)
        for k in range(len(hdrs) - 1, 0, -1):
            h_ = hdrs[k]
            later_refs[k - 1] = later_refs[k] | {int(r) for r in np.ravel(h_["ref_slot"])[:int(h_["n_ref"])]} | {int(h_["cur_slot"])} | \
                {slot for (pic, slot, _v) in rec["fills"] if pic == k}
        exported = []
        for k, blob in enumerate(rec["blobs"]):
            for (pic, slot, value) in rec["fills"]:
                if pic == k:
                    eng.fill_slot(slot, value)
            eng.submit(blob)
            slot = int(hdrs[k]["cur_slot"])
            exported.append((rec["out_idx"][k], hdrs[k], eng.export(slot)))
            if slot not in later_refs[k]:                  # nobody reads the picture again: overwrite it right behind the export
                eng.fill_slot(slot, 17 + k)
        for slot in range(32):                             # and every slot once all pictures are queued
            eng.fill_slot(slot, 3)
        torch.cuda.current_stream().synchronize()
        for idx, hdr, planes in exported:
            assert oracle_lib.md5_line(idx, hdr, _planes_np(planes)) == want[idx], f"picture {idx} of {os.path.basename(stream)}"
    finally:
        torch.cuda.synchronize()
        eng.close()


@pytest.mark.parametrize("name", ["b_416x240_10b_weighted", "c422_416x240_10b_lowdelay", "c444_416x240_8b_ra"])
def test_cropped_export_equals_cropped_readback(name):
    import torch
    from openhevc_b200 import FrameEngine
    from openhevc_b200 import worklist as W
    rec = oracle_lib.recorded_worklists(os.path.join(oracle_lib.ROOT, "tests", "golden", "streams", name + ".hevc"))
    hdr, _ = W.parse_blob(rec["blobs"][0])
    w, h, cfi, bd = int(hdr["width"]), int(hdr["height"]), int(hdr["chroma_format_idc"]), int(hdr["bit_depth"])
    sx, sy = int(cfi != 3), int(cfi == 1)
    eng = FrameEngine(w, h, cfi, bd, log2_ctb_size=int(hdr["log2_ctb_size"]), n_slots=32)
    try:
        eng.submit(rec["blobs"][0])
        slot = int(hdr["cur_slot"])
        x, y, cw, ch = 6, 4, w - 22, h - 16
        side = torch.cuda.Stream()
        got = eng.export(slot, crop=(x, y, cw, ch), stream=side)
        side.synchronize()
        full = eng.readback(slot)
        for p in range(3):
            hs, vs = (sx, sy) if p else (0, 0)
            want = full[p][y >> vs:(y + ch) >> vs, x >> hs:(x + cw) >> hs]
            assert np.array_equal(_planes_np(got)[p], want), p
    finally:
        torch.cuda.synchronize()
        eng.close()


def _rgb_case(w, h, cfi, bd, matrix, full_range, out_float, crop, seed):
    import torch
    from openhevc_b200 import yuv_to_rgb
    planes = random_planes(w, h, cfi, bd, seed)
    dev = [torch.from_numpy(p.view(np.int16) if bd > 8 else p).cuda() for p in planes]
    got = yuv_to_rgb(dev, cfi, bd, matrix={1: "bt709", 6: "bt601", 9: "bt2020"}[matrix], full_range=bool(full_range),
                     dtype=torch.float32 if out_float else torch.uint8, crop=crop).cpu().numpy()
    want = yuv_rgb_reference(planes, cfi, bd, matrix, full_range, out_float, crop or (0, 0, w, h))
    assert got.dtype == want.dtype and np.array_equal(got.view(np.uint8), want.view(np.uint8)), (w, h, cfi, bd, matrix, full_range, out_float, crop)


@pytest.mark.parametrize("matrix,full_range,out_float", [(9, 0, 1), (9, 0, 0), (1, 1, 1), (6, 0, 0)])
def test_yuv_to_rgb_full_size_4k_10bit(matrix, full_range, out_float):
    _rgb_case(3840, 2160, 1, 10, matrix, full_range, out_float, None, seed=matrix + 10 * full_range)


@pytest.mark.parametrize("bd", [8, 10, 12])
@pytest.mark.parametrize("cfi", [1, 2, 3])
def test_yuv_to_rgb_small_pictures(cfi, bd):
    for matrix in (1, 6, 9):
        for full_range in (0, 1):
            for out_float in (0, 1):
                for crop in (None, (3, 5, 37, 19), (1, 2, 13, 7)):
                    _rgb_case(48, 32, cfi, bd, matrix, full_range, out_float, crop, seed=cfi * 100 + bd)


@pytest.mark.parametrize("threads", ["1", "4"])
def test_cropped_stream_through_the_hooked_decoder(threads):
    """the host read-back path on a stream with a conformance window (output frames point inside their buffers)"""
    import subprocess
    from test_device_output_cpu import CROPPED, REFDIR
    decoder = os.path.join(REFDIR, "decode_b200")
    if not os.path.exists(decoder):
        pytest.skip("oracle/_ref/decode_b200 not built")
    out = subprocess.run([decoder, CROPPED, threads], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    assert [ln for ln in out.stdout.splitlines() if ln.startswith("frame ")] == open(CROPPED[:-5] + ".md5").read().splitlines()
