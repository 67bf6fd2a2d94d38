"""TEST INFRASTRUCTURE: ctypes access to the CPU oracle (oracle/hevc_oracle.c) and helpers that
compare the CUDA path with it.  Never imported by the product package."""
import ctypes as C
import glob
import hashlib
import io
import lzma
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
ORACLE_SO = os.path.join(ORACLE_DIR, "_ref", "libhevc_oracle.so")
KAT_REF = os.path.join(ORACLE_DIR, "_ref", "kat_ref")
REF_SO = os.path.join(ORACLE_DIR, "_ref", "libohevc_ref.so")

_lib = None


def build_oracle():
    subprocess.run(["make", "-C", ORACLE_DIR], check=True, capture_output=True)


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(ORACLE_SO):
            build_oracle()
        _lib = C.CDLL(ORACLE_SO)
        _lib.orc_execute_blob.restype = C.c_int
        _lib.orc_execute_blob.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_int]
    return _lib


def execute(blob, dpb):
    """dpb: list of slots, each a list of three numpy planes (any unsigned dtype).  Executes the blob on the
    CPU oracle and returns the reconstructed picture of slot hdr.cur_slot as three uint16 planes."""
    blob = np.ascontiguousarray(blob, np.uint8)
    planes16 = [[np.ascontiguousarray(p, np.uint16).copy() for p in slot] for slot in dpb]
    flat = [p for slot in planes16 for p in slot]
    ptrs = (C.c_void_p * len(flat))(*[p.ctypes.data for p in flat])
    rc = lib().orc_execute_blob(blob.ctypes.data, ptrs, len(dpb))
    if rc:
        raise RuntimeError(f"orc_execute_blob failed: {rc}")
    cur = int(blob[23])
    return planes16[cur]


REPLAY_SO = os.path.join(ORACLE_DIR, "_ref", "libreplay_ref.so")
_ref = None


def ref_lib():
    """the UNMODIFIED reference's tables driven by oracle/replay_ref.c (prebuilt into oracle/_ref/)"""
    global _ref
    if _ref is None:
        if not os.path.exists(REPLAY_SO):
            build_oracle()
        if not os.path.exists(REPLAY_SO):
            return None
        _ref = C.CDLL(REPLAY_SO)
        _ref.ref_execute_blob.restype = C.c_int
        _ref.ref_execute_blob.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int]
        _ref.ref_bench.restype = C.c_double
        _ref.ref_bench.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int, C.c_int, C.c_int]
        if hasattr(_ref, "ref_bench_stage_seconds"):
            _ref.ref_bench_stage_seconds.restype = None
            _ref.ref_bench_stage_seconds.argtypes = [C.POINTER(C.c_double)]
    return _ref


def _native(dpb, bit_depth):
    dt = np.uint16 if bit_depth > 8 else np.uint8
    planes = [[np.ascontiguousarray(p, dt).copy() for p in slot] for slot in dpb]
    flat = [p for slot in planes for p in slot]
    ptrs = (C.c_void_p * len(flat))(*[p.ctypes.data for p in flat])
    strides = (C.c_int64 * len(flat))(*[p.strides[0] for p in flat])
    return planes, ptrs, strides


def ref_execute(blob, dpb):
    """same contract as execute(), computed by the reference's own C functions"""
    blob = np.ascontiguousarray(blob, np.uint8)
    planes, ptrs, strides = _native(dpb, int(blob[21]))
    rc = ref_lib().ref_execute_blob(blob.ctypes.data, ptrs, strides, len(dpb))
    if rc:
        raise RuntimeError(f"ref_execute_blob failed: {rc}")
    return planes[int(blob[23])]


SHIM_SO = os.path.join(ORACLE_DIR, "_ref", "libb200hevc_shim.so")


def ref_execute_b200(blob, dpb):
    """The reference-side call sequence (oracle/replay_ref.c) issued through the B200 drop-in tables
    (libb200hevc_shim.so -> recorder -> GPU -> readback).  Needs a GPU."""
    blob = np.ascontiguousarray(blob, np.uint8)
    planes, ptrs, strides = _native(dpb, int(blob[21]))
    L = ref_lib()
    L.ref_execute_blob_b200.restype = C.c_int
    L.ref_execute_blob_b200.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int, C.c_char_p, C.c_char_p, C.c_int]
    err = C.create_string_buffer(512)
    rc = L.ref_execute_blob_b200(blob.ctypes.data, ptrs, strides, len(dpb), SHIM_SO.encode(), err, 512)
    if rc:
        raise RuntimeError(f"ref_execute_blob_b200 failed: {rc}: {err.value.decode()}")
    return planes[int(blob[23])]


def ref_bench(blobs, dpb, n_threads, iters):
    """seconds of wall time for n_threads x iters pictures on the reference C path"""
    blobs = [np.ascontiguousarray(b, np.uint8) for b in blobs]
    planes, ptrs, strides = _native(dpb, int(blobs[0][21]))
    bp = (C.c_void_p * len(blobs))(*[b.ctypes.data for b in blobs])
    t = ref_lib().ref_bench(bp, len(blobs), ptrs, strides, len(dpb), n_threads, iters)
    if t < 0:
        raise RuntimeError(f"ref_bench failed: {t}")
    return t


def ref_bench_stages():
    """thread-seconds the last ref_bench() run spent in the table calls of each stage (summed over its threads)"""
    out = (C.c_double * 5)()
    ref_lib().ref_bench_stage_seconds(out)
    return dict(zip(("mc", "residual", "intra", "deblock", "sao"), [float(v) for v in out]))


def check_decode_order(blob):
    """host-side validation of a blob's intra list: every neighbour unit an intra TU reads must be final
    (not covered by a *later* intra TU).  A violation would make the device wavefront wait forever."""
    from openhevc_b200 import worklist as W
    hdr, secs = W.parse_blob(blob)
    intra = secs[W.SEC_INTRA]
    w, h, cfi = int(hdr["width"]), int(hdr["height"]), int(hdr["chroma_format_idc"])
    order = []
    for p in range(3):
        pw, ph = W.plane_dims(w, h, cfi, p)
        order.append(np.full((ph // 4 + 1, pw // 4 + 1), -1, np.int64))
    for i, r in enumerate(intra):
        u = 1 << (int(r["log2"]) - 2)
        o = order[int(r["plane"])]
        assert (o[int(r["y"]) // 4:int(r["y"]) // 4 + u, int(r["x"]) // 4:int(r["x"]) // 4 + u] == -1).all(), f"intra TU {i} overlaps an earlier one"
        o[int(r["y"]) // 4:int(r["y"]) // 4 + u, int(r["x"]) // 4:int(r["x"]) // 4 + u] = i
    for i, r in enumerate(intra):
        n, x, y, f = 1 << int(r["log2"]), int(r["x"]), int(r["y"]), int(r["flags"])
        o = order[int(r["plane"])]
        need = []
        if f & W.INF_UP_LEFT: need.append((x - 1, y - 1))
        if f & W.INF_UP: need += [(x + k, y - 1) for k in range(0, n, 4)]
        if f & W.INF_UP_RIGHT: need += [(x + n + k, y - 1) for k in range(0, int(r["top_right_size"]), 4)]
        if f & W.INF_LEFT: need += [(x - 1, y + k) for k in range(0, n, 4)]
        if f & W.INF_BOTTOM_LEFT: need += [(x - 1, y + n + k) for k in range(0, int(r["bottom_left_size"]), 4)]
        for (px, py) in need:
            assert px >= 0 and py >= 0, f"intra TU {i} reads outside the picture"
            assert o[py // 4, px // 4] < i, f"intra TU {i} depends on later TU {o[py // 4, px // 4]}"
    return True


WORKLIST_DIR = os.path.join(ROOT, "tests", "golden", "worklists")


def md5_line(k, hdr, planes):
    w, h, bd = int(hdr["width"]), int(hdr["height"]), int(hdr["bit_depth"])
    md5 = [hashlib.md5((np.asarray(p).astype(np.uint8) if bd == 8 else np.asarray(p).astype("<u2")).tobytes()).hexdigest() for p in planes]
    return f"frame {k} {w}x{h} bd{bd} " + " ".join(md5)


def recorded_worklists(stream, threads="1"):
    """work lists the hooked decoder recorded for a committed stream with `threads` ("1", "4", "4w"; golden/make_golden.py), or None"""
    import zipfile
    member = os.path.basename(stream).replace(".hevc", "") + {"1": "", "4": ".f4", "4w": ".w4"}[threads] + ".npz.xz"
    for pack in sorted(glob.glob(os.path.join(WORKLIST_DIR, "pack_*.zip"))):
        with zipfile.ZipFile(pack) as zf:
            if member in zf.namelist():
                z = np.load(io.BytesIO(lzma.decompress(zf.read(member))))
                break
    else:
        return None
    return dict(blobs=[z["blob"][a:b] for a, b in zip(z["off"][:-1], z["off"][1:])], out_idx=[int(v) for v in z["out_idx"]],
                fills=[tuple(int(v) for v in f) for f in z["fills"]])


def replay_worklists(rec, gpu):
    """recorded work lists in decode order on one DPB, by the CUDA path or the CPU oracle: {output index: md5_line}"""
    from openhevc_b200 import worklist as W
    hdr, _ = W.parse_blob(rec["blobs"][0])
    w, h, cfi, bd = int(hdr["width"]), int(hdr["height"]), int(hdr["chroma_format_idc"]), int(hdr["bit_depth"])
    n_slots, lines = 32, {}
    if gpu:
        from openhevc_b200 import FrameEngine
        eng = FrameEngine(w, h, cfi, bd, log2_ctb_size=int(hdr["log2_ctb_size"]), n_slots=n_slots)
    else:
        dpb = [[np.zeros(W.plane_dims(w, h, cfi, p)[::-1], np.uint16) for p in range(3)] for _ in range(n_slots)]
    try:
        for k, blob in enumerate(rec["blobs"]):
            hdr, _ = W.parse_blob(blob)
            for (pic, slot, value) in rec["fills"]:
                if pic == k and gpu:
                    eng.fill_slot(slot, value)
                elif pic == k:
                    dpb[slot] = [np.full_like(p, value) for p in dpb[slot]]
            if gpu:
                out = eng.decode(blob)
            else:
                out = execute(blob, dpb)
                dpb[int(hdr["cur_slot"])] = out
            lines[rec["out_idx"][k]] = md5_line(rec["out_idx"][k], hdr, out)
    finally:
        if gpu:
            eng.close()
    return lines


def recorded_streams():
    import zipfile
    names = [n for p in glob.glob(os.path.join(WORKLIST_DIR, "pack_*.zip")) for n in zipfile.ZipFile(p).namelist()]
    return sorted(os.path.join(ROOT, "tests", "golden", "streams", n[:-7] + ".hevc") for n in names if n.count(".") == 2)
