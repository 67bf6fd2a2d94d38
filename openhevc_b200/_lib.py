"""ctypes binding of libb200hevc.so (include/b200hevc.h).  There is no CPU fallback: if the CUDA
library has not been built (python __graft_entry__.py build) importing this module fails loudly."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B200_LIB_PATH") or os.path.join(_HERE, "libb200hevc.so")     # (B200_LIB_PATH: tuning builds of the same library, tools/)


class B200Config(C.Structure):
    _fields_ = [("device", C.c_int32), ("width", C.c_int32), ("height", C.c_int32), ("chroma_format_idc", C.c_int32),
                ("bit_depth", C.c_int32), ("log2_ctb_size", C.c_int32), ("n_slots", C.c_int32), ("n_arenas", C.c_int32),
                ("max_blob_bytes", C.c_uint64), ("ext_frame_mem", C.c_void_p), ("ext_frame_bytes", C.c_uint64),
                ("n_lanes", C.c_int32), ("reserved0", C.c_int32)]


class B200Export(C.Structure):
    _fields_ = [("planes", C.c_void_p * 3), ("pitches", C.c_int64 * 3), ("crop_x", C.c_int32), ("crop_y", C.c_int32),
                ("crop_w", C.c_int32), ("crop_h", C.c_int32), ("after_event", C.c_void_p)]


class B200RgbArgs(C.Structure):
    _fields_ = [("planes", C.c_void_p * 3), ("pitches", C.c_int64 * 3), ("width", C.c_int32), ("height", C.c_int32),
                ("chroma_format_idc", C.c_int32), ("bit_depth", C.c_int32), ("crop_x", C.c_int32), ("crop_y", C.c_int32),
                ("crop_w", C.c_int32), ("crop_h", C.c_int32), ("matrix", C.c_int32), ("full_range", C.c_int32),
                ("out_float", C.c_int32), ("reserved0", C.c_int32), ("out", C.c_void_p)]


EXPORTS = [  # every symbol include/b200hevc.h declares
    "b200_ctx_create", "b200_ctx_destroy", "b200_last_error", "b200_dpb_bytes", "b200_slot_bytes", "b200_slot_devptr",
    "b200_stream", "b200_join", "b200_slot_begin_access", "b200_slot_end_access", "b200_host_alloc", "b200_host_free", "b200_frame_upload", "b200_frame_execute", "b200_frame_execute_ex", "b200_frame_submit",
    "b200_slot_upload", "b200_slot_readback", "b200_slot_wait_readback", "b200_slot_fill", "b200_wait_uploads", "b200_sync", "b200_set_profiling", "b200_get_stage_ms",
    "b200_launch_count", "b200_rec_create", "b200_rec_destroy", "b200_rec_begin", "b200_rec_set_refs", "b200_rec_tu", "b200_rec_pcm",
    "b200_host_register", "b200_host_unregister", "b200_frame_submit_ex", "b200_upload_wait", "b200_slot_readback_async", "b200_readback_wait", "b200_poll_errors",
    "b200_rec_bs_leaf", "b200_rec_set_dbd", "b200_slot_export_async", "b200_export_wait", "b200_export_event", "b200_yuv_to_rgb",
    "b200_rec_intra", "b200_rec_mc", "b200_rec_deblock", "b200_rec_sao", "b200_rec_set_cip", "b200_rec_set_tqb", "b200_rec_tu_parked", "b200_rec_ccp", "b200_rec_merge", "b200_rec_finish", "b200_intra_level_order",
]


def load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: build the CUDA extension first (python -c 'import __graft_entry__ as g; g.build()'). "
                          "openhevc_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    vp, i32, u64, i64 = C.c_void_p, C.c_int, C.c_uint64, C.c_int64
    sig = {
        "b200_ctx_create": (i32, [C.POINTER(B200Config), C.POINTER(vp)]),
        "b200_ctx_destroy": (None, [vp]),
        "b200_last_error": (C.c_char_p, [vp]),
        "b200_dpb_bytes": (u64, [C.POINTER(B200Config)]),
        "b200_slot_bytes": (u64, [vp]),
        "b200_slot_devptr": (vp, [vp, i32, i32, C.POINTER(u64)]),
        "b200_stream": (vp, [vp]),
        "b200_rec_bs_leaf": (i32, [vp, i32, i32, i32, i32, i32]),
        "b200_rec_set_dbd": (i32, [vp, vp]),
        "b200_host_register": (i32, [vp, u64]),
        "b200_host_unregister": (i32, [vp]),
        "b200_frame_submit_ex": (i32, [vp, vp, u64, C.POINTER(C.c_uint32)]),
        "b200_upload_wait": (i32, [vp, C.c_uint32]),
        "b200_slot_readback_async": (i32, [vp, i32, C.POINTER(vp), C.POINTER(i64), C.POINTER(C.c_uint32)]),
        "b200_readback_wait": (i32, [vp, C.c_uint32]),
        "b200_poll_errors": (i32, [vp]),
        "b200_slot_export_async": (i32, [vp, i32, C.POINTER(B200Export), C.POINTER(C.c_uint32)]),
        "b200_export_wait": (i32, [vp, C.c_uint32]),
        "b200_export_event": (vp, [vp, C.c_uint32]),
        "b200_yuv_to_rgb": (i32, [C.POINTER(B200RgbArgs), vp]),
        "b200_join": (i32, [vp]),
        "b200_slot_begin_access": (i32, [vp, i32, vp, i32]),
        "b200_slot_end_access": (i32, [vp, i32, vp, i32]),
        "b200_host_alloc": (vp, [u64]),
        "b200_host_free": (None, [vp]),
        "b200_frame_upload": (i32, [vp, vp, u64, i32]),
        "b200_frame_execute": (i32, [vp, i32]),
        "b200_frame_execute_ex": (i32, [vp, i32, i32, C.c_char_p, i32]),
        "b200_frame_submit": (i32, [vp, vp, u64]),
        "b200_slot_upload": (i32, [vp, i32, C.POINTER(vp), C.POINTER(i64)]),
        "b200_slot_readback": (i32, [vp, i32, C.POINTER(vp), C.POINTER(i64)]),
        "b200_slot_wait_readback": (i32, [vp, i32]),
        "b200_slot_fill": (i32, [vp, i32, i32]),
        "b200_wait_uploads": (i32, [vp]),
        "b200_sync": (i32, [vp]),
        "b200_set_profiling": (i32, [vp, i32]),
        "b200_get_stage_ms": (i32, [vp, C.POINTER(C.c_float)]),
        "b200_launch_count": (u64, [vp]),
        "b200_rec_create": (i32, [C.POINTER(B200Config), C.POINTER(vp)]),
        "b200_rec_destroy": (None, [vp]),
        "b200_rec_begin": (i32, [vp, i32, i32]),
        "b200_rec_set_refs": (i32, [vp, C.c_char_p, i32]),
        "b200_rec_tu": (i32, [vp, i32, i32, i32, i32, i32, i32, i32, vp, i32]),
        "b200_rec_pcm": (i32, [vp, i32, i32, i32, i32, vp]),
        "b200_rec_intra": (i32, [vp, i32, i32, i32, i32, i32, i32, i32, i32]),
        "b200_rec_mc": (i32, [vp, vp]),
        "b200_rec_deblock": (i32, [vp, i32, i32, i32, i32, i32, C.POINTER(i32), C.POINTER(C.c_uint8), C.POINTER(C.c_uint8)]),
        "b200_rec_sao": (i32, [vp, i32, i32, i32, vp]),
        "b200_rec_set_cip": (i32, [vp, i32, i32, i32, vp]),
        "b200_rec_set_tqb": (i32, [vp, i32, i32, i32, vp]),
        "b200_rec_tu_parked": (i32, [vp, i32, i32, i32, i32, i32, i32, i32, vp, C.POINTER(C.c_uint32)]),
        "b200_rec_ccp": (i32, [vp, i32, i32, i32, i32, i32, C.c_uint32, i32, C.c_uint32]),
        "b200_rec_merge": (i32, [vp, vp]),
        "b200_rec_finish": (i32, [vp, C.POINTER(vp), C.POINTER(u64)]),
        "b200_intra_level_order": (i32, [vp, C.c_uint32, i32, i32, i32, vp]),
    }
    for name in EXPORTS:
        fn = getattr(lib, name)          # AttributeError here == the .so does not export what the header declares
        fn.restype, fn.argtypes = sig[name]
    return lib
