"""Host-side mirror of the reference's frame life cycle for the B200 back end.

`FrameEngine` plays the role the patched decoder plays through b200_frame_begin/end/readback
(INTEGRATION.md): it owns one libb200hevc context (device-resident DPB, upload arenas, streams),
accepts one work-list blob per picture and hands planes back in the reference's AVFrame layout
(planar, uint8 for 8-bit / little-endian uint16 above; hevc_ps.c:1666-1688).
"""
import ctypes as C
import numpy as np

from . import _lib, device_output
from ._lib import B200Error
from .worklist import header, plane_dims

STAGES = ("mc", "residual", "intra", "deblock", "sao", "total")


class PinnedBuffer:
    """uint8 numpy view over cudaHostAlloc memory (b200_host_alloc)."""

    def __init__(self, lib, nbytes):
        self._lib, self.nbytes = lib, int(nbytes)
        self.ptr = lib.b200_host_alloc(self.nbytes)
        if not self.ptr:
            raise B200Error("b200_host_alloc failed (no CUDA device?)")
        self.array = np.ctypeslib.as_array(C.cast(self.ptr, C.POINTER(C.c_uint8)), shape=(self.nbytes,))

    def free(self):
        if self.ptr:
            self.array = None
            self._lib.b200_host_free(self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class FrameEngine:
    def __init__(self, width, height, chroma_format_idc=1, bit_depth=8, log2_ctb_size=6, n_slots=6, n_arenas=2,
                 device=0, max_blob_bytes=0, ext_frame_mem=None, ext_frame_bytes=0, n_lanes=0):
        self.lib = _lib.load()
        self.cfg = _lib.B200Config(device, width, height, chroma_format_idc, bit_depth, log2_ctb_size, n_slots, n_arenas,
                                   max_blob_bytes, ext_frame_mem, ext_frame_bytes, n_lanes, 0)
        self.width, self.height, self.cfi, self.bit_depth, self.n_slots = width, height, chroma_format_idc, bit_depth, n_slots
        self.dtype = np.uint16 if bit_depth > 8 else np.uint8
        h = C.c_void_p()
        rc = self.lib.b200_ctx_create(C.byref(self.cfg), C.byref(h))
        if rc:
            raise B200Error(f"b200_ctx_create failed ({rc}): {self.lib.b200_last_error(None).decode()}", rc)
        self.h = h
        self._pinned = []

    # -- helpers ---------------------------------------------------------------------------------
    def _chk(self, rc):
        if rc:
            raise B200Error(f"libb200hevc error {rc}: {self.lib.b200_last_error(self.h).decode()}", rc)

    def plane_shape(self, p):
        w, h = plane_dims(self.width, self.height, self.cfi, p)
        return h, w

    def new_host_frame(self, pinned=False):
        """three contiguous planes in AVFrame layout"""
        if not pinned:
            return [np.zeros(self.plane_shape(p), self.dtype) for p in range(3)]
        sizes = [int(np.prod(self.plane_shape(p))) * np.dtype(self.dtype).itemsize for p in range(3)]
        buf = PinnedBuffer(self.lib, sum(sizes))
        self._pinned.append(buf)
        out, o = [], 0
        for p in range(3):
            out.append(buf.array[o:o + sizes[p]].view(self.dtype).reshape(self.plane_shape(p)))
            o += sizes[p]
        return out

    def pinned(self, nbytes):
        buf = PinnedBuffer(self.lib, nbytes)
        self._pinned.append(buf)
        return buf.array

    @staticmethod
    def _plane_args(planes):
        ptrs = (C.c_void_p * 3)(*[p.ctypes.data for p in planes])
        strides = (C.c_int64 * 3)(*[p.strides[0] for p in planes])
        return ptrs, strides

    # -- frame life cycle --------------------------------------------------------------------------
    def upload_slot(self, slot, planes):
        planes = [np.ascontiguousarray(p, self.dtype) for p in planes]
        for p in range(3):
            assert planes[p].shape == self.plane_shape(p), (planes[p].shape, self.plane_shape(p))
        ptrs, strides = self._plane_args(planes)
        self._chk(self.lib.b200_slot_upload(self.h, slot, ptrs, strides))
        self._chk(self.lib.b200_sync(self.h))     # source arrays may be temporaries

    def fill_slot(self, slot, value):
        self._chk(self.lib.b200_slot_fill(self.h, slot, int(value)))

    def submit(self, blob):
        """upload + execute one picture (asynchronous)"""
        blob = np.ascontiguousarray(blob, np.uint8)
        self._chk(self.lib.b200_frame_submit(self.h, blob.ctypes.data, blob.nbytes))

    def upload(self, blob, arena):
        self._chk(self.lib.b200_frame_upload(self.h, blob.ctypes.data, blob.nbytes, arena))

    def execute(self, arena, cur_slot=-1, ref_slots=None):
        if cur_slot < 0 and ref_slots is None:
            self._chk(self.lib.b200_frame_execute(self.h, arena))
        else:
            rs = bytes(ref_slots) if ref_slots is not None else None
            self._chk(self.lib.b200_frame_execute_ex(self.h, arena, cur_slot, rs, len(rs) if rs is not None else 0))

    def readback(self, slot, out=None, sync=True):
        out = out if out is not None else self.new_host_frame()
        ptrs, strides = self._plane_args(out)
        self._chk(self.lib.b200_slot_readback(self.h, slot, ptrs, strides))
        if sync:
            self.sync()
        return out

    def export(self, slot, out=None, crop=None, stream=None):
        """the picture in DPB slot `slot` as three torch CUDA tensors (H, W): uint8 at 8 bit, int16 above; crop = (x, y, w, h)
        in luma samples.  Ordered on `stream` (default: torch's current stream) after the slot's last writer; a later picture
        that rewrites the slot waits for the copy.  No host synchronisation."""
        return device_output.export(self, slot, out, crop, stream)

    def wait_readback(self, slot):
        """block until the last read-back of `slot` has landed in host memory (the queue keeps running)"""
        self._chk(self.lib.b200_slot_wait_readback(self.h, slot))

    def sync(self):
        self._chk(self.lib.b200_sync(self.h))

    def join(self):
        """b200_stream() (lane 0) waits for every picture submitted so far; record timing events on it afterwards"""
        self._chk(self.lib.b200_join(self.h))

    def slot_begin_access(self, slot, stream, write):
        self._chk(self.lib.b200_slot_begin_access(self.h, slot, C.c_void_p(stream), int(write)))

    def slot_end_access(self, slot, stream, write):
        self._chk(self.lib.b200_slot_end_access(self.h, slot, C.c_void_p(stream), int(write)))

    def decode(self, blob, out=None):
        """submit + readback of the picture's DPB slot (blocking): what a caller of the reference's
        libOpenHevcDecode + GetOutput sees for one access unit."""
        self.submit(blob)
        return self.readback(int(header(blob)["cur_slot"]), out)

    # -- measurement ---------------------------------------------------------------------------------
    def set_profiling(self, on=True):
        self._chk(self.lib.b200_set_profiling(self.h, int(on)))

    def stage_ms(self):
        ms = (C.c_float * 6)()
        self._chk(self.lib.b200_get_stage_ms(self.h, ms))
        return dict(zip(STAGES, [float(v) for v in ms]))

    def launch_count(self):
        return int(self.lib.b200_launch_count(self.h))

    def slot_devptr(self, slot, plane):
        pitch = C.c_uint64()
        p = self.lib.b200_slot_devptr(self.h, slot, plane, C.byref(pitch))
        return p, int(pitch.value)

    def slot_bytes(self):
        return int(self.lib.b200_slot_bytes(self.h))

    def close(self):
        if getattr(self, "h", None):
            self.lib.b200_ctx_destroy(self.h)
            self.h = None
        for b in self._pinned:
            b.free()
        self._pinned = []

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
