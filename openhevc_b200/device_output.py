"""Decoded pictures as torch CUDA tensors: FrameEngine.export (b200_slot_export_async) and yuv_to_rgb (b200_yuv_to_rgb).

Planes are (H, W) tensors in the AVFrame sample layout: torch.uint8 at 8 bit, torch.int16 above (samples of up to 12 bit
fit int16 bit for bit; torch's uint16 has no CUDA kernels).  Work is ordered on a torch stream through CUDA events, never by
synchronising the host."""
import ctypes as C

from . import _lib

MATRICES = {"bt709": 1, "bt601": 6, "bt2020": 9}
_cuda = None
_rgb_lib = None          # (path, library) of yuv_to_rgb: one ctypes set-up, not one per picture


def _driver():
    """libcuda: cuStreamWaitEvent lets a torch stream wait on the export event of the library (a runtime event is a driver event)"""
    global _cuda
    if _cuda is None:
        _cuda = C.CDLL("libcuda.so.1")
        _cuda.cuStreamWaitEvent.restype = C.c_int
        _cuda.cuStreamWaitEvent.argtypes = [C.c_void_p, C.c_void_p, C.c_uint]
    return _cuda


def sample_dtype(bit_depth):
    import torch
    return torch.uint8 if bit_depth <= 8 else torch.int16


def _check_plane(t, dtype, what):
    import torch
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != dtype or t.dim() != 2 or t.stride(1) != 1:
        raise ValueError(f"{what}: expected a CUDA {dtype} tensor of shape (H, W) with unit column stride")


def export(engine, slot, out=None, crop=None, stream=None):
    """copy DPB slot `slot` of `engine` into three CUDA tensors, ordered on `stream` (default: torch's current stream):
    the copy starts after the work queued on `stream` so far and `stream` waits for the copy.  New tensors are allocated on
    `stream`; tensors passed as `out` must be free for writing once the work queued on `stream` has run."""
    import torch
    x, y, w, h = crop if crop is not None else (0, 0, engine.width, engine.height)
    sx, sy = int(engine.cfi != 3), int(engine.cfi == 1)
    shapes = [(h, w), (h >> sy, w >> sx), (h >> sy, w >> sx)]
    dt = sample_dtype(engine.bit_depth)
    dev = torch.device("cuda", engine.cfg.device)
    stream = stream if stream is not None else torch.cuda.current_stream(dev)
    if out is None:
        # allocated on `stream`: the caching allocator then only reuses memory whose earlier users `stream` is ordered after
        with torch.cuda.device(dev), torch.cuda.stream(stream):
            out = [torch.empty(s, dtype=dt, device=dev) for s in shapes]
    for p in range(3):
        _check_plane(out[p], dt, f"export plane {p}")
        if tuple(out[p].shape) != shapes[p]:
            raise ValueError(f"export plane {p}: shape {tuple(out[p].shape)}, the crop window needs {shapes[p]}")
    before = torch.cuda.Event()
    before.record(stream)
    e = _lib.B200Export()
    for p in range(3):
        e.planes[p] = out[p].data_ptr()
        e.pitches[p] = out[p].stride(0) * out[p].element_size()
    e.crop_x, e.crop_y, e.crop_w, e.crop_h = x, y, w, h
    e.after_event = before.cuda_event
    token = C.c_uint32()
    engine._chk(engine.lib.b200_slot_export_async(engine.h, slot, C.byref(e), C.byref(token)))
    ev = engine.lib.b200_export_event(engine.h, token.value)
    rc = _driver().cuStreamWaitEvent(C.c_void_p(stream.cuda_stream), C.c_void_p(ev), 0)
    if rc:
        raise RuntimeError(f"cuStreamWaitEvent failed ({rc})")
    return out


def yuv_to_rgb(planes, chroma_format_idc, bit_depth, matrix="bt709", full_range=False, dtype=None, out=None, crop=None):
    """planar RGB (3, H, W) of the YUV planes (CUDA tensors, AVFrame layout), computed by k_yuv_rgb on torch's current stream.
    dtype torch.uint8, or torch.float32 (default) in [0, 1]; matrix "bt601" / "bt709" / "bt2020" (non-constant luminance) or
    an H.265 matrix_coefficients value; crop = (x, y, w, h) in luma samples, any offsets and sizes."""
    import torch
    dtype = torch.float32 if dtype is None else dtype
    if dtype not in (torch.uint8, torch.float32):
        raise ValueError("yuv_to_rgb: dtype must be torch.uint8 or torch.float32")
    dt = sample_dtype(bit_depth)
    for p in range(3):
        _check_plane(planes[p], dt, f"yuv_to_rgb plane {p}")
    height, width = planes[0].shape
    x, y, w, h = crop if crop is not None else (0, 0, width, height)
    if out is None:
        out = torch.empty((3, h, w), dtype=dtype, device=planes[0].device)
    if out.dtype != dtype or tuple(out.shape) != (3, h, w) or not out.is_contiguous() or out.device != planes[0].device:
        raise ValueError(f"yuv_to_rgb: out must be a contiguous {dtype} tensor of shape {(3, h, w)} on {planes[0].device}")
    a = _lib.B200RgbArgs()
    for p in range(3):
        a.planes[p] = planes[p].data_ptr()
        a.pitches[p] = planes[p].stride(0) * planes[p].element_size()
    a.width, a.height, a.chroma_format_idc, a.bit_depth = width, height, chroma_format_idc, bit_depth
    a.crop_x, a.crop_y, a.crop_w, a.crop_h = x, y, w, h
    a.matrix = MATRICES[matrix] if isinstance(matrix, str) else int(matrix)
    a.full_range, a.out_float, a.out = int(bool(full_range)), int(dtype == torch.float32), out.data_ptr()
    global _rgb_lib
    if _rgb_lib is None or _rgb_lib[0] != _lib.LIB_PATH:
        _rgb_lib = (_lib.LIB_PATH, _lib.load())
    lib = _rgb_lib[1]
    with torch.cuda.device(planes[0].device):
        rc = lib.b200_yuv_to_rgb(C.byref(a), C.c_void_p(torch.cuda.current_stream().cuda_stream))
    if rc:
        raise RuntimeError(f"b200_yuv_to_rgb failed ({rc}{': unsupported matrix / chroma format / bit depth' if rc == -5 else ''})")
    return out
