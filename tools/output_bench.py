#!/usr/bin/env python
"""What device-resident output costs on one GPU; prints one JSON line.

 * k_yuv_rgb (b200_yuv_to_rgb) on a 3840x2160 4:2:0 10-bit picture, uint8 and float32 output; algorithmic bytes = every Y, Cb,
   Cr sample read once + every RGB sample written once; GB/s and the share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s)
 * b200_slot_export_async of one 4K slot (device-to-device copy, FrameEngine.export): the same way
 * the card's name and power limit, read in the same run
Timing: a long spin kernel is queued first, then the timed launches between two CUDA events.  The host enqueues all of them
while the device still spins, so the interval between the events is device time, not the rate at which Python issues calls;
`queued_before_start` records that this held (the start event had not completed when the last launch was queued).
Needs a GPU."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM_PEAK = 3.35e12          # H100 SXM data sheet
ITERS = 200


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    name, power = [v.strip() for v in q.splitlines()[0].split(",")]
    return name, power


def time_cuda(fn, iters=ITERS):
    """(seconds per call on the device, whether every call was queued before the first one started)"""
    import torch
    for _ in range(10):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    torch.cuda._sleep(400_000_000)                 # ~0.2 s at 2 GHz: longer than the host needs to queue `iters` calls
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    queued = not a.query()
    b.synchronize()
    return a.elapsed_time(b) * 1e-3 / iters, queued


def main():
    import torch
    from openhevc_b200 import FrameEngine, yuv_to_rgb
    name, power = card()
    res = {"gpu": name, "power_limit_w": power, "iters": ITERS}
    w, h, bd = 3840, 2160, 10
    g = torch.Generator(device="cuda").manual_seed(1)
    planes = [torch.randint(0, 1 << bd, s, dtype=torch.int16, device="cuda", generator=g) for s in ((h, w), (h // 2, w // 2), (h // 2, w // 2))]
    read = sum(p.numel() * 2 for p in planes)
    for dt, tag in ((torch.uint8, "uint8"), (torch.float32, "float32")):
        out = torch.empty((3, h, w), dtype=dt, device="cuda")
        t, queued = time_cuda(lambda: yuv_to_rgb(planes, 1, bd, matrix="bt2020", dtype=dt, out=out))
        nbytes = read + out.numel() * out.element_size()
        res[f"k_yuv_rgb_{tag}"] = {"us": round(t * 1e6, 2), "bytes": nbytes, "GBps": round(nbytes / t / 1e9, 1),
                                   "share_of_hbm_peak": round(nbytes / t / HBM_PEAK, 3), "queued_before_start": queued}
    eng = FrameEngine(w, h, 1, bd, n_slots=2)
    try:
        dst = eng.export(0)
        t, queued = time_cuda(lambda: eng.export(0, out=dst))
        nbytes = 2 * sum(p.numel() * 2 for p in dst)          # read + write
        res["export_4k_slot"] = {"us": round(t * 1e6, 2), "bytes": nbytes, "GBps": round(nbytes / t / 1e9, 1), "queued_before_start": queued}
    finally:
        torch.cuda.synchronize()
        eng.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
