#!/usr/bin/env python
"""BASELINE.json config 5: deblock + SAO saturation sweep.  Work lists that carry ONLY the two in-loop filter stages (deblock
grids + SAO grid of a synthetic picture; the MC / residual / intra sections are emptied) run back to back on 1..L compute lanes
(pictures in flight); reported: pictures/s and the achieved GB/s of the two stages together against their algorithmic bytes
(SURVEY.md 8d: 2 x B bytes per sample and stage + side tables).  Default geometry: 7680x4320 4:2:2 10-bit.

    python tools/dbk_sao_sweep.py [--workload c5_8k_422_main10] [--lanes 1,2,4,8] [--pictures 64]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def one(workload, lanes, pictures):
    import numpy as np
    import torch
    from openhevc_b200 import FrameEngine
    from openhevc_b200 import worklist as W
    from openhevc_b200.synth import FrameSynth, smooth_frame
    wl = bench.WORKLOADS[workload]
    w, h, cfi, bd = wl["width"], wl["height"], wl["cfi"], wl["bit_depth"]
    n_slots = 2 * lanes + 3                                # the last slot is a dummy reference: pictures without one all share the engine's "intra" lane
    eng = FrameEngine(w, h, cfi, bd, n_slots=n_slots, n_arenas=2)
    blob, st = FrameSynth(w, h, cfi, bd, seed=0xB2000005, refs=[0, 1], cur_slot=2, poc=1, p_intra=0.08).generate()
    hdr = blob[:256].view(W.header_dt)
    for s in (W.SEC_TU4, W.SEC_TU4 + 1, W.SEC_TU4 + 2, W.SEC_TU4 + 3, W.SEC_INTRA, W.SEC_MC):
        hdr["sec"][0][s]["count"] = 0                      # the filters only: they run on whatever the slot holds
    hdr["mc_big_count"] = 0
    pin = eng.pinned(blob.nbytes)
    pin[:blob.nbytes] = blob
    for s in range(n_slots):
        eng.upload_slot(s, smooth_frame(w, h, cfi, bd, 7 + s))
    eng.upload(pin[:blob.nbytes], 0)
    eng.sync()
    for k in range(8):
        eng.execute(0, k % (n_slots - 1), [n_slots - 1])
    eng.sync()
    st_ = torch.cuda.ExternalStream(eng.lib.b200_stream(eng.h))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st_)
    for k in range(pictures):
        eng.execute(0, k % (n_slots - 1), [n_slots - 1])
    eng.join()
    e1.record(st_)
    eng.sync(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    nbytes = st["bytes_deblock"] + st["bytes_sao"]
    eng.close()
    return {"lanes": lanes, "pictures": pictures, "pictures_per_s": pictures / (ms * 1e-3), "gbps_deblock_plus_sao": nbytes * pictures / (ms * 1e-3) / 1e9,
            "algorithmic_bytes_per_picture": nbytes}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c5_8k_422_main10")
    ap.add_argument("--lanes", default="1,2,4,8")
    ap.add_argument("--pictures", type=int, default=64)
    ap.add_argument("--one", type=int, default=0, help="(internal) run one lane count in this process: B200_LANES is read at context creation")
    a = ap.parse_args()
    if a.one:
        print(json.dumps(one(a.workload, a.one, a.pictures)))
        return
    peak = 3350.0                      # H100 SXM data sheet (HBM3); MEASURED_PEAKS.json replaces it
    try:
        peak = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        pass
    rows = []
    for l in [int(v) for v in a.lanes.split(",")]:
        r = subprocess.run([sys.executable, __file__, "--workload", a.workload, "--one", str(l), "--pictures", str(a.pictures)], capture_output=True, text=True,
                           env=dict(os.environ, B200_LANES=str(l)), timeout=1800)
        line = [x for x in r.stdout.splitlines() if x.startswith("{")]
        rows.append(json.loads(line[-1]) if line else {"lanes": l, "error": r.stderr[-300:]})
        if "gbps_deblock_plus_sao" in rows[-1]:
            rows[-1]["frac_of_hbm_peak"] = rows[-1]["gbps_deblock_plus_sao"] / peak
    print(json.dumps({"sweep": "deblock+sao", "workload": a.workload, "hbm_peak_gbs": peak, "rows": rows}))


if __name__ == "__main__":
    main()
