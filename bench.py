#!/usr/bin/env python
"""bench.py — decoded frames/s of openHEVC's pixel-reconstruction path on H100 GPUs.

Workload (BASELINE.json configs[2]/[3]): 3840x2160 Main10 4:2:0 random-access stream, hierarchical-B GOP 8,
intra period 32, synthetic work lists (openhevc_b200/synth.py, SURVEY.md §8d).  One *step* = one GOP
(8 pictures) per rank; pictures of GOP g are decoded by rank g mod N, anchors are broadcast over NCCL
(openhevc_b200/frame_parallel.py).  `value` = pictures/s with all work lists resident in HBM;
`e2e` = the same through the host-facing C ABI: pinned host blob -> H2D -> K1..K5 -> D2H of the picture.
--dump-outputs DIR writes the pictures of the last timed GOP of rank 0 as DIR/<name>.npy (float32).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

WORKLOADS = {
    "c3_4k_main10_ra": dict(width=3840, height=2160, cfi=1, bit_depth=10),
    "c2_1080p_main_ra": dict(width=1920, height=1080, cfi=1, bit_depth=8),
    "c1_832x480_main": dict(width=832, height=480, cfi=1, bit_depth=8, all_intra=True),
    "c3_4k_main10_intra": dict(width=3840, height=2160, cfi=1, bit_depth=10, all_intra=True),
    "c5_8k_422_main10": dict(width=7680, height=4320, cfi=2, bit_depth=10),
}
METRIC, UNIT = "decoded_frames_per_sec", "frames/s"


def workload_config(workload, wl, n_gpus):
    """the `config` of the JSON line: identical in both arms (the workload, not the implementation; what is specific to an arm --
    lanes, L2 note, launches -- lives in `arm`)"""
    return {"workload": workload, "picture": f"{wl['width']}x{wl['height']} 4:2:{'0' if wl['cfi'] == 1 else '2' if wl['cfi'] == 2 else '4'} {wl['bit_depth']}-bit",
            "gop": "all intra" if wl.get("all_intra") else "hierarchical-B 8, intra period 32", "step": "1 GOP (8 pictures) per rank",
            "stream": HEADLINE_STREAM.get(workload), "n_gpus": n_gpus}


def usable_cpus():
    """host threads this process can really run at once: the affinity mask, capped by the cgroup CPU quota
    (os.cpu_count() reports the machine, not the container)"""
    try:
        n = len(os.sched_getaffinity(0))
    except Exception:
        n = os.cpu_count() or 1
    for path in ("/sys/fs/cgroup/cpu.max", "/sys/fs/cgroup/cpu/cpu.cfs_quota_us"):
        try:
            f = open(path).read().split()
            if path.endswith("cpu.max"):
                quota, period = f[0], float(f[1])
            else:
                quota, period = f[0], float(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            if quota not in ("max", "-1"):
                n = max(1, min(n, int(float(quota) / period + 0.5)))
            break
        except Exception:
            continue
    return n


def make_blobs(wl, out_alloc=None):
    """the 9 distinct pictures of the periodic stream; symbolic reference table [0, 1], cur_slot 2"""
    from openhevc_b200.synth import FrameSynth
    from openhevc_b200 import frame_parallel as FP
    blobs, stats = [], []
    for i, (name, n_ref) in enumerate(FP.blob_specs()):
        if wl.get("all_intra"):                  # BASELINE.json config 1: I pictures only (the schedule still rotates the DPB slots)
            n_ref = 0
        s = FrameSynth(wl["width"], wl["height"], wl["cfi"], wl["bit_depth"], seed=0xB2000003 + i, refs=list(range(n_ref)),
                       cur_slot=2, poc=i, p_intra=0.08 if n_ref else 1.0, weighted=False)
        blob, st = s.generate()
        if out_alloc is not None:
            buf = out_alloc(blob.nbytes)
            buf[:blob.nbytes] = blob
            blob = buf[:blob.nbytes]
        blobs.append(blob); stats.append(st)
    return blobs, stats


def stream_mix():
    """how often each blob occurs per intra period (4 GOPs = 32 pictures)"""
    from openhevc_b200 import frame_parallel as FP
    mix = {}
    for g in range(FP.INTRA_PERIOD_GOPS):
        for p in FP.gop_pictures(g):
            mix[p.blob] = mix.get(p.blob, 0) + 1
    return mix


# ---- the REAL decoder on a real Annex-B stream (SURVEY.md §8d(i), BASELINE.json `metric`) --------------------------------------
# oracle/_ref/decode_ref = the unmodified reference (pure-C build of /root/reference, headless main_hm/main.c) and
# oracle/_ref/decode_b200 = the same decoder with the hook lines of INTEGRATION.md, pixel reconstruction on the GPU, both through
# the public libOpenHevc* API: Annex-B bytes in, host frames out.  Streams: committed recipes (tools/make_bench_streams.sh).
STREAM_DIR = os.path.join(ROOT, "oracle", "_ref", "streams")
STREAMS = {  # name: what it is
    "c3_4k_ra8_calm_65": "3840x2160 Main10 RA GOP 8, intra period 32, 65 pictures, lightly coded (~11 Mbit/s at 30 Hz: real-content bit rate)",
    "c3_4k_ra8_mid_65": "3840x2160 Main10 RA GOP 8, 65 pictures, --calm 0.5",
    "c3_4k_ra8_dense_33": "3840x2160 Main10 RA GOP 8, 33 pictures, dense random content (~110 Mbit/s: parse-bound worst case)",
    "c2_1080p_ra8_65": "1920x1080 8-bit RA GOP 8, 65 pictures",
    "c3_4k_wpp_ra8_calm_33": "3840x2160 Main10 RA GOP 8, 33 pictures, lightly coded, entropy_coding_sync (WPP: one substream per CTB row)",
    "c1_832x480_i_16": "832x480 8-bit all-intra, 16 pictures",
}
HEADLINE_STREAM = {"c3_4k_main10_ra": "c3_4k_ra8_calm_65", "c2_1080p_main_ra": "c2_1080p_ra8_65", "c1_832x480_main": "c1_832x480_i_16"}


def run_decoder(binary, stream, threads, passes, env=None, timeout=900):
    """one run of decode_ref / decode_b200 in timing mode (no MD5 work): the file is decoded `passes` times back to back by ONE
    decoder instance; returns frames, wall seconds and the steady-state rate (passes 2..n: start-up excluded)"""
    import re
    try:
        r = subprocess.run([os.path.join(ROOT, "oracle", "_ref", binary), stream, str(threads), "time", str(passes)], capture_output=True, text=True,
                           timeout=timeout, env=dict(os.environ, **(env or {})))
    except subprocess.TimeoutExpired:               # (the unmodified decoder's slice-threaded modes have been seen to hang on tile streams)
        return {"error": f"no result within {timeout} s", "rc": None}
    m = re.search(r"frames (\d+) time ([\d.]+) fps ([\d.]+) first_frame_s ([\d.]+) steady_fps ([\d.]+)", r.stdout)
    if r.returncode or not m:
        return {"error": (r.stderr or r.stdout)[-300:], "rc": r.returncode}
    out = {"frames": int(m.group(1)), "sec": float(m.group(2)), "fps_incl_startup": float(m.group(3)), "first_pass_s": float(m.group(4)),
           "steady_fps": float(m.group(5)), "passes": passes, "threads": threads}
    rep = re.search(r"b200 shim: pictures (\d+) h2d_bytes (\d+) d2h_bytes (\d+)", r.stderr)     # B200_SHIM_REPORT=1
    if rep and int(rep.group(1)):
        out.update(h2d_bytes_per_picture=int(rep.group(2)) / int(rep.group(1)), d2h_bytes_per_picture=int(rep.group(3)) / int(rep.group(1)))
    return out


def decoder_md5_ok(binary, stream, threads, env=None):
    """every output picture's plane MD5s equal the ones the unmodified decoder wrote (single thread) when the stream was made"""
    want_path = stream[:-5] + ".md5"
    if not os.path.exists(want_path):
        return None
    try:
        r = subprocess.run([os.path.join(ROOT, "oracle", "_ref", binary), stream, str(threads)], capture_output=True, text=True, timeout=300, env=dict(os.environ, **(env or {})))
    except subprocess.TimeoutExpired:
        return False
    got = [l for l in r.stdout.splitlines() if l.startswith("frame ")]
    want = open(want_path).read().splitlines()
    return r.returncode == 0 and got == want


def stream_block(name, arms, threads_all, device, budget_s=2.5, with_single=True, oversubscribe=False):
    """fps of the arms ("reference", "b200") on one stream, 1 thread and `threads_all` frame threads.  Pass counts are chosen so
    that every timed (steady) region lasts about budget_s or more."""
    path = os.path.join(STREAM_DIR, name + ".hevc")
    if not os.path.exists(path) or not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "decode_ref")):
        return {"unavailable": "stream or decoder binaries missing (tools/make_bench_streams.sh, __graft_entry__.build())"}
    n = len(open(path[:-5] + ".md5").read().splitlines()) if os.path.exists(path[:-5] + ".md5") else 65
    env = {"B200_DEVICE": str(device), "B200_SHIM_REPORT": "1"}
    out = {"what": STREAMS.get(name, name), "bytes": os.path.getsize(path), "pictures": n, "host_threads": threads_all}
    # oversubscribe: also 2 x the usable cores as frame threads, for BOTH arms -- frame threads block on each other's progress
    # (ff_thread_await_progress), so more threads than cores fill the gaps; SURVEY.md 8d(i): "report the best multithreaded fps with
    # the core count".  `best` names the fastest multithreaded run of each arm.
    tset = sorted({1, threads_all}) if with_single else [threads_all]
    if oversubscribe:
        tset = sorted(set(tset) | {2 * threads_all})
    for arm in arms:
        binary = "decode_ref" if arm == "reference" else "decode_b200"
        res = {}
        for t in tset:
            probe = run_decoder(binary, path, t, 2, env)
            if "error" in probe:
                res[f"threads_{t}"] = probe
                continue
            passes = int(min(64, max(2, 1 + budget_s * probe["steady_fps"] / n + 0.999)))
            best = probe if passes <= 2 else run_decoder(binary, path, t, passes, env)
            if t > 1 and "error" not in best:            # frame-threaded runs vary by +-10 % from run to run (scheduling): the better of two, both arms alike
                again = run_decoder(binary, path, t, max(2, passes), env)
                if "error" not in again and again["steady_fps"] > best["steady_fps"]:
                    best = again
                best["runs"] = 2
            res[f"threads_{t}"] = best if "error" not in best else probe
        if arm == "b200":
            res["md5_equal_reference_decoder"] = {f"threads_{t}": decoder_md5_ok(binary, path, t, env) for t in tset}
        out[arm] = res
    for arm in arms:
        multi = {t: out[arm][f"threads_{t}"]["steady_fps"] for t in tset if t > 1 and "steady_fps" in out[arm].get(f"threads_{t}", {})}
        if multi:
            bt = max(multi, key=multi.get)
            out[arm]["best"] = {"threads": bt, "steady_fps": multi[bt]}
    try:
        for t in tset:
            out[f"speedup_threads_{t}"] = out["b200"][f"threads_{t}"]["steady_fps"] / out["reference"][f"threads_{t}"]["steady_fps"]
        out["speedup_best_vs_best"] = out["b200"]["best"]["steady_fps"] / out["reference"]["best"]["steady_fps"]
    except Exception:
        pass
    return out


def thread_modes_block(name, threads_all, device, budget_s=1.5):
    """SURVEY.md 8d(i): the reference's three ways of using host threads -- frame threads (hevc -f 1), slice / WPP threads inside one
    picture (-f 2) and slice threads inside frame threads (-f 4, pthread.c:57-71) -- on a stream that carries entry points (WPP), both
    arms, steady fps.  The hooked decoder's pictures are checked against the single-threaded reference in every mode (the reference's
    own slice-threaded runs are not deterministic on 4K WPP streams -- its pictures are timed, not compared)."""
    path = os.path.join(STREAM_DIR, name + ".hevc")
    if not os.path.exists(path) or not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "decode_ref")):
        return {"unavailable": "stream or decoder binaries missing (tools/make_bench_streams.sh, __graft_entry__.build())"}
    n = len(open(path[:-5] + ".md5").read().splitlines()) if os.path.exists(path[:-5] + ".md5") else 33
    env = {"B200_DEVICE": str(device), "B200_SHIM_REPORT": "1"}
    ns = max(2, min(threads_all, 16))
    modes = {"frame": str(threads_all), "slice": f"{ns}w", "frame_slice": "4x"}
    out = {"what": STREAMS.get(name, name), "pictures": n, "host_threads": threads_all,
           "modes": {"frame": f"-f 1, {threads_all} frame threads", "slice": f"-f 2, {ns} WPP threads in one picture",
                     "frame_slice": f"-f 4, 4 WPP threads per picture x {min(threads_all // 4 + 1, 16)} frame threads"}}
    for arm in ("reference", "b200"):
        binary = "decode_ref" if arm == "reference" else "decode_b200"
        res = {}
        for mode, t in modes.items():
            probe = run_decoder(binary, path, t, 2, env, timeout=90)
            if "error" in probe:
                res[mode] = probe
                continue
            passes = int(min(64, max(2, 1 + budget_s * probe["steady_fps"] / n + 0.999)))
            best = probe if passes <= 2 else run_decoder(binary, path, t, passes, env, timeout=90)
            res[mode] = best if "error" not in best else probe
        if arm == "b200":
            res["md5_equal_reference_decoder"] = {mode: decoder_md5_ok(binary, path, t, env) for mode, t in modes.items()}
        ok = {m: r["steady_fps"] for m, r in res.items() if isinstance(r, dict) and "steady_fps" in r}
        if ok:
            bm = max(ok, key=ok.get)
            res["best"] = {"mode": bm, "steady_fps": ok[bm]}
        out[arm] = res
    try:
        for mode in modes:
            out[f"speedup_{mode}"] = out["b200"][mode]["steady_fps"] / out["reference"][mode]["steady_fps"]
        out["speedup_best_vs_best"] = out["b200"]["best"]["steady_fps"] / out["reference"]["best"]["steady_fps"]
    except Exception:
        pass
    return out


class ClockSampler:
    Q = "clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, index):
        self.rows, self.proc = [], None
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(index), f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "50"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append((time.time(), line.strip()))

    def wait_first(self, timeout=8.0):
        """nvidia-smi needs up to a few seconds before its first line: the timed region must not start before it"""
        t_end = time.time() + timeout
        while self.proc and not self.rows and time.time() < t_end:
            time.sleep(0.05)

    def stop(self, t0, t1):
        if not self.proc:
            return None
        time.sleep(0.15)
        self.proc.terminate()
        sm, mx, reasons = [], [], set()
        inside = [r for r in self.rows if t0 - 0.05 <= r[0] <= t1 + 0.15]
        if not inside and self.rows:             # timed region shorter than the sampling period: the nearest sample
            inside = [min(self.rows, key=lambda r: abs(r[0] - 0.5 * (t0 + t1)))]
        for (t, line) in inside:
            f = [x.strip() for x in line.split(",")]
            try:
                sm.append(float(f[0])); mx.append(float(f[1]))
            except Exception:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        if not sm:
            return None
        return {"sm_mhz": statistics.median(sm), "sm_max_mhz": max(mx), "reasons": sorted(reasons), "samples": len(sm)}


def run_reference(args, wl, rank):
    """--impl reference: the reference's own C functions (oracle/_ref, built from /root/reference) replaying the
    same work lists on the host cores, frame-parallel over pthreads like its frame threads."""
    if rank != 0:
        return
    if args.dump_outputs:
        print("bench.py: --dump-outputs applies to the GPU path only; the reference arm writes nothing", file=sys.stderr)
    import oracle_lib
    from openhevc_b200.synth import smooth_frame
    if oracle_lib.ref_lib() is None:
        print(json.dumps({"impl": "reference", "unavailable": "oracle/_ref/libreplay_ref.so missing (reference build not shipped)"}), file=_REAL_STDOUT, flush=True)
        return
    blobs, _ = make_blobs(wl)
    mix = stream_mix()
    seq = [blobs[b] for b, n in sorted(mix.items()) for _ in range(n)]
    rng = np.random.default_rng(1)
    seq = [seq[i] for i in rng.permutation(len(seq))]
    dpb = [smooth_frame(wl["width"], wl["height"], wl["cfi"], wl["bit_depth"], 7 + k) for k in range(3)]
    threads = min(usable_cpus(), 256)

    def iters_for(gops):
        return max(1, -(-gops * 8 // threads))
    if args.warmup:
        oracle_lib.ref_bench(seq, dpb, threads, 1)
    it = iters_for(args.steps)
    sec = oracle_lib.ref_bench(seq, dpb, threads, it)
    n = threads * it
    fps = n / sec
    try:
        stages = {k: {"ms_per_picture_one_core": 1e3 * v / n} for k, v in oracle_lib.ref_bench_stages().items()}
    except Exception:
        stages = None
    e2e = {"value": fps, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0, "what": "replay of the work lists (no stream available)"}
    sb = None
    hs = HEADLINE_STREAM.get(args.workload)
    if hs and not args.no_stream:
        sb = stream_block(hs, ["reference"], threads, 0, with_single=False, oversubscribe=True)
        try:
            best = sb["reference"]["best"]
            e2e = {"value": best["steady_fps"], "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0,
                   "what": f"unmodified reference decoder (oracle/_ref/decode_ref) on {hs}.hevc, best of {threads} and {2 * threads} frame threads ({best['threads']}) on {threads} usable cores, Annex-B bytes in, frames out"}
        except Exception:
            pass
    line = {"metric": METRIC, "value": fps, "unit": UNIT, "impl": "reference", "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": 1e3 * sec / max(1, n / 8), "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u16" if wl["bit_depth"] > 8 else "u8",
            "data": "synthetic", "config": workload_config(args.workload, wl, args.gpus), "arm": {"pictures_timed": n},
            "mpixels_per_s": fps * wl["width"] * wl["height"] / 1e6,
            "cpu_baseline": {"value": fps, "unit": UNIT, "cores": threads, "kind": "reference",
                             "sample": f"{n} pictures of the bench stream mix, {threads} threads x {it} pictures, reference C tables (-O3 -fno-tree-vectorize, no asm)",
                             "stages": stages},
            "e2e": e2e, "stream_e2e": sb}
    print(json.dumps(line), file=_REAL_STDOUT, flush=True)


DUMP_SAMPLES = 1 << 19        # per plane: 8 pictures x 3 planes x 2 MB of float32 stay under 64 MB


def dump_outputs(out_dir, eng, FP, rank, world, steps):
    """the pictures of the last GOP of the timed schedule on this rank, read back from their DPB slots (nothing later writes
    them); a plane larger than DUMP_SAMPLES is stored flat as a fixed, seeded sample of DUMP_SAMPLES samples"""
    class Record:
        def __init__(self):
            self.pics = []

        def decode(self, pic, g=None):
            self.pics.append((g, pic))

        def exchange_anchors(self, *a):
            pass
    rec = Record()
    FP.run_schedule(rec, rank, world, steps)
    g_last = max(g for g, _ in rec.pics)
    os.makedirs(out_dir, exist_ok=True)
    eng.sync()
    for k, pic in enumerate(p for g, p in rec.pics if g == g_last):
        planes = eng.readback(pic.cur_slot)
        for p, (name, a) in enumerate(zip(("y", "cb", "cr"), planes)):
            a = a.astype(np.float32)
            if a.size > DUMP_SAMPLES:
                idx = np.sort(np.random.default_rng(3 * k + p).choice(a.size, DUMP_SAMPLES, replace=False))
                a = a.reshape(-1)[idx]
            np.save(os.path.join(out_dir, f"gop{g_last}_pic{k}_{name}.npy"), a)


_REAL_STDOUT = sys.stdout


def main():
    # keep stdout clean for the ONE JSON line: libraries (NCCL banner, ...) write to fd 1; everything but the final
    # line goes to stderr
    global _REAL_STDOUT
    sys.stdout.flush()
    _REAL_STDOUT = os.fdopen(os.dup(1), "w")
    os.dup2(2, 1)
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=512, help="GOPs (8 pictures) per rank in the timed region (several ranks: rounded up to 4)")
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--workload", default="c3_4k_main10_ra", choices=sorted(WORKLOADS))
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-stream", action="store_true", help="skip the real-decoder stream block (e2e falls back to the work-list replay)")
    ap.add_argument("--streams", default="headline,mid,dense,modes", help="which streams the stream_e2e block decodes")
    ap.add_argument("--dump-outputs", metavar="DIR", help="write the pictures of the last timed GOP (rank 0) to DIR/<name>.npy")
    args = ap.parse_args()
    wl = WORKLOADS[args.workload]
    rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    if args.impl == "reference":
        return run_reference(args, wl, rank)
    args.warmup = max(args.warmup, 3)

    import torch
    import torch.distributed as dist
    from openhevc_b200 import FrameEngine, _lib
    from openhevc_b200 import frame_parallel as FP
    from openhevc_b200.synth import smooth_frame
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device; openhevc_b200 has no CPU fallback")
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))

    # ---- engine with the DPB inside a torch tensor (so NCCL can address slots) --------------------------------
    lib = _lib.load()
    cfg = _lib.B200Config(local, wl["width"], wl["height"], wl["cfi"], wl["bit_depth"], 6, FP.N_SLOTS, 16, 0, None, 0, 0, 0)
    slot_bytes = int(lib.b200_dpb_bytes(cfg)) // FP.N_SLOTS
    dpb = torch.zeros(FP.N_SLOTS * slot_bytes, dtype=torch.uint8, device=f"cuda:{local}")
    eng = FrameEngine(wl["width"], wl["height"], wl["cfi"], wl["bit_depth"], n_slots=FP.N_SLOTS, n_arenas=16, device=local,
                      ext_frame_mem=dpb.data_ptr(), ext_frame_bytes=dpb.numel())
    assert eng.slot_bytes() == slot_bytes
    blobs, stats = make_blobs(wl, out_alloc=eng.pinned)
    mix = stream_mix()
    npic_mix = sum(mix.values())
    eng.upload_slot(FP.anchor_slot(-1), smooth_frame(wl["width"], wl["height"], wl["cfi"], wl["bit_depth"], 7))
    for b, blob in enumerate(blobs):
        eng.upload(blob, b)
    eng.sync()
    backend = FP.GpuBackend(eng, dpb, slot_bytes, world, list(range(FP.N_BLOBS)))

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    # ---- value: device-resident work lists ----------------------------------------------------------------------
    sampler = ClockSampler(local) if rank == 0 else None
    FP.run_schedule(backend, rank, world, args.warmup)
    if sampler:
        sampler.wait_first()
    eng.sync(); barrier()
    l0 = eng.launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.time()
    e0.record(backend.compute)
    n_mine = FP.run_schedule(backend, rank, world, args.steps)
    eng.join()                                   # lane 0 waits for the pictures on every lane, then the end event
    e1.record(backend.compute)
    eng.sync(); torch.cuda.synchronize()
    t1 = time.time()
    ms = torch.tensor([e0.elapsed_time(e1)], device=f"cuda:{local}")
    launches = eng.launch_count() - l0
    barrier()
    clocks = sampler.stop(t0, t1) if sampler else None
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    ms = float(ms.item())
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, eng, FP, rank, world, args.steps)
    n_total = n_mine * world
    fps = n_total / (ms * 1e-3)

    # ---- per-stage times of every distinct picture (CUDA events inside the library, on its compute stream) ----
    eng.set_profiling(True)
    stage_ms = {k: 0.0 for k in ("mc", "residual", "intra", "deblock", "sao", "total")}
    reps = 3
    stage_by_blob = {}
    for b in range(FP.N_BLOBS):
        pic = next(p for g in range(FP.INTRA_PERIOD_GOPS) for p in FP.gop_pictures(g) if p.blob == b)
        acc = {k: 0.0 for k in stage_ms}
        for _ in range(reps):
            eng.execute(b, pic.cur_slot, pic.ref_slots)
            for k, v in eng.stage_ms().items():
                acc[k] += v / reps
        stage_by_blob[FP.blob_specs()[b][0] + f"#{b}"] = {k: round(v, 4) for k, v in acc.items()}
        for k in stage_ms:
            stage_ms[k] += acc[k] * mix[b] / npic_mix
    eng.set_profiling(False)
    B = 2 if wl["bit_depth"] > 8 else 1
    abytes = {k: sum(stats[b]["bytes_" + k] * mix[b] for b in mix) / npic_mix for k in ("mc", "residual", "intra", "deblock", "sao")}
    peaks_path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(peaks_path):
        peak, peak_src = float(json.load(open(peaks_path))["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    else:
        peak, peak_src = 3350.0, "H100 SXM data sheet (HBM3, 700 W card), not measured"
    stages = {k: {"ms": stage_ms[k], "algorithmic_bytes": abytes[k], "gbps": abytes[k] / (stage_ms[k] * 1e-3) / 1e9 if stage_ms[k] > 0 else None}
              for k in abytes}
    dom = max(abytes, key=lambda k: stage_ms[k])
    roofline = {"bound": "hbm", "kernel": {"mc": "k_mc", "residual": "k_residual", "intra": "k_intra", "deblock": "k_deblock", "sao": "k_sao"}[dom],
                "achieved": stages[dom]["gbps"], "peak": peak, "unit": "GB/s", "frac": stages[dom]["gbps"] / peak, "peak_source": peak_src,
                "share_of_step": stage_ms[dom] / stage_ms["total"], "stages": stages,
                "stage_ms_by_picture": stage_by_blob, "intra_levels": {FP.blob_specs()[b][0] + f"#{b}": (stats[b].get("intra_levels"), stats[b].get("intra_levels_in_ctb")) for b in range(FP.N_BLOBS)},
                "whole_picture": {"algorithmic_bytes": sum(abytes.values()), "ms": stage_ms["total"],
                                  "gbps": sum(abytes.values()) / (stage_ms["total"] * 1e-3) / 1e9}}

    # ---- e2e: pinned host work list -> H2D -> kernels -> D2H of the reconstructed picture, every picture ----------
    host_out = [eng.new_host_frame(pinned=True) for _ in range(24)]

    class E2E(FP.GpuBackend):
        def __init__(self, *a):
            super().__init__(*a)
            self.k = 0
            self.inflight = []

        def decode(self, pic, g=None):
            a = self.k % 16
            self.eng.upload(blobs[pic.blob], a)
            self.eng.execute(a, pic.cur_slot, pic.ref_slots)
            self.eng.readback(pic.cur_slot, host_out[self.k % 24], sync=False)
            self.k += 1
            self.inflight.append(pic.cur_slot)
            if len(self.inflight) > 12:         # bound the run-ahead of the host thread (host buffers are reused after 24): wait for
                self.eng.wait_readback(self.inflight.pop(0))   # ONE old picture to land, the queue behind it keeps running

    be2 = E2E(eng, dpb, slot_bytes, world, list(range(FP.N_BLOBS)))
    e2e_steps = max(2, args.steps // 2)
    FP.run_schedule(be2, rank, world, 1)
    eng.sync(); barrier()
    w0 = time.perf_counter()
    n_e2e = FP.run_schedule(be2, rank, world, e2e_steps)
    eng.sync(); torch.cuda.synchronize()
    w1 = torch.tensor([time.perf_counter() - w0], device=f"cuda:{local}")
    barrier()
    if world > 1:
        dist.all_reduce(w1, op=dist.ReduceOp.MAX)
    e2e_fps = n_e2e * world / float(w1.item())
    h2d = sum(blobs[b].nbytes * mix[b] for b in mix) / npic_mix * 8
    d2h = sum(int(np.prod(eng.plane_shape(p))) for p in range(3)) * B * 8

    # ---- CPU baseline: the reference's own C path on this box's host cores (rank 0, N=1 only) --------------------
    cpu = None
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        try:
            import oracle_lib
            if oracle_lib.ref_lib() is not None:
                rng = np.random.default_rng(1)
                seq = [np.array(blobs[b]) for b, n in sorted(mix.items()) for _ in range(n)]
                seq = [seq[i] for i in rng.permutation(len(seq))]
                cdpb = [smooth_frame(wl["width"], wl["height"], wl["cfi"], wl["bit_depth"], 7 + k) for k in range(3)]
                threads = min(usable_cpus(), 256)
                it = 6 if wl["width"] >= 3840 else 24       # ~20-30 s of CPU work (threads x it pictures)
                sec = oracle_lib.ref_bench(seq, cdpb, threads, it)
                cpu = {"value": threads * it / sec, "unit": UNIT, "cores": threads, "kind": "reference",
                       "sample": f"{threads * it} pictures of the same stream mix ({threads} threads x {it}), reference C tables via oracle/replay_ref.c, {sec:.1f} s"}
                try:                             # SURVEY.md §8d(ii): the same work lists, per stage, on the host cores beside each GPU kernel
                    st = oracle_lib.ref_bench_stages()
                    S = sum(int(np.prod(eng.plane_shape(p))) for p in range(3))
                    cpu["stages"] = {k: {"ms_per_picture_one_core": 1e3 * v / (threads * it),
                                         "gpu_stage_speedup_vs_one_core": (v / (threads * it)) / (stage_ms[k] * 1e-3) if stage_ms.get(k) else None} for k, v in st.items()}
                    cpu["msamples_per_s_one_core"] = S * threads * it / sum(st.values()) / 1e6
                except Exception:
                    pass
        except Exception as ex:                  # the baseline is a report, never a reason to lose the bench line
            cpu = {"value": None, "unit": UNIT, "cores": 0, "kind": "reference", "sample": f"failed: {ex}"}

    # ---- the real decoder on real streams: THE end-to-end number (BASELINE.json metric: decoded fps vs the reference CPU decoder) ----
    # Every rank decodes the stream on its own GPU with its share of the host cores (replicas: the host parse is what limits it).
    e2e_replay = {"value": e2e_fps, "unit": UNIT, "h2d_bytes_per_step": int(h2d), "d2h_bytes_per_step": int(d2h), "steps": e2e_steps,
                  "mpixels_per_s": e2e_fps * wl["width"] * wl["height"] / 1e6,
                  "what": "work-list replay: pinned host blob -> H2D -> K0..K5 -> D2H of every picture through the C ABI (no parse)"}
    e2e_line, stream_e2e = dict(e2e_replay), None
    hs = HEADLINE_STREAM.get(args.workload)
    if hs and not args.no_stream:
        eng.sync()
        threads_all = max(1, usable_cpus() // world)
        mine = stream_block(hs, ["b200"] if world > 1 else ["reference", "b200"], threads_all, local, with_single=(world == 1), oversubscribe=True)
        best = mine.get("b200", {}).get("best", {})
        sfps = torch.tensor([best.get("steady_fps", 0.0) or 0.0], device=f"cuda:{local}", dtype=torch.float64)
        if world > 1:
            dist.all_reduce(sfps, op=dist.ReduceOp.SUM)
        stream_e2e = {hs: mine}
        if rank == 0 and world == 1:
            for tag, nm in (("mid", "c3_4k_ra8_mid_65"), ("dense", "c3_4k_ra8_dense_33")):
                if tag in args.streams.split(",") and args.workload == "c3_4k_main10_ra":
                    stream_e2e[nm] = stream_block(nm, ["reference", "b200"], threads_all, local, budget_s=1.5, with_single=False)
            if "modes" in args.streams.split(",") and args.workload == "c3_4k_main10_ra":
                stream_e2e["thread_modes_c3_4k_wpp_ra8_calm_33"] = thread_modes_block("c3_4k_wpp_ra8_calm_33", threads_all, local)
        if float(sfps.item()) > 0:
            b = mine["b200"][f"threads_{best['threads']}"]
            e2e_line = {"value": float(sfps.item()), "unit": UNIT,
                        "h2d_bytes_per_step": int(8 * b.get("h2d_bytes_per_picture", 0)), "d2h_bytes_per_step": int(8 * b.get("d2h_bytes_per_picture", 0)),
                        "mpixels_per_s": float(sfps.item()) * wl["width"] * wl["height"] / 1e6,
                        "what": f"hooked reference decoder (oracle/_ref/decode_b200: CABAC parse on {best['threads']} host frame threads per GPU -- best of {threads_all} and {2 * threads_all} on {threads_all} usable cores --, pixel path on the GPU) on {hs}.hevc: "
                                "Annex-B bytes in, every picture read back to pinned host frames; steady state of one decoder instance (first pass excluded)",
                        "md5_equal_reference_decoder": mine["b200"].get("md5_equal_reference_decoder")}

    if rank == 0:
        line = {"metric": METRIC, "value": fps, "unit": UNIT, "n_gpus": world, "steps": n_mine // 8, "warmup": args.warmup,
                "ms_per_step": ms / (n_mine / 8), "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
                "dtype": "u16" if wl["bit_depth"] > 8 else "u8", "data": "synthetic",
                "config": workload_config(args.workload, wl, world),
                "arm": {"lanes": int(os.environ.get("B200_LANES", "8")), "parallelism": f"frame-parallel x{world}: intra periods (32 pictures) per GPU, one anchor per period sent to the next GPU over NCCL (send/recv)" if world > 1 else "single GPU",
                        "l2": "inputs larger than L2: 9 work lists (%.0f MB) + %d-slot DPB (%.0f MB) cycled" % (sum(b.nbytes for b in blobs) / 1e6, FP.N_SLOTS, FP.N_SLOTS * slot_bytes / 1e6)},
                "mpixels_per_s": fps * wl["width"] * wl["height"] / 1e6,
                "gpu_launches": int(launches), "clocks": clocks,
                "e2e": e2e_line, "e2e_replay": e2e_replay, "stream_e2e": stream_e2e,
                "roofline": roofline, "cpu_baseline": cpu,
                "nccl_p2p_bytes_per_step": int(backend.bcast_bytes / max(1, n_mine / 8)) if world > 1 else 0}
        print(json.dumps(line), file=_REAL_STDOUT, flush=True)
    eng.close()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
