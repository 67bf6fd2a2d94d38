#!/usr/bin/env python
"""Generates the committed golden fixtures: small synthetic pictures executed by the UNMODIFIED reference's own C
functions (oracle/_ref/libohevc_ref.so through oracle/replay_ref.c).  Run in the build container (needs /root/reference
to have been compiled by oracle/build_ref.sh):  python tests/golden/make_golden.py
Each fixture = the work-list blob, the DPB contents it reads (generator seeds) and the reconstructed picture;
worklists/<stream>.npz.xz = work lists the hooked decoder (oracle/_ref/decode_b200, record only) wrote for a committed stream."""
import glob
import io
import lzma
import os
import subprocess
import sys
import tempfile
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import oracle_lib  # noqa: E402
from openhevc_b200.synth import FrameSynth, smooth_frame  # noqa: E402

CASES = [  # name, w, h, cfi, bd, refs, kwargs
    ("i_420_8", 128, 64, 1, 8, [], dict(exotic=0.05)),
    ("b_420_10_weighted", 192, 128, 1, 10, [1, 2], dict(weighted=True, max_mv=100)),
    ("b_422_10", 128, 128, 2, 10, [1, 2], dict(sao_restore=True)),
    ("p_444_8", 128, 64, 3, 8, [2], dict(exotic=0.05)),
    ("b_420_12", 128, 64, 1, 12, [1, 2], {}),
]
# compressed bytes of work lists kept per stream (at least one picture).  The lists are this project's wire format
# (include/b200hevc_worklist.h) as the recorder writes it: a change to either needs worklists() run again.
WORKLIST_CAP = 60_000


def main():
    assert oracle_lib.ref_lib() is not None, "reference build missing"
    for name, w, h, cfi, bd, refs, kw in CASES:
        blob, _ = FrameSynth(w, h, cfi, bd, seed=sum(map(ord, name)), refs=refs, cur_slot=0, **kw).generate()
        dpb = [smooth_frame(w, h, cfi, bd, 900 + k) for k in range(3)]
        out = oracle_lib.ref_execute(blob, dpb)
        np.savez_compressed(os.path.join(HERE, name + ".npz"), blob=blob, geom=np.array([w, h, cfi, bd]), dpb_seeds=np.array([900, 901, 902]),
                            y=out[0], cb=out[1], cr=out[2])
        print(name, os.path.getsize(os.path.join(HERE, name + ".npz")))
    worklists()
    dropin()


def dropin():
    """tests/test_dropin_gpu.py: MD5s of the pictures the reference's own tables make from its cases"""
    import test_dropin_gpu as T
    from openhevc_b200 import worklist as W
    with open(T.REFERENCE_MD5, "w") as f:
        for c in T.CASES:
            blob, dpb = T.case(*c)
            f.write(oracle_lib.md5_line(0, W.parse_blob(blob)[0], oracle_lib.ref_execute(blob, dpb)) + "\n")


def dump(stream, threads, d):
    subprocess.run([os.path.join(oracle_lib.ORACLE_DIR, "_ref", "decode_b200"), stream, threads, "quiet"], check=True, capture_output=True,
                   env=dict(os.environ, B200_SHIM_DUMP=d))
    return [np.fromfile(p, np.uint8) for p in sorted(glob.glob(os.path.join(d, "pic_*.blob")))]


def worklists():
    """work lists of the first pictures of every committed stream (and with the threads test_stream_dropin.py uses), packed < 1 MB"""
    import test_stream_dropin as T
    from openhevc_b200 import worklist as W
    os.makedirs(os.path.join(HERE, "worklists"), exist_ok=True)
    packs = [[]]
    for stream in sorted(glob.glob(os.path.join(HERE, "streams", "*.hevc"))):
        for threads in ("1", "4", "4w"):
            if (threads == "4" and (stream not in T.THREADED or os.path.basename(stream).startswith(T.IS_PCM_STREAMS))) or \
                    (threads == "4w" and stream not in T.WPP_STREAMS):
                continue
            name, data = os.path.basename(stream)[:-5] + {"1": "", "4": ".f4", "4w": ".w4"}[threads] + ".npz.xz", worklist_file(stream, threads, W)
            if len(data) >= 1 << 20:
                continue                           # the 4K stream: one picture is too large
            if sum(len(d) for _, d in packs[-1]) + len(data) > 980_000:
                packs.append([])
            packs[-1].append((name, data))
    for i, group in enumerate(packs):
        with zipfile.ZipFile(os.path.join(HERE, "worklists", f"pack_{i:02d}.zip"), "w", zipfile.ZIP_STORED) as z:
            for name, data in group:
                z.writestr(name, data)


def worklist_file(stream, threads, W):
    n_md5 = len(open(stream[:-5] + ".md5").read().splitlines())
    with tempfile.TemporaryDirectory() as d:
        blobs = dump(stream, threads, d)
        fills = []
        for k, p in enumerate(sorted(glob.glob(os.path.join(d, "pic_*.blob")))):
            if os.path.exists(p[:-5] + ".fill"):
                fills += [(k, *[int(v) for v in line.split()]) for line in open(p[:-5] + ".fill")]
    order, cvs = [], -1                         # output order: by coded video sequence (a new one at every POC 0), then by POC
    for b in blobs:
        poc = int(W.parse_blob(b)[0]["poc"])
        cvs += poc == 0
        order.append((cvs, poc))
    out_idx = [sorted(order).index(o) for o in order]
    keep, size = 0, 0                          # pictures whose work lists fit WORKLIST_CAP (compressed one by one: an estimate)
    for k in range(len(blobs)):
        size += len(lzma.compress(blobs[k].tobytes(), preset=6))
        if out_idx[k] >= n_md5 or (keep and size > WORKLIST_CAP):
            break
        keep = k + 1
    buf = io.BytesIO()
    np.savez(buf, blob=np.concatenate(blobs[:keep]), off=np.cumsum([0] + [len(b) for b in blobs[:keep]]), out_idx=np.array(out_idx[:keep]),
             fills=np.array([f for f in fills if f[0] < keep], np.int64).reshape(-1, 3))
    return lzma.compress(buf.getvalue(), preset=9 | lzma.PRESET_EXTREME)


if __name__ == "__main__":
    main()
