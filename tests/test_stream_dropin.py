"""The real decoder, end to end: committed synthetic Annex-B streams (tools/hevc_stream_gen.py) decoded by
 (a) the UNMODIFIED reference (oracle/_ref/decode_ref -> libohevc_ref.so) and
 (b) the reference carrying the three table hooks + four frame hooks of INTEGRATION.md
     (oracle/_ref/decode_b200 -> libohevc_b200.so -> libb200hevc_shim.so -> GPU),
both through the public libOpenHevc* API, single thread and with frame threads (hevc -p 4 -f 1).  Per-picture plane MD5s must be identical
(BASELINE config 1: 832x480 8-bit, I pictures, bit-exact gate)."""
import glob
import os
import subprocess

import pytest

import oracle_lib

HERE = os.path.dirname(os.path.abspath(__file__))
REFDIR = os.path.join(os.path.dirname(HERE), "oracle", "_ref")
STREAMS = sorted(glob.glob(os.path.join(HERE, "golden", "streams", "*.hevc")))      # run order: tests/conftest.py


def run(binary, stream, threads=1, env=None, want_stderr=False):
    """threads: N = frame threads (hevc -p N -f 1), "Nw" = slice / WPP threads (-f 2)"""
    out = subprocess.run([os.path.join(REFDIR, binary), stream, str(threads)], capture_output=True, text=True, timeout=600,
                         env=dict(os.environ, **(env or {})))
    assert out.returncode == 0, out.stderr[-2000:]
    frames = [l for l in out.stdout.splitlines() if l.startswith("frame ")]
    return (frames, out.stderr) if want_stderr else frames


# streams whose decoding reads s->is_pcm[] (transquant bypass, PCM with the loop filter off): the reference never clears that
# array between pictures (hevc.c:147), so its own output depends on which pictures a context decoded before, i.e. on the
# number of frame threads; the arbiter for such runs is the reference run the same way, not the committed single-thread MD5
IS_PCM_STREAMS = ("tqb_", "pcm_416x240_10b_lfoff", "tskip_416x240_8b", "ccp_416x240_8b_ra")
REPEATED = [s for s in STREAMS if os.path.basename(s).startswith(("b_", "p_", "wpp_416", "tiles_416", "cip_416", "ra_416"))]
WPP_STREAMS = [s for s in STREAMS if os.path.basename(s).startswith(("wpp_", "tiles_"))]      # streams with entry points: slice threads really run


def replay_recorded(stream, threads="1"):
    """without the reference build: the work lists the hooked decoder recorded for this stream with these threads
    (golden/worklists/) on the CUDA path, every stored picture against the committed MD5s"""
    rec = oracle_lib.recorded_worklists(stream, threads)
    if rec is None:
        pytest.skip("oracle/_ref/decode_b200 not built and no recorded work lists stored for this stream")
    want = open(stream[:-5] + ".md5").read().splitlines()
    for k, line in sorted(oracle_lib.replay_worklists(rec, gpu=True).items()):
        assert line == want[k], f"picture {k} differs:\n got {line}\nwant {want[k]}"


def test_streams_committed():
    assert len(STREAMS) >= 3


@pytest.mark.parametrize("stream", STREAMS, ids=[os.path.basename(s) for s in STREAMS])
def test_reference_decoder_reproduces_committed_md5(stream):
    """CPU: the plain reference build still produces the committed hashes (pins the fixtures)"""
    if not os.path.exists(os.path.join(REFDIR, "decode_ref")):
        pytest.skip("oracle/_ref/decode_ref not built")
    want = open(stream[:-5] + ".md5").read().splitlines()
    assert run("decode_ref", stream) == want


@pytest.mark.gpu
@pytest.mark.parametrize("stream", STREAMS, ids=[os.path.basename(s) for s in STREAMS])
def test_hooked_decoder_is_bit_exact_on_the_same_stream(stream):
    if not os.path.exists(os.path.join(REFDIR, "decode_b200")):
        return replay_recorded(stream)
    want = open(stream[:-5] + ".md5").read().splitlines()
    got = run("decode_b200", stream)
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g == w, f"picture differs:\n got {g}\nwant {w}"


@pytest.mark.parametrize("stream", [s for s in STREAMS if "/b_" in s or "/p_" in s], ids=os.path.basename)
def test_reference_decoder_frame_threads(stream):
    """CPU: the reference's frame threading is deterministic on these streams (precondition of the GPU test below)"""
    if not os.path.exists(os.path.join(REFDIR, "decode_ref")):
        pytest.skip("oracle/_ref/decode_ref not built")
    assert run("decode_ref", stream, threads=4) == open(stream[:-5] + ".md5").read().splitlines()


# frame threads on the GPU: one or two streams per feature (every stream runs with 4 frame threads in the CPU suite, recorder ->
# oracle, tests/test_stream_oracle_cpu.py; here every run starts processes and CUDA contexts)
THREADED = [s for s in STREAMS if os.path.basename(s).startswith((
    "b_", "p_", "c3_", "i_416", "wpp_", "cip_416", "ra_", "tiles_832", "slices_416x240_10b", "tqb_416x240_10b", "pcm_416x240_10b", "tskip_416x240_8b",
    "missing_", "c422_832", "c444_416x240_8b", "ccp_", "amp_416", "tmvp_416x240_10b", "calm_416", "qpd_416x240_10b"))]


@pytest.mark.gpu
@pytest.mark.parametrize("stream", THREADED, ids=os.path.basename)
def test_hooked_decoder_with_frame_threads(stream):
    """4 frame threads: thread-local recorders, pictures reach the GPU in decode order through the shim's ticket.
    The arbiter is the unmodified reference run with the same thread count (on streams shorter than the thread
    count its own flush logic, main_hm/main.c:283, drops the delayed pictures -- the drop-in must behave the same)."""
    if not os.path.exists(os.path.join(REFDIR, "decode_b200")) or not os.path.exists(os.path.join(REFDIR, "decode_ref")):
        if os.path.basename(stream).startswith(IS_PCM_STREAMS):
            pytest.skip("oracle/_ref/decode_ref not built: its output with frame threads differs from the committed MD5s on this stream")
        return replay_recorded(stream, "4")
    want = run("decode_ref", stream, threads=4)
    committed = open(stream[:-5] + ".md5").read().splitlines()
    if not os.path.basename(stream).startswith(IS_PCM_STREAMS):
        # (transquant-bypass streams: the reference never clears s->is_pcm between pictures, hevc.c:147, so its own output
        #  depends on the thread count there; the drop-in reads the same array and must follow the reference run the same way)
        assert [l.split()[2:] for l in want] == [l.split()[2:] for l in committed[:len(want)]]
    if "/b_" in stream or "/p_" in stream:
        assert want == committed
    for rep in range(2 if stream in REPEATED else 1):     # a second run catches state left behind by the first (a subset: every run starts a process + CUDA context)
        assert run("decode_b200", stream, threads=4) == want


@pytest.mark.parametrize("stream", WPP_STREAMS, ids=os.path.basename)
def test_reference_decoder_wpp_threads(stream):
    """CPU: entropy_coding_sync streams (one CABAC substream per CTB row + entry points) decode identically with the
    reference's WPP worker threads (hls_slice_data_wpp, hevc.c:3082) -- pins the entry points the generator writes"""
    if not os.path.exists(os.path.join(REFDIR, "decode_ref")):
        pytest.skip("oracle/_ref/decode_ref not built")
    assert len(WPP_STREAMS) >= 3
    # (up to three attempts: the unmodified decoder's slice-threaded pixel path is not race-free -- on 1080p / 4K WPP streams its
    #  output differs from run to run now and then, DESIGN.md 6; one exact run shows that the entry points are right)
    want = open(stream[:-5] + ".md5").read().splitlines()
    assert any(run("decode_ref", stream, threads="4w") == want for _ in range(3))


@pytest.mark.gpu
@pytest.mark.parametrize("stream", WPP_STREAMS, ids=os.path.basename)
def test_hooked_decoder_with_wpp_threads(stream):
    """4 WPP worker threads record ONE picture concurrently into their own recorders; b200_frame_end merges them"""
    if not os.path.exists(os.path.join(REFDIR, "decode_b200")):
        return replay_recorded(stream, "4w")
    want = open(stream[:-5] + ".md5").read().splitlines()
    for rep in range(2 if stream in REPEATED else 1):
        assert run("decode_b200", stream, threads="4w") == want


@pytest.mark.gpu
@pytest.mark.parametrize("stream", [s for s in STREAMS if os.path.exists(s[:-5] + ".gen.txt")], ids=os.path.basename)
@pytest.mark.parametrize("threads", [1, "4w"])
def test_table_calls_equal_what_the_generator_wrote(stream, threads):
    """B200_SHIM_STATS: the table calls the decoder made per picture == the syntax elements the generator wrote
    (the decoder parses the stream as written, also when the calls come from worker threads)"""
    import re
    if not os.path.exists(os.path.join(REFDIR, "decode_b200")):
        pytest.skip("oracle/_ref/decode_b200 not built")
    if threads != 1 and stream not in WPP_STREAMS:
        pytest.skip("no entry points: slice threads fall back to one thread")
    if stream not in REPEATED:
        pytest.skip("the same check runs for every stream in the CPU suite (tests/test_stream_oracle_cpu.py, record-only shim)")
    gen = [tuple(int(v) for v in m.groups()) for m in re.finditer(r"intra_pred (\d+) transform_add (\d+) prediction units (\d+)", open(stream[:-5] + ".gen.txt").read())]
    _, err = run("decode_b200", stream, threads=threads, env={"B200_SHIM_STATS": "1"}, want_stderr=True)
    got = [tuple(int(v) for v in m.groups()) for m in re.finditer(r"b200 picture \d+: intra_pred (\d+) transform_add (\d+) mc (\d+)", err)]
    assert len(got) == len(gen)
    for (gi, gt, gm), (wi, wt, wp) in zip(got, gen):
        assert (gi, gt) == (wi, wt) and gm == 3 * wp


# ---- BASELINE.json configs at their stated shape (SURVEY.md 8d: >= 64 pictures, random access GOP 8): RECIPES, not committed bytes --
# tools/make_bench_streams.sh regenerates the streams (fixed seeds) into oracle/_ref/streams/ and pins each with the per-picture
# MD5s of the unmodified decoder (decode_ref, one thread); __graft_entry__.build() runs it when the files are missing.
RECIPE_DIR = os.path.join(REFDIR, "streams")
RECIPES = ["c1_832x480_i_16", "c2_1080p_ra8_65", "c2_1080p_wpp_ra8_33", "c3_4k_ra8_calm_65", "c3_4k_ra8_mid_65", "c3_4k_ra8_dense_33", "c5_8k_422_wpp_tiles_9"]


@pytest.mark.gpu
@pytest.mark.parametrize("threads", [1, 8])
@pytest.mark.parametrize("name", RECIPES)
def test_baseline_shape_streams_are_bit_exact(name, threads):
    """832x480 all-intra (config 1), 1920x1080 8-bit and 3840x2160 Main10 random access, GOP 8, intra period 32, 65 pictures
    (configs 2-4; lightly, moderately and densely coded), 7680x4320 4:2:2 Main10 with WPP inside 4x2 tiles (config 5): the hooked
    decoder, 1 thread and 8 frame threads, every picture against the MD5s of the unmodified decoder.  (Config 5 runs without
    slice threads: the reference's own -f 2 path is not deterministic on WPP-in-tiles streams here -- decode_ref 4w differs from
    run to run and can hang -- so there is nothing to compare a threaded run with.)"""
    stream, md5 = os.path.join(RECIPE_DIR, name + ".hevc"), os.path.join(RECIPE_DIR, name + ".md5")
    if not (os.path.exists(stream) and os.path.exists(md5) and os.path.exists(os.path.join(REFDIR, "decode_b200"))):
        pytest.skip("recipe stream not generated (tools/make_bench_streams.sh)")
    if threads == 8 and name in ("c1_832x480_i_16", "c5_8k_422_wpp_tiles_9"):
        pytest.skip("fewer pictures than delayed frames: the reference's flush logic (main_hm/main.c:283) drops pictures with that many threads")
    assert run("decode_b200", stream, threads) == open(md5).read().splitlines()


@pytest.mark.gpu
@pytest.mark.parametrize("threads", ["4w", "2x", "4x"])
def test_frame_threads_with_slice_threads_inside_are_bit_exact(threads):
    """VERDICT r1 item 9, hevc -f 4 (libavcodec/pthread.c:57-71: N slice threads per picture, cpus / N + 1 frame threads): several
    pictures are in progress at once and every one of them is recorded by several WPP workers.  A table call carries no context,
    so the execute2 jobs announce the picture they work for (b200_worker_begin, hevc.c:2764 / 2847 / 2931); b200_frame_end folds
    the workers' lists into their picture's.  1920x1080 WPP stream, hierarchical-B GOP 8, 33 pictures; "4w" = slice threads only."""
    stream, md5 = os.path.join(RECIPE_DIR, "c2_1080p_wpp_ra8_33.hevc"), os.path.join(RECIPE_DIR, "c2_1080p_wpp_ra8_33.md5")
    if not (os.path.exists(stream) and os.path.exists(md5) and os.path.exists(os.path.join(REFDIR, "decode_b200"))):
        pytest.skip("recipe stream not generated (tools/make_bench_streams.sh)")
    assert run("decode_b200", stream, threads) == open(md5).read().splitlines()
    # the same at 3840x2160 Main10.  (The arbiter is the SINGLE-threaded reference: on this stream the unmodified decoder's own -f 2 /
    # -f 4 runs come out different from run to run -- 6 to 20 of 33 pictures wrong, a race in its host pixel path between WPP rows and
    # frame-thread progress -- while the drop-in, whose pixels are made on the device in decode order, is exact in every mode.)
    stream, md5 = os.path.join(RECIPE_DIR, "c3_4k_wpp_ra8_calm_33.hevc"), os.path.join(RECIPE_DIR, "c3_4k_wpp_ra8_calm_33.md5")
    if os.path.exists(stream) and os.path.exists(md5):
        assert run("decode_b200", stream, threads) == open(md5).read().splitlines()


@pytest.mark.gpu
@pytest.mark.parametrize("threads", ["1", "4", "2x"])
def test_two_decoders_in_one_process(threads):
    """VERDICT r1 item 9: two decoder instances open at once in one process, fed alternately from one thread, then the first is
    closed and a third opened on its stream (oracle/decode_two.c).  The shim keeps a device context, a submission thread and a ticket
    order per instance; hevc_decode_free gives them back (b200_decoder_close)."""
    binary = os.path.join(REFDIR, "decode_two_b200")
    if not os.path.exists(binary):
        pytest.skip("oracle/_ref/decode_two_b200 not built")
    # (streams longer than the frame-thread count, which for "2x" is cpus / 2 + 1, at most 16: the reference's flush logic drops
    #  pictures of shorter ones, main_hm/main.c:283)
    if threads == "2x":
        a, b = os.path.join(RECIPE_DIR, "c2_1080p_wpp_ra8_33"), os.path.join(RECIPE_DIR, "c2_1080p_ra8_65")
    else:
        a, b = os.path.join(RECIPE_DIR, "c2_1080p_ra8_65"), os.path.join(HERE, "golden", "streams", "ra_416x240_8b")
    if not (os.path.exists(a + ".hevc") and os.path.exists(a + ".md5") and os.path.exists(b + ".md5")):
        pytest.skip("recipe stream not generated (tools/make_bench_streams.sh)")
    out = subprocess.run([binary, a + ".hevc", b + ".hevc", threads], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-2000:]
    for tag, name in (("A", a), ("B", b), ("C", a)):
        got = [l[2:] for l in out.stdout.splitlines() if l.startswith(tag + " frame ")]
        assert got == open(name + ".md5").read().splitlines(), f"decoder {tag} ({os.path.basename(name)})"


@pytest.mark.gpu
@pytest.mark.parametrize("env", [{"B200_DBD": "0"}, {"B200_DBD": "2"}], ids=lambda e: ",".join(f"{k}={v}" for k, v in e.items()))
def test_switchable_paths_are_bit_exact_on_a_random_access_stream(env):
    """the paths behind environment switches, on the device: deblocking control recorded from the reference's own filter calls
    (B200_DBD=0) and derived AND compared on the device (B200_DBD=2) -- 1920x1080 random access, 65 pictures, 4 frame threads"""
    stream, md5 = os.path.join(RECIPE_DIR, "c2_1080p_ra8_65.hevc"), os.path.join(RECIPE_DIR, "c2_1080p_ra8_65.md5")
    if not (os.path.exists(stream) and os.path.exists(md5) and os.path.exists(os.path.join(REFDIR, "decode_b200"))):
        pytest.skip("recipe stream not generated (tools/make_bench_streams.sh)")
    frames, err = run("decode_b200", stream, 4, env=env, want_stderr=True)
    assert "Error" not in err, err[-1500:]
    assert frames == open(md5).read().splitlines()
