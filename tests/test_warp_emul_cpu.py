"""CPU suite: the CUDA kernels' own source on the CPU.

tests/emul/ compiles openhevc_b200/csrc/kernels.cu + engine.cu + recorder.cpp UNCHANGED with g++ against a stand-in
<cuda_runtime.h> (tests/emul/warp/): every CUDA thread is a fiber, the lanes of a warp meet in lock-step at each
__shfl_*_sync / __syncwarp / vote / __syncthreads, kernel launches, copies and events complete at once.  The result,
oracle/_ref/libb200hevc_emul.so, has the C ABI of libb200hevc.so.  These tests load it IN PLACE of the CUDA library -- only
here, the product never does -- and run

 * the GPU parity and limits tests (tests/test_parity_gpu.py, tests/test_*_limits_gpu.py; same functions, same seeds)
   against the oracle, and
 * the real decoder with the B200 hooks on the committed streams (decode_b200, the emulated library pre-loaded) against
   the MD5s of the unmodified reference decoder,

so a kernel or engine change is checked bit-exactly before a GPU is spent on it.  Not shown by this: memory-model races,
stream / event ordering, anything about speed -- that stays with `-m gpu`."""
import glob
import os
import subprocess
import sys

import pytest

import oracle_lib
import test_loop_filter_limits_gpu as LF
import test_mc_limits_gpu as MC
import test_residual_intra_limits_gpu as RI

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REFDIR = os.path.join(ROOT, "oracle", "_ref")
EMUL = os.path.join(REFDIR, "libb200hevc_emul.so")
STREAMS = sorted(glob.glob(os.path.join(HERE, "golden", "streams", "*.hevc")))
SMALL = [s for s in STREAMS if "416x240" in s or "256x128" in s]
# one stream per feature through the emulated device (every stream runs through the CPU oracle in tests/test_stream_oracle_cpu.py)
EMULATED = [s for s in SMALL if os.path.basename(s).startswith((
    "amp_416", "b_", "bd12_", "c422_416", "c444_416x240_8b", "calm_416", "ccp_", "cip_416x240_8b", "dbkoff_", "i_256", "missing_", "nodbk_", "nofilter_",
    "p_", "pcm_416x240_10b", "qpd_416x240_8b", "ra_416", "saochroma_", "saoluma_", "slices_416x240_10b", "tiles_416x240_10b", "tmvp_416x240_10b",
    "tqb_416x240_10b", "tskip_416x240_8b", "wpp_416"))]

needs_emul = pytest.mark.skipif(not os.path.exists(EMUL), reason="oracle/_ref/libb200hevc_emul.so not built (make -C tests/emul)")


@pytest.fixture
def emulated(monkeypatch):
    """FrameEngine loads the emulated library instead of libb200hevc.so for the duration of one test"""
    from openhevc_b200 import _lib
    monkeypatch.setattr(_lib, "LIB_PATH", EMUL)
    return True


@needs_emul
def test_emulated_library_has_the_product_abi():
    import ctypes
    from openhevc_b200 import _lib
    lib = ctypes.CDLL(EMUL)
    for name in _lib.EXPORTS:
        assert hasattr(lib, name), name


PARITY = ["test_weighted_prediction_and_sao_restore", "test_constrained_intra_pred", "test_sao_restore_of_bypass_pus", "test_intra_only_small_blocks",
          "test_stages_individually", "test_far_out_of_picture_motion", "test_pcm_and_exotic_transform_paths", "test_malformed_blobs_are_rejected_not_executed",
          "test_malformed_inter_records_are_rejected_on_the_device", "test_empty_work_list_and_smallest_pictures"]
# tests/test_mc_limits_gpu.py: inter prediction at the limits of its input space, and block-form lists that leave tiles unwritten
MC_LIMITS = ["test_mc_block_with_tiles_in_two_buckets", "test_small_tile_region_need_not_be_bucket_ordered", "test_malformed_block_lists_are_rejected_on_the_device"]


@needs_emul
@pytest.mark.parametrize("name", PARITY)
def test_gpu_parity_test_on_the_emulated_kernels(emulated, name):
    import test_parity_gpu
    getattr(test_parity_gpu, name)()


@needs_emul
@pytest.mark.parametrize("name", MC_LIMITS)
def test_mc_limits_on_the_emulated_kernels(emulated, name):
    import test_mc_limits_gpu
    getattr(test_mc_limits_gpu, name)()


# the cases of the limits files on synthetic pictures and random grids (K1, K3's constrained-intra rules, K4, K5), every
# parameter set the GPU run takes
LIMITS = [(LF, "test_sao_limits", LF.SAO_CASES), (LF, "test_deblock_limits", LF.DBK_CASES), (LF, "test_sao_restore_limits", LF.RESTORE_CASES),
          (RI, "test_constrained_intra_rules", RI.CIP_CASES), (MC, "test_mc_synthetic_pictures", MC.MC_CASES)]


@needs_emul
@pytest.mark.parametrize("module,name,args", [pytest.param(m, n, a, id=f"{n}-{a}".replace(" ", "")) for m, n, cases in LIMITS for a in cases])
def test_limits_case_on_the_emulated_kernels(emulated, module, name, args):
    getattr(module, name)(*args)


@needs_emul
@pytest.mark.parametrize("cfi,bd", [(1, 8), (1, 10), (1, 12), (2, 10), (3, 8)])
def test_mc_limits_sweep_on_the_emulated_kernels(emulated, cfi, bd):
    import test_mc_limits_gpu
    test_mc_limits_gpu.test_mc_sweep(cfi, bd)


@needs_emul
@pytest.mark.parametrize("w,h,cfi,bd", [(16, 16, 1, 8), (72, 40, 1, 10), (24, 40, 2, 10), (40, 24, 3, 8)])
def test_mc_limits_small_pictures_on_the_emulated_kernels(emulated, w, h, cfi, bd):
    import test_mc_limits_gpu
    test_mc_limits_gpu.test_mc_sweep_small_pictures(w, h, cfi, bd)


@needs_emul
@pytest.mark.parametrize("cfi,bd", [(1, 8), (1, 10), (1, 12), (2, 10), (3, 8)])
def test_residual_limits_sweep_on_the_emulated_kernels(emulated, cfi, bd):
    """tests/test_residual_intra_limits_gpu.py: the residual sweep with impulses at every 37th coefficient position (the
    GPU run takes every position)"""
    import test_residual_intra_limits_gpu as T
    T.run_residual_sweep((256, 128, cfi, bd), seed=10 * cfi + bd, impulse_step=37)


@needs_emul
@pytest.mark.parametrize("cfi,bd", [(1, 8), (1, 10), (1, 12), (2, 10), (3, 8)])
def test_intra_limits_sweep_on_the_emulated_kernels(emulated, cfi, bd):
    import test_residual_intra_limits_gpu as T
    T.test_intra_sweep(cfi, bd)


@needs_emul
@pytest.mark.parametrize("name", ["test_residual_sweep_small_pictures", "test_intra_sweep_small_pictures", "test_intra_dense_zorder"])
def test_residual_intra_limits_small_and_dense_on_the_emulated_kernels(emulated, name):
    """one of the three geometries the GPU run takes for each (the residual sweep with impulses at every 37th position)"""
    import test_residual_intra_limits_gpu as T
    if name == "test_residual_sweep_small_pictures":
        T.run_residual_sweep((72, 40, 1, 10), seed=1, impulse_step=37)
    else:
        getattr(T, name)(*{"test_intra_sweep_small_pictures": (24, 40, 2, 12), "test_intra_dense_zorder": (72, 40, 2, 10)}[name])


@needs_emul
def test_rdpcm_rejection_on_the_emulated_kernels(emulated):
    import test_residual_intra_limits_gpu as T
    T.test_rdpcm_on_transformed_or_pcm_blocks_is_rejected()


@needs_emul
@pytest.mark.parametrize("w,h,cfi,bd", [(256, 128, 1, 8), (256, 128, 1, 10), (192, 128, 2, 10), (192, 128, 3, 8), (320, 192, 1, 12)])
def test_sequence_all_stages_on_the_emulated_kernels(emulated, w, h, cfi, bd):
    import test_parity_gpu
    test_parity_gpu.test_sequence_all_stages(w, h, cfi, bd)


@needs_emul
@pytest.mark.parametrize("bd", [8, 10])
def test_cross_component_prediction_on_the_emulated_kernels(emulated, bd):
    import test_parity_gpu
    test_parity_gpu.test_cross_component_prediction(bd)


@needs_emul
@pytest.mark.parametrize("cfi,bd", [(1, 8), (2, 10)])
def test_grey_reference_fill_on_the_emulated_kernels(emulated, cfi, bd):
    import test_parity_gpu
    test_parity_gpu.test_grey_reference_fill(cfi, bd)


@needs_emul
def test_golden_fixtures_on_the_emulated_kernels(emulated):
    import test_golden
    for path in test_golden.FIXTURES:
        test_golden.test_cuda_reproduces_reference_golden(path)


# environment switches (read once per process, hence a child process each): one compute lane, and other lane orders of the
# emulator.  B200_EMUL_ORDER changes the order in which the emulator runs the lanes between two collectives (reverse / shuffled):
# a kernel that needs a barrier it does not have passes in one order and fails in another.
VARIANTS = [dict(B200_EMUL_ORDER="reverse"), dict(B200_EMUL_ORDER="random:7"), dict(B200_EMUL_ORDER="random:3"), dict(B200_LANES="1")]


@needs_emul
@pytest.mark.parametrize("env", VARIANTS, ids=lambda e: ",".join(f"{k}={v}" for k, v in e.items()))
def test_switch_variants_on_the_emulated_kernels(env):
    code = ("import sys; sys.path[:0] = [%r, %r]\n"
            "from openhevc_b200 import _lib; _lib.LIB_PATH = %r\n"
            "import test_parity_gpu as T\n"
            "T.run_sequence(256, 128, 1, 10, seeds=[11, 12, 13], exotic=0.04)\n"
            "T.run_sequence(192, 128, 2, 8, seeds=[14, 15], p_intra=0.05)\n"
            "T.run_sequence(192, 128, 1, 8, seeds=[16, 17, 18], weighted=True)\n" % (ROOT, HERE, EMUL))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900, env=dict(os.environ, **env))
    assert r.returncode == 0, r.stderr[-3000:]


@needs_emul
def test_intra_limits_sweep_in_reverse_lane_order():
    """the intra sweep with the emulator running the lanes between two collectives in reverse order"""
    code = ("import sys; sys.path[:0] = [%r, %r]\n"
            "from openhevc_b200 import _lib; _lib.LIB_PATH = %r\n"
            "import test_residual_intra_limits_gpu as R\n"
            "R.test_intra_sweep(1, 10)\n"
            "R.test_intra_dense_zorder(72, 40, 2, 10)\n" % (ROOT, HERE, EMUL))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900, env=dict(os.environ, B200_EMUL_ORDER="reverse"))
    assert r.returncode == 0, r.stderr[-3000:]


@needs_emul
def test_smoke_on_the_emulated_kernels(emulated, capsys):
    import __graft_entry__
    __graft_entry__.smoke()
    assert "smoke ok" in capsys.readouterr().out


def test_address_sanitizer_sees_no_out_of_bounds_access_in_the_kernels():
    """the emulated library built with -fsanitize=address: device allocations are exact-size heap blocks and shared memory is
    static storage, so a kernel reading or writing one element too far -- which a GPU run forgives silently -- aborts here.
    Includes the malformed work lists that the device-side validation must reject before any kernel trusts them."""
    asan_lib = os.path.join(REFDIR, "libb200hevc_emul_asan.so")
    rt = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.exists(asan_lib) or not os.path.isabs(rt) or not os.path.exists(rt):
        pytest.skip("no address sanitizer build / runtime")
    code = ("import sys; sys.path[:0] = [%r, %r]\n"
            "from openhevc_b200 import _lib; _lib.LIB_PATH = %r\n"
            "import test_parity_gpu as T\n"
            "T.run_sequence(256, 128, 1, 10, seeds=[11, 12, 13], exotic=0.04)\n"
            "T.run_sequence(192, 128, 2, 8, seeds=[66, 67], cip=True, p_intra=0.5)\n"
            "T.test_far_out_of_picture_motion()\n"
            "T.test_malformed_blobs_are_rejected_not_executed()\n"
            "T.test_malformed_inter_records_are_rejected_on_the_device()\n"
            "import test_mc_limits_gpu as M\n"
            "M.test_malformed_block_lists_are_rejected_on_the_device()\n"
            "M.test_mc_sweep(1, 10)\n"
            "import test_residual_intra_limits_gpu as R\n"
            "R.test_rdpcm_on_transformed_or_pcm_blocks_is_rejected()\n"
            "R.test_intra_sweep(1, 12)\n" % (ROOT, HERE, asan_lib))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=1800,
                       env=dict(os.environ, LD_PRELOAD=rt, ASAN_OPTIONS="detect_leaks=0:detect_stack_use_after_return=0"))
    assert r.returncode == 0 and "ERROR: AddressSanitizer" not in r.stderr, r.stderr[-4000:]


@pytest.mark.parametrize("stream", [s for s in SMALL if os.path.basename(s).startswith(("b_416", "cip_416x240_8b", "tqb_416x240_10b", "c422_416", "ccp_416x240_8b"))], ids=os.path.basename)
def test_thread_sanitizer_sees_no_data_race_in_the_kernels(stream):
    """the emulated library built with -fsanitize=thread: every CUDA thread is a TSan fiber, and the only happens-before edges
    are the ones the CUDA model gives -- a completed warp collective among its participants, __syncthreads in the block, block
    and kernel boundaries.  Two lanes touching the same shared-memory or global word without such an edge in between is a
    reported race (what compute-sanitizer racecheck looks for; a removed __syncwarp gives eight reports on one P picture).
    Real decoder, hooks, emulated device: pictures must still be right, and the sanitizer must stay silent."""
    tsan_lib = os.path.join(REFDIR, "libb200hevc_emul_tsan.so")
    rt = subprocess.run(["gcc", "-print-file-name=libtsan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.exists(tsan_lib) or not os.path.isabs(rt) or not os.path.exists(rt) or not os.path.exists(os.path.join(REFDIR, "decode_b200")):
        pytest.skip("no thread sanitizer build / runtime / hooked decoder")
    out = subprocess.run([os.path.join(REFDIR, "decode_b200"), stream, "1"], capture_output=True, text=True, timeout=1800,
                         env=dict(os.environ, LD_PRELOAD=rt + " " + tsan_lib, TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0"))
    if "FATAL: ThreadSanitizer" in out.stderr and "unexpected memory mapping" in out.stderr:
        pytest.skip("thread sanitizer cannot map its shadow memory in this environment")
    assert "WARNING: ThreadSanitizer" not in out.stderr, out.stderr[:6000]
    assert out.returncode == 0, out.stderr[-2000:]
    assert [l for l in out.stdout.splitlines() if l.startswith("frame ")] == open(stream[:-5] + ".md5").read().splitlines()


def decode_emulated(stream, threads):
    out = subprocess.run([os.path.join(REFDIR, "decode_b200"), stream, threads], capture_output=True, text=True, timeout=900,
                         env=dict(os.environ, LD_PRELOAD=EMUL))
    assert out.returncode == 0, out.stderr[-2000:]
    return [l for l in out.stdout.splitlines() if l.startswith("frame ")]


@needs_emul
@pytest.mark.parametrize("stream", EMULATED, ids=os.path.basename)
def test_hooked_decoder_on_the_emulated_kernels(stream):
    """real decoder -> shim -> recorder -> engine -> emulated K0..K5 -> read-back == unmodified reference decoder"""
    if not os.path.exists(os.path.join(REFDIR, "decode_b200")):
        pytest.skip("oracle/_ref/decode_b200 not built (needs /root/reference)")
    want = open(stream[:-5] + ".md5").read().splitlines()
    assert decode_emulated(stream, "1") == want
    if os.path.basename(stream).startswith(("wpp_416", "tiles_832")):
        # frame threads whose pictures are decoded by slice threads (hevc -f 4, pthread.c:57-71): several pictures in progress, each
        # recorded by several workers that b200_worker_begin attaches to the right one
        assert decode_emulated(stream, "2x") == want


@needs_emul
@pytest.mark.parametrize("threads", ["1", "4", "2x"])
def test_two_decoders_in_one_process_on_the_emulated_kernels(threads):
    """VERDICT r1 item 9: the shim's state is per decoder instance (device context, submission thread, ticket order, read-back
    table), found through the context every hook is handed.  oracle/decode_two.c opens two decoders, feeds them alternately from
    one thread, closes the first and opens a third on the same stream (hevc_decode_free -> b200_decoder_close gives the instance
    back); every picture of all three must equal the unmodified single decoder's.  "4": frame threads, "2x": frame threads with two
    slice threads each on WPP / tile streams."""
    binary = os.path.join(REFDIR, "decode_two_b200")
    if not os.path.exists(binary):
        pytest.skip("oracle/_ref/decode_two_b200 not built (needs /root/reference)")
    gold = os.path.join(HERE, "golden", "streams")
    a, b = ("wpp_416x240_8b_lowdelay", "tiles_832x480_8b_lowdelay") if threads == "2x" else ("b_416x240_10b_weighted", "ra_416x240_8b")
    args = [os.path.join(gold, a + ".hevc"), os.path.join(gold, b + ".hevc"), threads]
    out = subprocess.run([binary] + args, capture_output=True, text=True, timeout=900, env=dict(os.environ, LD_PRELOAD=EMUL))
    assert out.returncode == 0, out.stderr[-2000:]
    # the arbiter: the unmodified decoder driven the same way (with more frame threads than pictures -- "2x" means cpus / 2 + 1 of
    # them -- its flush logic drops pictures, main_hm/main.c:283, and the drop-in must do the same); where it outputs everything,
    # that equals the committed single-decoder MD5s
    ref = subprocess.run([os.path.join(REFDIR, "decode_two_ref")] + args, capture_output=True, text=True, timeout=900)
    assert ref.returncode == 0
    for tag, name in (("A", a), ("B", b), ("C", a)):
        got = [l[2:] for l in out.stdout.splitlines() if l.startswith(tag + " frame ")]
        want = [l[2:] for l in ref.stdout.splitlines() if l.startswith(tag + " frame ")]
        committed = open(os.path.join(gold, name + ".md5")).read().splitlines()
        # (where the reference outputs every picture the committed single-decoder MD5s are the arbiter: its own slice-threaded runs
        #  are not race-free in the host pixel path)
        assert got == (committed if len(want) == len(committed) else want), f"decoder {tag} ({name})"
    assert any(l.startswith("A frame ") for l in out.stdout.splitlines())


# the streams that stress the deblocking control: QP deltas, beta / tc and chroma QP offsets, PCM with the loop filter off,
# transquant bypass, slices / tiles without filtering across, asymmetric partitions, 4:2:2 / 4:4:4 chroma edge spacing, B pictures
DBD_CHECKED = [s for s in EMULATED if os.path.basename(s).startswith(("amp_", "b_", "c422_", "c444_", "dbkoff_", "pcm_", "qpd_", "ra_416", "slices_", "tiles_", "tqb_"))]


@needs_emul
@pytest.mark.parametrize("stream", DBD_CHECKED, ids=os.path.basename)
def test_device_derived_deblocking_parameters_equal_the_recorded_ones(stream):
    """SURVEY.md 8f N2.  By default the device derives boundary strengths, tc and beta itself (k_dbd.cuh) and the two host
    functions that do it in the reference return at once; with B200_DBD=2 the reference derives them as well, its filter calls
    are recorded, and the device compares its grid with the recorded one entry by entry (k_dbd_compare -> an error from the
    decoder).  Pictures must also still equal the unmodified decoder's."""
    if not os.path.exists(os.path.join(REFDIR, "decode_b200")):
        pytest.skip("oracle/_ref/decode_b200 not built (needs /root/reference)")
    out = subprocess.run([os.path.join(REFDIR, "decode_b200"), stream, "1"], capture_output=True, text=True, timeout=900, env=dict(os.environ, LD_PRELOAD=EMUL, B200_DBD="2"))
    assert out.returncode == 0 and "Error" not in out.stderr, out.stderr[-2000:]
    assert [l for l in out.stdout.splitlines() if l.startswith("frame ")] == open(stream[:-5] + ".md5").read().splitlines()


@needs_emul
def test_the_check_mode_catches_a_wrong_derivation():
    """the same with a library whose derivation is deliberately wrong in a few entries (tests/emul/Makefile, -DB200_DBD_FAULT):
    the comparison must fail loudly, i.e. the check above has teeth"""
    fault = os.path.join(REFDIR, "libb200hevc_emul_fault.so")
    if not os.path.exists(fault) or not os.path.exists(os.path.join(REFDIR, "decode_b200")):
        pytest.skip("fault-injection build missing")
    stream = os.path.join(HERE, "golden", "streams", "p_416x240_8b.hevc")
    out = subprocess.run([os.path.join(REFDIR, "decode_b200"), stream, "1"], capture_output=True, text=True, timeout=900, env=dict(os.environ, LD_PRELOAD=fault, B200_DBD="2"))
    assert "Error" in out.stderr
    out = subprocess.run([os.path.join(REFDIR, "decode_b200"), stream, "1"], capture_output=True, text=True, timeout=900, env=dict(os.environ, LD_PRELOAD=fault, B200_DBD="0"))
    assert "Error" not in out.stderr                      # the fault only sits in the derivation
    assert [l for l in out.stdout.splitlines() if l.startswith("frame ")] == open(stream[:-5] + ".md5").read().splitlines()


@needs_emul
@pytest.mark.parametrize("stream", [s for s in SMALL if os.path.basename(s).startswith(("b_", "ra_416", "wpp_416", "tiles_416x240_10b", "cip_416"))], ids=os.path.basename)
@pytest.mark.parametrize("threads", ["4", "4w"])
def test_hooked_decoder_with_threads_on_the_emulated_kernels(stream, threads):
    if not os.path.exists(os.path.join(REFDIR, "decode_b200")):
        pytest.skip("oracle/_ref/decode_b200 not built (needs /root/reference)")
    if threads == "4w" and not os.path.basename(stream).startswith(("wpp_", "tiles_")):
        pytest.skip("no entry points: slice threads fall back to one thread")
    ref = subprocess.run([os.path.join(REFDIR, "decode_ref"), stream, threads], capture_output=True, text=True, timeout=600)
    want = [l for l in ref.stdout.splitlines() if l.startswith("frame ")]
    if not want:
        pytest.skip("the reference outputs no picture of this stream with that many threads")
    assert decode_emulated(stream, threads) == want


@needs_emul
def test_tables_through_shim_on_the_emulated_kernels():
    """tests/test_dropin_gpu.py's comparison (reference call sequence through the reference's C tables vs through the shim) with the
    emulated device behind the shim; child process, the emulated library pre-loaded"""
    if oracle_lib.ref_lib() is None or not os.path.exists(oracle_lib.SHIM_SO):
        pytest.skip("prebuilt oracle/_ref/libreplay_ref.so or libb200hevc_shim.so missing")
    code = ("import sys; sys.path[:0] = [%r, %r]\n"
            "import test_dropin_gpu as T\n"
            "T.test_tables_through_shim_equal_reference_tables(256, 128, 1, 10, [1, 2], dict(weighted=True))\n"
            "T.test_tables_through_shim_equal_reference_tables(192, 128, 2, 10, [2], {})\n"
            "T.test_tables_through_shim_equal_reference_tables(192, 128, 3, 8, [1, 2], dict(sao_restore=True))\n"
            "T.test_tables_through_shim_equal_reference_tables(192, 128, 2, 8, [1], dict(cip=True, p_intra=0.6))\n" % (ROOT, HERE))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900, env=dict(os.environ, LD_PRELOAD=EMUL))
    assert r.returncode == 0, r.stderr[-3000:]


def corrupted_copy(stream, seed, path):
    """three single-bit errors in the last two thirds of the file (slice data, occasionally a header)"""
    import random
    rnd = random.Random(seed)
    data = bytearray(open(stream, "rb").read())
    for _ in range(3):
        data[rnd.randrange(len(data) // 3, len(data))] ^= 1 << rnd.randrange(8)
    open(path, "wb").write(data)


@needs_emul
@pytest.mark.parametrize("threads", ["1", "4"])
@pytest.mark.parametrize("seed", [1, 4, 0])
def test_corrupted_stream_neither_hangs_nor_loses_pictures(tmp_path, seed, threads):
    """Bit errors make the reference abandon a picture in the middle (hls_slice_data comes back short, the error is swallowed) and
    carry on.  The drop-in must do the same: same number of pictures, no error, no dead lock -- with frame threads the pictures
    behind an abandoned one wait for its ticket, so it is closed (with what was recorded: the part the reference reconstructed
    too) when its packet ends (b200_frame_readback(s, NULL), INTEGRATION.md).  Seeds 1 and 4 abandon a picture; before that
    fix they hung with four frame threads.  Pictures decoded before the first damaged one must be identical; the damaged ones
    differ only where neither decoder wrote anything (stale buffer contents)."""
    if not os.path.exists(os.path.join(REFDIR, "decode_b200")):
        pytest.skip("oracle/_ref/decode_b200 not built (needs /root/reference)")
    stream = os.path.join(HERE, "golden", "streams", "b_416x240_10b_weighted.hevc")
    bad = str(tmp_path / "corrupt.hevc")
    corrupted_copy(stream, seed, bad)
    ref = subprocess.run([os.path.join(REFDIR, "decode_ref"), bad, threads], capture_output=True, text=True, timeout=120)
    want = [l for l in ref.stdout.splitlines() if l.startswith("frame ")]
    got = decode_emulated(bad, threads)                      # asserts returncode 0; its own timeout catches a dead lock
    assert len(got) == len(want)
    clean = open(stream[:-5] + ".md5").read().splitlines()
    n_clean = 0
    while n_clean < len(want) and want[n_clean] == clean[n_clean]:
        n_clean += 1
    assert got[:n_clean] == want[:n_clean]


@needs_emul
@pytest.mark.parametrize("threads", ["1", "4"])
def test_geometry_change_in_mid_stream(tmp_path, threads):
    """three streams back to back: 416x240 8-bit, 256x128 8-bit, 416x240 10-bit.  A new SPS means a new device context, plane
    sizes and sample width; with frame threads the pictures of the old sequence are still being parsed on other threads when the
    first picture of the new one begins, so the shim drains them first (G.in_flight)."""
    if not os.path.exists(os.path.join(REFDIR, "decode_b200")):
        pytest.skip("oracle/_ref/decode_b200 not built (needs /root/reference)")
    names = ["p_416x240_8b", "i_256x128_8b_nosao", "b_416x240_10b_weighted"]
    path = str(tmp_path / "concat.hevc")
    with open(path, "wb") as f:
        for n in names:
            f.write(open(os.path.join(HERE, "golden", "streams", n + ".hevc"), "rb").read())
    ref = subprocess.run([os.path.join(REFDIR, "decode_ref"), path, threads], capture_output=True, text=True, timeout=120)
    want = [l for l in ref.stdout.splitlines() if l.startswith("frame ")]
    assert len(want) == 13
    assert decode_emulated(path, threads) == want


def damaged(kind):
    src = open(os.path.join(HERE, "golden", "streams", "ra_416x240_8b.hevc"), "rb").read()
    if kind == "truncated":
        return src[:int(len(src) * 0.7)]                                   # ends in the middle of a NAL unit
    starts = [i for i in range(len(src) - 3) if src[i:i + 3] == b"\x00\x00\x01"]
    units = [src[i:j] for i, j in zip(starts, starts[1:] + [len(src)])]
    first_irap = next(k for k, u in enumerate(units) if (u[3] >> 1) & 0x3f in (19, 20))
    return b"\x00" + b"".join(u for k, u in enumerate(units) if k != first_irap)     # the IDR picture is gone: every reference of the first GOP is missing


@needs_emul
@pytest.mark.parametrize("threads", ["1", "4"])
@pytest.mark.parametrize("kind", ["truncated", "no_idr"])
def test_damaged_streams_behave_like_the_reference(tmp_path, kind, threads):
    """a stream cut off in the middle of a NAL unit, and one whose first picture was lost (the decoder generates grey references,
    hevc_refs.c:538-606 -> b200_frame_fill): same pictures as the unmodified decoder, no error, no dead lock"""
    if not os.path.exists(os.path.join(REFDIR, "decode_b200")):
        pytest.skip("oracle/_ref/decode_b200 not built (needs /root/reference)")
    path = str(tmp_path / (kind + ".hevc"))
    open(path, "wb").write(damaged(kind))
    ref = subprocess.run([os.path.join(REFDIR, "decode_ref"), path, threads], capture_output=True, text=True, timeout=120)
    want = [l for l in ref.stdout.splitlines() if l.startswith("frame ")]
    assert want
    assert decode_emulated(path, threads) == want
