"""CPU suite (-m "not gpu"): the oracle against the reference build, host logic, C-ABI exports."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_lib
from openhevc_b200 import worklist as W
from openhevc_b200.synth import FrameSynth, smooth_frame


def test_oracle_pinned_against_reference_tables(built):
    """oracle/kat_ref links the UNMODIFIED reference C tables (oracle/_ref/libohevc_ref.so) and compares every
    slot of SURVEY.md §8(a) with the restatement, bit for bit, on seeded random inputs (8/10/12 bit)."""
    if not os.path.exists(oracle_lib.KAT_REF):
        pytest.skip("oracle/_ref/kat_ref not built (reference sources absent and no prebuilt binary)")
    out = subprocess.run([oracle_lib.KAT_REF, "600"], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert " 0 mismatches" in out.stdout


def test_blob_roundtrip_and_layout():
    s = FrameSynth(128, 64, cfi=1, bit_depth=8, seed=1, refs=[1, 2], cur_slot=0)
    blob, st = s.generate()
    hdr, secs = W.parse_blob(blob)
    assert hdr["total_bytes"] == blob.nbytes and hdr["width"] == 128 and hdr["cur_slot"] == 0
    assert all(int(hdr["sec"][k]["off"]) % 256 == 0 for k in range(W.SEC_COUNT))
    assert len(secs[W.SEC_MC]) == st["n_mc_tiles"] and (secs[W.SEC_MC]["w"].astype(int) * secs[W.SEC_MC]["h"] <= 256).all()
    L = W.DbkLayout(128, 64, 1)
    assert len(secs[W.SEC_DBK]) == L.total


def test_numpy_mirror_matches_the_c_header(tmp_path):
    """every field of every dtype of worklist.py at the offset and with the size the C compiler gives the struct field of the
    same name in include/b200hevc_worklist.h, every struct of the same size, and every constant of the same value"""
    lines, want = [], []
    for struct, dt in {"B200Section": W.section_dt, "B200BlobHeader": W.header_dt, "B200TuRec": W.tu_dt, "B200IntraRec": W.intra_dt, "B200McRec": W.mc_dt,
                       "B200SaoRec": W.sao_dt, "B200CcpRec": W.ccp_dt, "B200CipHeader": W.cip_header_dt}.items():
        lines.append(f'printf("{struct} %zu\\n", sizeof({struct}));')
        want.append(f"{struct} {dt.itemsize}")
        for name, (fdt, off) in dt.fields.items():
            lines.append(f'printf("{struct}.{name} %zu %zu\\n", offsetof({struct}, {name}), sizeof((({struct} *)0)->{name}));')
            want.append(f"{struct}.{name} {off} {fdt.itemsize}")
    for name, value in vars(W).items():
        if name.isupper() and isinstance(value, int):
            lines.append(f'printf("{name} %lld\\n", (long long)B200_{"BLOB_" if name in ("MAGIC", "VERSION") else ""}{name});')
            want.append(f"{name} {value}")
    src = tmp_path / "layout.c"
    src.write_text("#include <stddef.h>\n#include <stdio.h>\n#include \"b200hevc_worklist.h\"\nint main(void)\n{\n" + "\n".join(lines) + "\nreturn 0;\n}\n")
    subprocess.run(["cc", "-I", os.path.join(oracle_lib.ROOT, "include"), "-o", str(tmp_path / "layout"), str(src)], check=True)
    assert subprocess.run([str(tmp_path / "layout")], capture_output=True, text=True, check=True).stdout.splitlines() == want


@pytest.mark.parametrize("cfi,bd,refs", [(1, 8, []), (1, 10, [1, 2]), (2, 10, [1]), (3, 8, [1, 2])])
def test_synth_is_in_decode_order_and_oracle_runs(cfi, bd, refs):
    w, h = 192, 128
    s = FrameSynth(w, h, cfi=cfi, bit_depth=bd, seed=7 + cfi + bd, refs=refs, cur_slot=0, exotic=0.05, sao_restore=True)
    blob, st = s.generate()
    assert oracle_lib.check_decode_order(blob)
    dpb = [smooth_frame(w, h, cfi, bd, 100 + k) for k in range(3)]
    out = oracle_lib.execute(blob, dpb)
    maxv = (1 << bd) - 1
    assert all(p.max() <= maxv for p in out)
    # determinism + the oracle must not touch the reference slots
    out2 = oracle_lib.execute(blob, dpb)
    assert all((a == b).all() for a, b in zip(out, out2))


@pytest.mark.parametrize("cfi,bd,refs,kw", [(1, 8, [], {}), (1, 10, [1, 2], dict(weighted=True)), (2, 10, [1, 2], {}), (3, 8, [2], dict(sao_restore=True)), (1, 12, [1], {}),
                                            # constrained_intra_pred (hevcpred_template.c:116-249): inter pictures with 12 % / 45 % intra CUs
                                            (1, 8, [1, 2], dict(cip=True)), (1, 10, [1], dict(cip=True, p_intra=0.45)), (2, 10, [1, 2], dict(cip=True, p_intra=0.3)),
                                            (3, 8, [2], dict(cip=True, p_intra=0.3, split_bias=2.0))])
def test_oracle_equals_reference_at_picture_level(built, cfi, bd, refs, kw):
    """whole synthetic pictures: restatement (oracle/hevc_oracle.c) == the reference's own table functions
    driven by oracle/replay_ref.c -- MC incl. emulated edges, all transforms, intra_pred(), deblock, SAO."""
    if oracle_lib.ref_lib() is None:
        pytest.skip("oracle/_ref/libreplay_ref.so not available")
    w, h = 320, 192
    blob, st = FrameSynth(w, h, cfi=cfi, bit_depth=bd, seed=90 + cfi + bd, refs=refs, cur_slot=0, exotic=0.05, max_mv=100, **kw).generate()
    dpb = [smooth_frame(w, h, cfi, bd, 200 + k) for k in range(3)]
    a = oracle_lib.execute(blob, dpb)
    oracle_lib.assert_same(a, oracle_lib.ref_execute(blob, dpb), "oracle against the reference tables")


def test_oracle_properties_linearity_of_residual():
    """size-independent property: with prediction 0 and no clipping the IDCT stage is linear:
    recon(a) + recon(b) - recon(0) == recon(a + b) whenever intermediate clips do not trigger."""
    lib = oracle_lib.lib()
    lib.orc_idct.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
    rng = np.random.default_rng(3)
    for log2 in (2, 3, 4, 5):
        n = 1 << log2
        a = (rng.integers(-40, 41, (n, n)) * 64).astype(np.int16)     # multiples of 64: both stages stay exact
        b = (rng.integers(-40, 41, (n, n)) * 64).astype(np.int16)
        s = (a + b).astype(np.int16)
        outs = []
        for m in (a, b, s):
            m = m.copy()
            lib.orc_idct(m.ctypes.data, log2, n, 8)
            outs.append(m.astype(np.int64))
        assert np.abs(outs[0] + outs[1] - outs[2]).max() <= 2      # rounding of the two >> stages only


def test_c_abi_exports_every_declared_symbol(built):
    """the shared library loads (no GPU needed) and exports exactly what include/b200hevc.h declares"""
    from openhevc_b200 import _lib
    import re
    hdr = open(os.path.join(oracle_lib.ROOT, "include", "b200hevc.h")).read()
    declared = set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", hdr))
    assert declared == set(_lib.EXPORTS), declared ^ set(_lib.EXPORTS)
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name)


def test_table_level_library_exports_every_declared_symbol(built):
    """libb200hevc_shim.so (the table-level drop-in, include/b200hevc_tables.h) loads without a GPU and exports every entry
    point the reference-side hook lines of INTEGRATION.md call"""
    import ctypes
    import re
    hdr = open(os.path.join(oracle_lib.ROOT, "include", "b200hevc_tables.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b((?:ff_hevcdsp|ff_hevcpred|ff_videodsp)_init_b200|b200_[a-z0-9_]+)\s*\(", hdr))
    assert {"ff_hevcdsp_init_b200", "ff_hevcpred_init_b200", "ff_videodsp_init_b200", "b200_frame_begin", "b200_frame_end",
            "b200_frame_readback", "b200_frame_fill", "b200_host_pixels_unused"} <= declared
    path = oracle_lib.SHIM_SO
    if not os.path.exists(path):
        pytest.skip("libb200hevc_shim.so not built (needs the reference headers)")
    lib = ctypes.CDLL(path)
    for name in declared:
        assert hasattr(lib, name), name


def test_no_gpu_means_loud_failure_not_fallback(built):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from openhevc_b200 import FrameEngine, B200Error
    with pytest.raises(B200Error, match="no CUDA device|CUDA"):
        FrameEngine(64, 64)


TU_ARGS = ("plane", "x", "y", "log2", "kind", "flags", "col_limit")


def replay_through_recorders(blob, geom, n_workers):
    """Replays a blob's records through the C recorder the way the decoder's table calls would arrive.  With
    n_workers > 1 the calls of CTB row k go to recorder k % n_workers (WPP / slice threads: every worker has its own
    B200Rec and its own, lazily built reference table) and the workers are folded into recorder 0 with b200_rec_merge."""
    w, h, cfi, bd = geom
    hdr, secs = W.parse_blob(blob)
    recs = [W.Recorder(geom, int(hdr["cur_slot"])) for _ in range(n_workers)]
    tables = [[] for _ in range(n_workers)]

    def who(plane, y):
        vs = 1 if (plane and cfi == 1) else 0
        return ((int(y) << vs) >> 6) % n_workers

    pool = secs[W.SEC_COEFF]
    # replay in an order the decoder could have used: intra pred call immediately followed by its residual
    parked = {}
    for k in range(4):
        for t in secs[W.SEC_TU4 + k]:
            if t["flags"] & W.TUF_PARK:
                parked[W.tu_dense(t, pool)[1]] = t
    for ir in secs[W.SEC_INTRA]:
        r = recs[who(ir["plane"], ir["y"])]
        r.intra(*(ir[f] for f in ("plane", "x", "y", "log2", "mode", "flags", "top_right_size", "bottom_left_size")))
        if ir["resid_off"] != W.NO_RESID:
            t = parked[int(ir["resid_off"])]
            r.tu(*(t[f] for f in TU_ARGS), W.tu_dense(t, pool)[0], 1)
    for k in range(4):
        for t in secs[W.SEC_TU4 + k]:
            if t["flags"] & W.TUF_PARK:
                continue
            recs[who(t["plane"], t["y"])].tu(*(t[f] for f in TU_ARGS), W.tu_dense(t, pool)[0], -1)
    ref_slots = [int(v) for v in hdr["ref_slot"][:int(hdr["n_ref"])]]
    for m in secs[W.SEC_MC]:
        k = who(m["plane"], m["y"])
        mm = np.array([m])
        for f in ("ref0", "ref1") if m["flags"] & W.MCF_BI else ("ref0",):     # the worker's own table, in order of first use
            slot = ref_slots[int(m[f])]
            if slot not in tables[k]:
                tables[k].append(slot)
            mm[f] = tables[k].index(slot)
        recs[k].mc(mm)
    L = W.DbkLayout(w, h, cfi)
    grid = secs[W.SEC_DBK]
    for p in range(3):
        for d in range(2):
            v = L.view(grid, p, d)
            ys, xs = np.nonzero(v)
            done = set()
            for gy, gx in zip(ys, xs):
                x, y = (gx * 8, gy * 4) if d == 0 else (gx * 4, gy * 8)
                x0, y0 = (x, y & ~7) if d == 0 else (x & ~7, y)      # a table call covers two segments
                if (x0, y0) in done:
                    continue
                done.add((x0, y0))
                ent = [int(v[(y0 // 4 + j), gx]) if d == 0 else int(v[gy, x0 // 4 + j]) for j in range(2)]
                beta = max((e >> 6) & 127 for e in ent)
                recs[who(p, y0)].deblock(p, 1 - d, x0, y0, beta, [e & 63 for e in ent], [(e >> 13) & 1 for e in ent], [(e >> 14) & 1 for e in ent])
    sg = secs[W.SEC_SAO]
    nctb = len(sg) // 3
    cw = (w + 63) // 64
    for p in range(3):
        hs, vs = ((1 if cfi != 3 else 0), (1 if cfi == 1 else 0)) if p else (0, 0)
        for i in range(nctb):
            recs[(i // cw) % n_workers].sao(p, ((i % cw) * 64) >> hs, ((i // cw) * 64) >> vs, sg[p * nctb + i])
    for k in range(n_workers):
        recs[k].set_refs(tables[k])
    for k in range(1, n_workers):
        recs[0].merge(recs[k])
    return recs[0].finish()


def test_recorder_matches_numpy_builder(built):
    """the C recorder (host-only code path of libb200hevc.so) and the numpy builder produce equivalent blobs"""
    w, h, cfi, bd = 128, 64, 1, 8
    s = FrameSynth(w, h, cfi=cfi, bit_depth=bd, seed=11, refs=[1, 2], cur_slot=3, exotic=0.05)
    blob, _ = s.generate()
    hdr, secs = W.parse_blob(blob)
    rblob = replay_through_recorders(blob, (w, h, cfi, bd), 1)
    # same picture on the oracle from both blobs
    dpb = [smooth_frame(w, h, cfi, bd, 50 + k) for k in range(4)]
    a = oracle_lib.execute(blob, dpb)
    b = oracle_lib.execute(rblob, dpb)
    assert all((x == y).all() for x, y in zip(a, b))
    rh, rs = W.parse_blob(rblob)
    assert len(rs[W.SEC_MC]) == len(secs[W.SEC_MC]) and len(rs[W.SEC_INTRA]) == len(secs[W.SEC_INTRA])


@pytest.mark.parametrize("n_workers,cfi,refs", [(2, 1, [1, 2]), (3, 1, []), (3, 2, [2, 1])])
def test_recorder_merge_of_worker_threads(built, n_workers, cfi, refs):
    """WPP / slice threads: per-worker recorders (CTB rows interleaved) merged at frame end give the same picture,
    and the merged intra list is still in a valid dependency order"""
    w, h, bd = 192, 320, 10
    blob, _ = FrameSynth(w, h, cfi=cfi, bit_depth=bd, seed=77 + n_workers, refs=refs, cur_slot=3, exotic=0.05, p_intra=0.3 if refs else 1.0).generate()
    rblob = replay_through_recorders(blob, (w, h, cfi, bd), n_workers)
    oracle_lib.check_decode_order(rblob)
    dpb = [smooth_frame(w, h, cfi, bd, 60 + k) for k in range(4)]
    a = oracle_lib.execute(blob, dpb)
    b = oracle_lib.execute(rblob, dpb)
    assert all((x == y).all() for x, y in zip(a, b))
    rh, rs = W.parse_blob(rblob)
    assert sorted(int(v) for v in rh["ref_slot"][:int(rh["n_ref"])]) == sorted(refs)
