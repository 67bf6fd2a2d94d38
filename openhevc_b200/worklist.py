"""numpy mirror of include/b200hevc_worklist.h (blob v3) — builder and parser.

Host-side only.  The structured dtypes below are byte-for-byte the C structs; a blob built here
is what the C recorder (csrc/recorder.cpp) produces for the same table calls.
"""
import numpy as np

MAGIC = 0x4C573242
VERSION = 3
TU_DENSE = 0xFFFF
(SEC_COEFF, SEC_TU4, SEC_TU8, SEC_TU16, SEC_TU32, SEC_INTRA, SEC_MC, SEC_DBK, SEC_SAO, SEC_COUNT) = range(10)

TU_IDCT, TU_DC, TU_DST, TU_SKIP, TU_BYPASS, TU_PCM = range(6)
TUF_RDPCM, TUF_RDPCM_VERT, TUF_PARK = 1, 2, 4
INF_UP_LEFT, INF_UP, INF_UP_RIGHT, INF_LEFT, INF_BOTTOM_LEFT, INF_FILTER, INF_STRONG = 1, 2, 4, 8, 16, 32, 64
MCF_BI, MCF_WEIGHTED, MCF_CHROMA = 1, 2, 4
SAO_NONE, SAO_BAND, SAO_EDGE = 0, 1, 2
NO_RESID = 0xFFFFFFFF
FRAME_HAS_DEBLOCK, FRAME_HAS_SAO, FRAME_CIP, FRAME_TQB = 1, 2, 4, 8

section_dt = np.dtype([("off", "<u4"), ("count", "<u4")])
header_dt = np.dtype([
    ("magic", "<u4"), ("version", "<u4"), ("total_bytes", "<u4"), ("poc", "<i4"),
    ("width", "<u2"), ("height", "<u2"), ("chroma_format_idc", "u1"), ("bit_depth", "u1"),
    ("log2_ctb_size", "u1"), ("cur_slot", "u1"), ("flags", "<u4"),
    ("sec", section_dt, (SEC_COUNT,)), ("ref_slot", "u1", (16,)), ("n_ref", "u1"), ("pad", "u1", (3,)),
    ("mc_big_count", "<u4"), ("cip", section_dt), ("tqb", section_dt), ("ccp", section_dt), ("dbd", section_dt), ("reserved_section", section_dt),
    ("reserved", "<u4", (64 - 23 - 2 * SEC_COUNT,)),
])
tu_dt = np.dtype([("x", "<u2"), ("y", "<u2"), ("plane", "u1"), ("log2", "u1"), ("kind", "u1"), ("flags", "u1"),
                  ("col_limit", "u1"), ("pad", "u1"), ("nnz", "<u2"), ("coeff_off", "<u4")])
intra_dt = np.dtype([("x", "<u2"), ("y", "<u2"), ("plane", "u1"), ("log2", "u1"), ("mode", "u1"), ("flags", "u1"),
                     ("top_right_size", "u1"), ("bottom_left_size", "u1"), ("pad", "u1", (2,)), ("resid_off", "<u4")])
mc_dt = np.dtype([("x", "<u2"), ("y", "<u2"), ("w", "u1"), ("h", "u1"), ("plane", "u1"), ("flags", "u1"),
                  ("sx0", "<i2"), ("sy0", "<i2"), ("sx1", "<i2"), ("sy1", "<i2"), ("ref0", "u1"), ("ref1", "u1"),
                  ("frac0", "u1"), ("frac1", "u1"), ("w0", "<i2"), ("w1", "<i2"), ("o0", "<i2"), ("o1", "<i2"),
                  ("denom", "u1"), ("pad", "u1", (3,))])
sao_dt = np.dtype([("type", "u1"), ("param", "u1"), ("borders", "u1"), ("edges", "u1"), ("variant", "u1"), ("tqb", "u1"),
                   ("offset_val", "<i2", (5,))])
assert header_dt.itemsize == 256 and tu_dt.itemsize == 16 and intra_dt.itemsize == 16 and mc_dt.itemsize == 32 and sao_dt.itemsize == 16

DBK_PRESENT = 0x8000


def dbk_pack(tc, beta, no_p=0, no_q=0):
    return DBK_PRESENT | (int(tc) & 63) | ((int(beta) & 127) << 6) | ((int(no_p) & 1) << 13) | ((int(no_q) & 1) << 14)


def plane_dims(width, height, cfi, plane):
    hs = 1 if (plane and cfi != 3) else 0
    vs = 1 if (plane and cfi == 1) else 0
    return width >> hs, height >> vs


class DbkLayout:
    """b200_dbk_layout(): offsets / strides (uint16 units) of the six edge-parameter grids."""

    def __init__(self, width, height, cfi):
        self.off, self.stride, self.rows = {}, {}, {}
        o = 0
        for p in range(3):
            pw, ph = plane_dims(width, height, cfi, p)
            dims = [((pw + 7) >> 3, (ph + 3) >> 2), ((pw + 3) >> 2, (ph + 7) >> 3)]
            for d in range(2):
                self.off[p, d], self.stride[p, d], self.rows[p, d] = o, dims[d][0], dims[d][1]
                o = (o + dims[d][0] * dims[d][1] + 63) // 64 * 64
        self.total = o

    def view(self, grid, plane, direction):
        o, s, r = self.off[plane, direction], self.stride[plane, direction], self.rows[plane, direction]
        return grid[o:o + s * r].reshape(r, s)


def split_mc_tiles(recs):
    """Same tiling as b200_rec_mc(): every block becomes tiles of <= 16x16 (blocks taller than 8) or <= 32x8 samples (vectorised per block shape)."""
    if len(recs) == 0:
        return np.zeros(0, mc_dt)
    out = []
    shapes = np.unique(np.stack([recs["w"], recs["h"]], 1), axis=0)
    for w, h in shapes:
        w, h = int(w), int(h)
        sel = recs[(recs["w"] == w) & (recs["h"] == h)]
        tiles, tx = [], 0
        twmax = 16 if h > 8 else 32
        while tx < w:
            tw = min(twmax, w - tx)
            maxh = 8 if tw > 16 else 16
            tiles += [(tx, ty, tw, min(maxh, h - ty)) for ty in range(0, h, maxh)]
            tx += tw
        for (tx, ty, tw, th) in tiles:
            t = sel.copy()
            t["x"] += tx; t["y"] += ty; t["w"] = tw; t["h"] = th
            t["sx0"] += tx; t["sy0"] += ty; t["sx1"] += tx; t["sy1"] += ty
            out.append(t)
    return np.concatenate(out)


def order_mc(recs):
    """B200_SEC_MC order (B200BlobHeader.mc_big_count): big tiles in the given order, then the <= 8x8 tiles bucketed by
    (chroma, bi) -- same stable bucketing as b200_rec_finish().  Returns (ordered records, mc_big_count)."""
    recs = np.ascontiguousarray(recs, mc_dt)
    small = (recs["w"] <= 8) & (recs["h"] <= 8)
    key = np.where(small, 1 + np.where(recs["flags"] & MCF_CHROMA, 2, 0) + np.where(recs["flags"] & MCF_BI, 1, 0), 0)
    return recs[np.argsort(key, kind="stable")], int((~small).sum())


def tu_dense(t, pool):
    """(dense NxN coefficients, parked-pool index or None) of one TU record -- mirror of b200_tu_data / b200_tu_expand"""
    n2 = 1 << (2 * int(t["log2"]))
    o = int(t["coeff_off"])
    park = None
    if t["flags"] & TUF_PARK:
        park = int(pool[o].astype(np.uint16)) | (int(pool[o + 1].astype(np.uint16)) << 16)
        o += 2
    if t["nnz"] == TU_DENSE:
        return np.array(pool[o:o + n2]), park
    d = np.zeros(n2, np.int16)
    e = pool[o:o + 2 * int(t["nnz"])].reshape(-1, 2)
    d[e[:, 0].astype(np.uint16)] = e[:, 1]
    return d, park


def level_order(intra, width, height, cfi):
    """Permutation that sorts decode-order intra records by dependency level (stable) -- computed by the same host
    routine the C recorder uses (b200_intra_level_order in libb200hevc.so; pure host code, no GPU needed)."""
    from . import _lib
    lib = _lib.load()
    intra = np.ascontiguousarray(intra, intra_dt)
    perm = np.zeros(len(intra), np.uint32)
    rc = lib.b200_intra_level_order(intra.ctypes.data, len(intra), width, height, cfi, perm.ctypes.data)
    if rc < 0:
        raise ValueError(f"b200_intra_level_order failed: {rc}")
    return perm, rc


def build_blob(width, height, cfi, bit_depth, log2_ctb, cur_slot, poc=0, coeff=None, tu=None, intra=None, mc=None,
               dbk=None, sao=None, out=None, ref_slots=(), cip=None, tqb=None):
    """Assemble a blob.  tu: dict {2,3,4,5 -> tu_dt array}; dbk: uint16 array (DbkLayout.total) or None;
    sao: sao_dt array [3*ctb_count] or None.  `out`: optional uint8 buffer (e.g. pinned) to build into.
    cip: None, or (log2_min_pu, bool array [min_pu_height, min_pu_width], True = intra PU) for a constrained_intra_pred picture.
    tqb: None, or (log2_min_pu, bool array [min_pu_height, min_pu_width], True = PCM-without-loop-filter / transquant-bypass PU);
    the CTBs of `sao` that contain such PUs are marked."""
    coeff = np.zeros(0, np.int16) if coeff is None else np.ascontiguousarray(coeff, np.int16)
    tu = tu or {}
    parts = [None] * SEC_COUNT
    parts[SEC_COEFF] = coeff
    for k in range(4):
        parts[SEC_TU4 + k] = np.ascontiguousarray(tu.get(k + 2, np.zeros(0, tu_dt)), tu_dt)
    parts[SEC_INTRA] = np.ascontiguousarray(intra if intra is not None else np.zeros(0, intra_dt), intra_dt)
    parts[SEC_MC], mc_big = order_mc(mc if mc is not None else np.zeros(0, mc_dt))
    parts[SEC_DBK] = np.ascontiguousarray(dbk if dbk is not None else np.zeros(0, np.uint16), np.uint16)
    parts[SEC_SAO] = np.ascontiguousarray(sao if sao is not None else np.zeros(0, sao_dt), sao_dt)
    hdr = np.zeros(1, header_dt)
    hdr["magic"], hdr["version"], hdr["poc"] = MAGIC, VERSION, poc
    hdr["width"], hdr["height"], hdr["chroma_format_idc"], hdr["bit_depth"] = width, height, cfi, bit_depth
    hdr["log2_ctb_size"], hdr["cur_slot"] = log2_ctb, cur_slot
    assert len(ref_slots) <= 16
    hdr["n_ref"] = len(ref_slots)
    hdr["mc_big_count"] = mc_big
    hdr["ref_slot"][0][:len(ref_slots)] = list(ref_slots)
    hdr["flags"] = (FRAME_HAS_DEBLOCK if len(parts[SEC_DBK]) else 0) | (FRAME_HAS_SAO if len(parts[SEC_SAO]) else 0)
    off = 256
    for s, p in enumerate(parts):
        hdr["sec"][0][s] = (off, len(p))
        off = (off + p.nbytes + 255) // 256 * 256
    cip_words = None
    if cip is not None:
        log2_pu, bitmap = cip
        bitmap = np.ascontiguousarray(bitmap, bool)
        bits = np.packbits(bitmap.reshape(-1), bitorder="little")
        bits = np.concatenate([bits, np.zeros(-len(bits) % 4, np.uint8)]).view("<u4")
        cip_words = np.concatenate([np.array([log2_pu, bitmap.shape[1], bitmap.shape[0], 0], "<u4"), bits])
        hdr["cip"][0] = (off, len(cip_words))
        hdr["flags"] |= FRAME_CIP
        off = (off + cip_words.nbytes + 255) // 256 * 256
    tqb_words = None
    if tqb is not None and len(parts[SEC_SAO]):
        log2_pu, bitmap = tqb
        bitmap = np.ascontiguousarray(bitmap, bool)
        bits = np.packbits(bitmap.reshape(-1), bitorder="little")
        bits = np.concatenate([bits, np.zeros(-len(bits) % 4, np.uint8)]).view("<u4")
        tqb_words = np.concatenate([np.array([log2_pu, bitmap.shape[1], bitmap.shape[0], 0], "<u4"), bits])
        hdr["tqb"][0] = (off, len(tqb_words))
        hdr["flags"] |= FRAME_TQB
        off = (off + tqb_words.nbytes + 255) // 256 * 256
        # mark the CTBs
        per = (1 << log2_ctb) >> log2_pu
        cw, ch = (width + (1 << log2_ctb) - 1) >> log2_ctb, (height + (1 << log2_ctb) - 1) >> log2_ctb
        g = parts[SEC_SAO] = parts[SEC_SAO].copy()
        for cy in range(ch):
            for cx in range(cw):
                if bitmap[cy * per:(cy + 1) * per, cx * per:(cx + 1) * per].any():
                    for pl in range(3):
                        g["tqb"][(pl * ch + cy) * cw + cx] = 1
    hdr["total_bytes"] = off
    if out is None:
        out = np.zeros(off, np.uint8)
    else:
        assert out.dtype == np.uint8 and out.size >= off
        out = out[:off]
    out[:256] = hdr.view(np.uint8)
    for s, p in enumerate(parts):
        o = int(hdr["sec"][0][s]["off"])
        out[o:o + p.nbytes] = p.view(np.uint8).reshape(-1)
    if cip_words is not None:
        o = int(hdr["cip"][0]["off"])
        out[o:o + cip_words.nbytes] = cip_words.view(np.uint8)
    if tqb_words is not None:
        o = int(hdr["tqb"][0]["off"])
        out[o:o + tqb_words.nbytes] = tqb_words.view(np.uint8)
    return out


def parse_blob(blob):
    """Inverse of build_blob (views into the blob)."""
    blob = np.frombuffer(blob, np.uint8) if not isinstance(blob, np.ndarray) else blob
    hdr = blob[:256].view(header_dt)[0]
    assert hdr["magic"] == MAGIC and hdr["version"] == VERSION
    dts = [np.int16, tu_dt, tu_dt, tu_dt, tu_dt, intra_dt, mc_dt, np.uint16, sao_dt]
    secs = []
    for s in range(SEC_COUNT):
        o, n = int(hdr["sec"][s]["off"]), int(hdr["sec"][s]["count"])
        secs.append(blob[o:o + n * np.dtype(dts[s]).itemsize].view(dts[s]))
    return hdr, secs
