#!/usr/bin/env python
"""Synthetic Annex-B HEVC stream writer (intra pictures) — TEST INFRASTRUCTURE.

No encoder or sample bit stream exists in the build environment (SURVEY.md §0), so the streams that drive the
*real* reference decoder (oracle/_ref/decode_ref vs decode_b200, tests/test_stream_*.py) are written here: a random
but syntax-valid coding structure (CTB quadtrees, 2Nx2N / NxN intra CUs with MPM / remaining-mode signalling,
residual quadtrees, residual_coding() with last-position, coded-sub-block, significance, greater1/2, remaining
levels and signs, per-CTB SAO, in-loop deblocking on) entropy-coded with a from-scratch CABAC *encoder*
(ITU-T H.265 9.3.4).  The context initialisation values and their layout are standard tables; they are parsed at
generation time from the reference source (libavcodec/hevc_cabac.c: num_bins_in_se / init_values) so that the
context numbering is guaranteed to be the decoder's — which is why this tool runs in the build container only;
the streams it produces are committed under tests/golden/.
"""
import argparse
import os
import re
import sys

import numpy as np

REF = os.environ.get("REF", "/root/reference")

# ----------------------------------------------------------------------------------------------------------------
# bit writing / NAL units
# ----------------------------------------------------------------------------------------------------------------
class BitWriter:
    def __init__(self):
        self.bits = []

    def u(self, n, v):
        for i in range(n - 1, -1, -1):
            self.bits.append((v >> i) & 1)

    def ue(self, v):
        v += 1
        n = v.bit_length()
        self.u(n - 1, 0)
        self.u(n, v)

    def se(self, v):
        self.ue(2 * v - 1 if v > 0 else -2 * v)

    def trailing(self):
        self.bits.append(1)
        while len(self.bits) % 8:
            self.bits.append(0)

    def bytes(self):
        assert len(self.bits) % 8 == 0
        return bytes(int("".join(map(str, self.bits[i:i + 8])), 2) for i in range(0, len(self.bits), 8))


def nal(nal_type, payload, layer=0, tid=0):
    hdr = bytes([(nal_type << 1) | (layer >> 5), ((layer & 31) << 3) | (tid + 1)])
    out, zeros = bytearray(), 0
    for b in payload:                     # emulation prevention
        if zeros >= 2 and b <= 3:
            out.append(3)
            zeros = 0
        out.append(b)
        zeros = zeros + 1 if b == 0 else 0
    return b"\x00\x00\x00\x01" + hdr + bytes(out)


# ----------------------------------------------------------------------------------------------------------------
# CABAC encoder (H.265 9.3.4.x, encoder side as in the HM description)
# ----------------------------------------------------------------------------------------------------------------
RANGE_TAB_LPS = [
    [128, 176, 208, 240], [128, 167, 197, 227], [128, 158, 187, 216], [123, 150, 178, 205], [116, 142, 169, 195], [111, 135, 160, 185], [105, 128, 152, 175], [100, 122, 144, 166],
    [95, 116, 137, 158], [90, 110, 130, 150], [85, 104, 123, 142], [81, 99, 117, 135], [77, 94, 111, 128], [73, 89, 105, 122], [69, 85, 100, 116], [66, 80, 95, 110],
    [62, 76, 90, 104], [59, 72, 86, 99], [56, 69, 81, 94], [53, 65, 77, 89], [51, 62, 73, 85], [48, 59, 69, 80], [46, 56, 66, 76], [43, 53, 63, 72],
    [41, 50, 59, 69], [39, 48, 56, 65], [37, 45, 54, 62], [35, 43, 51, 59], [33, 41, 48, 56], [32, 39, 46, 53], [30, 37, 43, 50], [29, 35, 41, 48],
    [27, 33, 39, 45], [26, 31, 37, 43], [24, 30, 35, 41], [23, 28, 33, 39], [22, 27, 32, 37], [21, 26, 30, 35], [20, 24, 29, 33], [19, 23, 27, 31],
    [18, 22, 26, 30], [17, 21, 25, 28], [16, 20, 23, 27], [15, 19, 22, 25], [14, 18, 21, 24], [14, 17, 20, 23], [13, 16, 19, 22], [12, 15, 18, 21],
    [12, 14, 17, 20], [11, 14, 16, 19], [11, 13, 15, 18], [10, 12, 15, 17], [10, 12, 14, 16], [9, 11, 13, 15], [9, 11, 12, 14], [8, 10, 12, 14],
    [8, 9, 11, 13], [7, 9, 11, 12], [7, 9, 10, 12], [7, 8, 10, 11], [6, 8, 9, 11], [6, 7, 9, 10], [6, 7, 8, 9], [2, 2, 2, 2]]
TRANS_LPS = [0, 0, 1, 2, 2, 4, 4, 5, 6, 7, 8, 9, 9, 11, 11, 12, 13, 13, 15, 15, 16, 16, 18, 18, 19, 19, 21, 21, 22, 22, 23, 24,
             24, 25, 26, 26, 27, 27, 28, 29, 29, 30, 30, 30, 31, 32, 32, 33, 33, 33, 34, 34, 35, 35, 35, 36, 36, 36, 37, 37, 37, 38, 38, 63]


def verify_tables_against_reference():
    """the range table above is typed from the standard; check it against the decoder's own generated table"""
    import ctypes
    so = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libohevc_ref.so")
    if not os.path.exists(so):
        return
    lib = ctypes.CDLL(so)
    lib.ff_init_cabac_states()
    tab = (ctypes.c_uint8 * (512 + 4 * 2 * 64 + 4 * 64 + 63)).in_dll(lib, "ff_h264_cabac_tables")
    for q in range(4):
        for st in range(64):
            for mps in range(2):
                assert tab[512 + 128 * q + 2 * st + mps] == RANGE_TAB_LPS[st][q], (q, st)
    for st in range(63):
        assert tab[1024 + 128 + 2 * st] >> 1 == min(st + 1, 62), st                   # MPS transition
    for st in range(1, 63):
        assert tab[1024 + 127 - 2 * st] >> 1 == TRANS_LPS[st], (st, tab[1024 + 127 - 2 * st])   # LPS transition


class Cabac:
    def __init__(self, init_values, qp):
        self.low, self.range, self.outstanding, self.first = 0, 510, 0, True
        self.bits = []
        self.state = []
        for iv in init_values:
            m, n = (iv >> 4) * 5 - 45, ((iv & 15) << 3) - 16
            pre = min(max(((m * min(max(qp, 0), 51)) >> 4) + n, 1), 126)
            self.state.append([pre - 64, 1] if pre > 63 else [63 - pre, 0])

    def _put(self, b):
        if self.first:
            self.first = False
        else:
            self.bits.append(b)
        while self.outstanding:
            self.bits.append(1 - b)
            self.outstanding -= 1

    def _renorm(self):
        while self.range < 256:
            if self.low < 256:
                self._put(0)
            elif self.low >= 512:
                self.low -= 512
                self._put(1)
            else:
                self.low -= 256
                self.outstanding += 1
            self.range <<= 1
            self.low <<= 1

    def encode(self, ctx, b):
        st = self.state[ctx]
        lps = RANGE_TAB_LPS[st[0]][(self.range >> 6) & 3]
        self.range -= lps
        if b != st[1]:
            self.low += self.range
            self.range = lps
            if st[0] == 0:
                st[1] = 1 - st[1]
            st[0] = TRANS_LPS[st[0]]
        else:
            st[0] = min(st[0] + 1, 62)
        self._renorm()

    def bypass(self, b):
        self.low <<= 1
        if b:
            self.low += self.range
        if self.low >= 1024:
            self._put(1)
            self.low -= 1024
        elif self.low < 512:
            self._put(0)
        else:
            self.low -= 512
            self.outstanding += 1

    def bypass_bits(self, n, v):
        for i in range(n - 1, -1, -1):
            self.bypass((v >> i) & 1)

    def terminate(self, b):
        self.range -= 2
        if b:
            self.low += self.range
            self.range = 2
            self._renorm()
            self._put((self.low >> 9) & 1)
            self.bits.append((self.low >> 8) & 1)
            self.bits.append(1)                      # rbsp_stop_one_bit doubles as the last written bit (9.3.4.5)
        else:
            self._renorm()


# ----------------------------------------------------------------------------------------------------------------
# context layout, parsed from the decoder's own tables
# ----------------------------------------------------------------------------------------------------------------
def load_contexts():
    src = open(os.path.join(REF, "libavcodec", "hevc_cabac.c")).read()
    src = re.sub(r"#if COM16_C806_EMT.*?#endif", "", src, flags=re.S)
    body = src[src.index("num_bins_in_se[]"):]
    body = body[body.index("{") + 1:body.index("};")]
    names, counts = [], []
    for m in re.finditer(r"(\d+)\s*,\s*//\s*([A-Za-z0-9_,\[\] ]+)", body):
        counts.append(int(m.group(1)))
        names.append(m.group(2).strip())
    off, o = {}, 0
    for nme, c in zip(names, counts):
        off[nme] = o
        o += c
    iv = src[src.index("init_values[3][HEVC_CONTEXTS]"):]
    iv = iv[iv.index("{") + 1:iv.index("};")]
    iv = re.sub(r"//.*", "", iv).replace("CNU", "154")
    rows = [[int(v) for v in re.findall(r"\d+", grp)] for grp in re.findall(r"\{([^{}]*)\}", iv)]
    assert len(rows) == 3 and all(len(rw) == o for rw in rows), [len(rw) for rw in rows]
    return off, rows                                       # rows[init_type], init_type = 2 - slice_type (I -> 0)


# ----------------------------------------------------------------------------------------------------------------
# scans (6.5.3 - 6.5.5)
# ----------------------------------------------------------------------------------------------------------------
def diag_scan(n):
    out, x, y = [], 0, 0
    while len(out) < n * n:
        while y >= 0:
            if x < n and y < n:
                out.append((x, y))
            y -= 1
            x += 1
        y, x = x, 0
    return out


def horiz_scan(n):
    return [(x, y) for y in range(n) for x in range(n)]


def scan_tables(log2, scan_idx):
    """(sub-block order, position order inside a sub-block) as lists of (x, y)"""
    nsb = 1 << (log2 - 2)
    if scan_idx == 0:
        return diag_scan(nsb), diag_scan(4)
    if scan_idx == 1:
        return horiz_scan(nsb), horiz_scan(4)
    return [(y, x) for (x, y) in horiz_scan(nsb)], [(y, x) for (x, y) in horiz_scan(4)]


SIG_CTX_4x4 = [0, 1, 4, 5, 2, 3, 4, 5, 6, 6, 8, 8, 7, 7, 8, 8]


class StreamGen:
    def __init__(self, width, height, bit_depth=8, seed=1, qp=30, sao=True, ctb_log2=6, weighted=False, wpp=False, cip=False, tqb=0.0, tiles=None, lf_across_tiles=True, tskip=0.0, pcm=0.0, pcm_lf_off=False, slices=1, lf_across_slices=True, cfi=1, calm=0.0, ccp=False, amp=False, qpd=False, dbk_offsets=(0, 0), chroma_qp_offsets=(0, 0), tmvp=False, no_dbk=False, sao_planes="both"):
        self.W, self.H, self.bd, self.qp, self.sao, self.ctb_log2 = width, height, bit_depth, qp, sao, ctb_log2
        self.weighted = weighted
        self.conf_win = None                # (L, R, T, B) luma samples of the SPS conformance window, None = flag 0
        self.cip = cip                      # pps constrained_intra_pred_flag (hevcpred_template.c:116-249)
        self.tqb = tqb                      # share of CUs with cu_transquant_bypass_flag (pps transquant_bypass_enable_flag when > 0)
        self.cfi = cfi                      # chroma_format_idc: 1 = 4:2:0, 2 = 4:2:2 (two stacked chroma blocks per TU, RExt), 3 = 4:4:4 (chroma like luma, RExt)
        assert cfi in (1, 2, 3) and not (cfi != 1 and pcm > 0)
        self.slices, self.lf_across_slices = slices, lf_across_slices   # independent slices per picture, each starting a CTB row
        assert slices == 1 or not (tiles or wpp), "several slices are generated without tiles / WPP only"
        self.pcm, self.pcm_lf_off = pcm, pcm_lf_off   # share of 2Nx2N intra CUs (8x8 .. 32x32) coded as PCM; pcm_loop_filter_disabled_flag
        self.dbk_offsets, self.chroma_qp_offsets = dbk_offsets, chroma_qp_offsets   # pps_beta_offset_div2 / pps_tc_offset_div2 (-6..6); pps_cb / cr_qp_offset (-12..12)
        self.sao_planes = sao_planes        # slice_sao_luma_flag / slice_sao_chroma_flag: "both", "luma" or "chroma"
        self.no_dbk = no_dbk                # pps_deblocking_filter_disabled_flag: no deblocking at all (pictures without a deblock section)
        self.tmvp = tmvp                    # sps_temporal_mvp_enabled_flag: temporal merge / AMVP candidates from the collocated picture (host side only)
        self.qpd = qpd                      # pps cu_qp_delta_enabled_flag, one delta per 32x32 quantisation group (diff_cu_qp_delta_depth = log2_ctb - 5)
        self.qp_coded = 1
        self.amp = amp                      # sps amp_enabled_flag: asymmetric motion partitions 2NxnU / 2NxnD / nLx2N / nRx2N above the minimum CB size
        self.ccp = ccp                      # pps cross_component_prediction_enabled_flag (4:4:4 only, hevc.c:1186-1197, 1295-1360)
        assert not ccp or cfi == 3
        self.calm = calm                    # 0 = densely coded random content (default), 1 = lightly coded: more skipped / larger CUs, fewer and sparser residual blocks
        self.tskip = tskip                  # share of 4x4 TUs with transform_skip_flag (pps transform_skip_enabled_flag when > 0)
        self.cu_bypass = 0
        self.tiles = tiles                  # (columns, rows), uniform spacing: one CABAC substream + entry point per tile, tile scan
        self.lf_across_tiles = lf_across_tiles
        # tiles and WPP together (BASELINE.json config 5; hevc.c:2834 hls_decode_entry_wpp_in_tiles): one substream per CTB row of every tile
        self.wpp = wpp                                                    # entropy_coding_sync: one CABAC substream per CTB row
        self.slice_type = 2                                               # 0 B, 1 P, 2 I
        self.nrefs = [0, 0]
        self.reorder = 0                    # sps_max_num_reorder_pics: 2 for the hierarchical-B plan of stream(pattern="RA")
        self.plan = None
        self.max_merge = 3
        self.stats = []
        self.rng = np.random.default_rng(seed)
        self.off, self.init_rows = load_contexts()
        src = open(os.path.join(REF, "libavcodec", "hevc.c")).read()      # 4:2:2 chroma mode mapping (8.4.3), from the decoder's own table
        body = src[src.index("tab_mode_idx[]"):]
        self.tab_mode_idx = [int(v) for v in re.findall(r"\d+", body[body.index("{") + 1:body.index("}")])]
        assert len(self.tab_mode_idx) == 35
        self.min_cb_log2, self.min_tb_log2, self.max_tb_log2 = 3, 2, 5
        self.max_th_depth_intra = 2

    # ---- parameter sets -------------------------------------------------------------------------------------
    def ptl(self, w):
        prof = 4 if getattr(self, "cfi", 1) >= 2 else (2 if self.bd > 8 else 1)   # Main / Main10 / format range extensions
        w.u(2, 0); w.u(1, 0); w.u(5, prof)                                 # profile space, tier, profile idc
        for i in range(32):
            w.u(1, 1 if (i in (1, 2) and prof != 4) or (i == 4 and prof == 4) else 0)
        w.u(1, 1); w.u(1, 0); w.u(1, 0); w.u(1, 1)                        # progressive, interlaced, non-packed, frame-only
        w.u(16, 0); w.u(16, 0); w.u(12, 0)
        w.u(8, 153)                                                        # level 5.1

    def vps(self):
        w = BitWriter()
        w.u(4, 0); w.u(2, 3); w.u(6, 0); w.u(3, 0); w.u(1, 1); w.u(16, 0xFFFF)
        self.ptl(w)
        w.u(1, 1); w.ue(4); w.ue(self.reorder); w.ue(0)                   # sub_layer_ordering_info, dpb 5, reorder, latency
        w.u(6, 0); w.ue(0)                                                 # max_layer_id, num_layer_sets_minus1
        w.u(1, 0)                                                          # timing info
        w.u(1, 0)                                                          # extension
        w.trailing()
        return nal(32, w.bytes())

    def sps(self):
        w = BitWriter()
        w.u(4, 0); w.u(3, 0); w.u(1, 1)
        self.ptl(w)
        w.ue(0)                                                            # sps id
        w.ue(self.cfi)                                                     # chroma_format_idc
        if self.cfi == 3:
            w.u(1, 0)                                                      # separate_colour_plane_flag (hevc_ps.c:1597)
        w.ue(self.W); w.ue(self.H)
        if self.conf_win:                                                  # conformance window: offsets in chroma sample units
            sw, sh = (1 if self.cfi == 3 else 2), (2 if self.cfi == 1 else 1)
            w.u(1, 1)
            for v, unit in zip(self.conf_win, (sw, sw, sh, sh)):
                w.ue(v // unit)
        else:
            w.u(1, 0)
        w.ue(self.bd - 8); w.ue(self.bd - 8)
        w.ue(4)                                                            # log2_max_poc_lsb - 4
        w.u(1, 1); w.ue(4); w.ue(self.reorder); w.ue(0)                   # sub_layer_ordering_info: dpb 5, num_reorder, latency
        w.ue(self.min_cb_log2 - 3); w.ue(self.ctb_log2 - self.min_cb_log2)
        w.ue(self.min_tb_log2 - 2); w.ue(self.max_tb_log2 - self.min_tb_log2)
        w.ue(2); w.ue(self.max_th_depth_intra)                             # max_transform_hierarchy_depth inter / intra
        w.u(1, 0)                                                          # scaling lists
        w.u(1, 1 if self.amp else 0)                                       # amp_enabled_flag
        w.u(1, 1 if self.sao else 0)                                       # sample_adaptive_offset_enabled
        w.u(1, int(self.pcm > 0))                                          # pcm_enabled_flag
        if self.pcm > 0:
            w.u(4, self.bd - 1); w.u(4, self.bd - 1)                       # pcm sample bit depth luma / chroma (minus 1): full depth
            w.ue(0); w.ue(2)                                               # log2_min_pcm_cb_size - 3 (8), log2_diff_max_min (.. 32)
            w.u(1, int(self.pcm_lf_off))                                   # pcm_loop_filter_disabled_flag
        w.ue(0)                                                            # num_short_term_ref_pic_sets
        w.u(1, 0)                                                          # long term refs
        w.u(1, int(self.tmvp))                                             # sps_temporal_mvp_enabled_flag
        w.u(1, 1)                                                          # strong intra smoothing
        w.u(1, 0)                                                          # vui
        w.u(1, 0)                                                          # extension
        w.trailing()
        return nal(33, w.bytes())

    def pps(self):
        w = BitWriter()
        w.ue(0); w.ue(0)
        w.u(1, 0); w.u(1, 0); w.u(3, 0)                                    # dependent slices, output flag, extra bits
        w.u(1, 0)                                                          # sign data hiding
        w.u(1, 0)                                                          # cabac_init_present
        w.ue(0); w.ue(0)
        w.se(0)                                                            # init_qp_minus26
        w.u(1, int(self.cip))                                              # constrained intra pred
        w.u(1, int(self.tskip > 0))                                        # transform skip (log2_max_transform_skip_block_size = 2)
        w.u(1, int(self.qpd))                                              # cu_qp_delta_enabled_flag
        if self.qpd:
            w.ue(max(self.ctb_log2 - 5, 0))                                # diff_cu_qp_delta_depth
        w.se(self.chroma_qp_offsets[0]); w.se(self.chroma_qp_offsets[1])   # pps_cb_qp_offset / pps_cr_qp_offset
        w.u(1, 0)                                                          # slice chroma qp offsets present
        w.u(1, int(self.weighted)); w.u(1, int(self.weighted))             # weighted pred / bipred
        w.u(1, int(self.tqb > 0))                                          # transquant bypass
        w.u(1, int(bool(self.tiles))); w.u(1, int(self.wpp))               # tiles, entropy_coding_sync (WPP)
        if self.tiles:
            w.ue(self.tiles[0] - 1); w.ue(self.tiles[1] - 1)               # num_tile_columns_minus1, num_tile_rows_minus1
            w.u(1, 1)                                                      # uniform_spacing_flag
            w.u(1, int(self.lf_across_tiles))                              # loop_filter_across_tiles_enabled_flag
        w.u(1, 1)                                                          # loop filter across slices
        if self.no_dbk:
            w.u(1, 1); w.u(1, 0); w.u(1, 1)                                # deblocking_filter_control_present, override_enabled = 0, pps_deblocking_filter_disabled = 1
        elif self.dbk_offsets != (0, 0):
            w.u(1, 1); w.u(1, 0); w.u(1, 0)                                # deblocking_filter_control_present, override_enabled = 0, pps_deblocking_filter_disabled = 0
            w.se(self.dbk_offsets[0]); w.se(self.dbk_offsets[1])           # pps_beta_offset_div2, pps_tc_offset_div2 (hevc_ps.c:2354-2363)
        else:
            w.u(1, 0)                                                      # deblocking filter control present
        w.u(1, 0)                                                          # scaling list data
        w.u(1, 0)                                                          # lists modification
        w.ue(0)                                                            # log2_parallel_merge_level - 2
        w.u(1, 0)                                                          # slice header extension
        if self.ccp:
            w.u(1, 1); w.u(1, 1); w.u(7, 0)                                # pps_extension_present, pps_range_extensions_flag, 7 more (hevc_ps.c:2421-2423)
            if self.tskip > 0:
                w.ue(0)                                                    # log2_max_transform_skip_block_size_minus2
            w.u(1, 1)                                                      # cross_component_prediction_enabled_flag
            w.u(1, 0)                                                      # chroma_qp_offset_list_enabled_flag
            w.ue(0); w.ue(0)                                               # log2_sao_offset_scale_luma / _chroma
        else:
            w.u(1, 0)                                                      # pps extension
        w.trailing()
        return nal(34, w.bytes())

    # ---- slice ----------------------------------------------------------------------------------------------------
    def slice_nal(self, pic=0, slice_type=2):
        """all slices of one picture.  pic: decode-order index (== POC, low-delay); slice_type 2 I (IDR when pic == 0), 1 P, 0 B"""
        ctb = 1 << self.ctb_log2
        self.cw, self.ch = (self.W + ctb - 1) >> self.ctb_log2, (self.H + ctb - 1) >> self.ctb_log2
        self.ct_depth = np.zeros((self.H >> 3, self.W >> 3), np.int32)
        self.ipm = np.ones((self.H >> 2, self.W >> 2), np.int32)           # INTRA_DC default
        self.skip = np.zeros((self.H >> 3, self.W >> 3), np.int32)
        self.cnt = dict(intra_pred=0, transform_add=0, pu=0)
        nsl = max(1, min(self.slices, self.ch))
        rows = [(j * self.ch) // nsl for j in range(nsl + 1)]             # slice j covers CTB rows rows[j] .. rows[j + 1] - 1
        out = b""
        for j in range(nsl):
            out += self.one_slice(pic, slice_type, rows[j] * self.cw, rows[j + 1] * self.cw)
        self.stats.append(dict(self.cnt))
        return out

    def one_slice(self, pic, slice_type, ctb_start, ctb_end):
        self.slice_type = slice_type
        self.slice_start = ctb_start
        idr = pic == 0
        plan = self.plan[pic] if self.plan else None       # random access: POC and reference picture set from the GOP plan
        poc = plan["poc"] if plan else pic
        if plan and not idr:
            ntot = len(plan["neg"]) + len(plan["pos"])
            nref = min(ntot, 2)
        else:
            nref = 0 if slice_type == 2 else min(pic, 2)
        self.nrefs = [nref, nref if slice_type == 0 else 0]
        w = BitWriter()
        w.u(1, int(ctb_start == 0))                                        # first_slice_segment_in_pic
        if idr:
            w.u(1, 0)                                                      # no_output_of_prior_pics (IRAP)
        w.ue(0)                                                            # pps id
        if ctb_start:
            w.u(max(1, (self.cw * self.ch - 1).bit_length()), ctb_start)   # slice_segment_address, Ceil(Log2(PicSizeInCtbsY)) bits
        w.ue(slice_type)
        if not idr:
            w.u(8, poc & 255)                                              # pic_order_cnt_lsb
            w.u(1, 0)                                                      # short_term_ref_pic_set_sps_flag
            if plan:
                w.ue(len(plan["neg"])); w.ue(len(plan["pos"]))             # num_negative_pics, num_positive_pics
                prev = poc
                for q in plan["neg"]:                                      # closest first
                    w.ue(prev - q - 1); w.u(1, 1); prev = q                # delta_poc_s0_minus1, used_by_curr_pic_s0
                prev = poc
                for q in plan["pos"]:
                    w.ue(q - prev - 1); w.u(1, 1); prev = q                # delta_poc_s1_minus1, used_by_curr_pic_s1
            else:
                nneg = min(pic, 2)
                w.ue(nneg); w.ue(0)                                        # num_negative_pics, num_positive_pics
                for _ in range(nneg):
                    w.ue(0); w.u(1, 1)                                     # delta_poc_s0_minus1, used_by_curr_pic
        if self.tmvp and not idr:
            w.u(1, 1)                                                      # slice_temporal_mvp_enabled_flag
        if self.sao:
            w.u(1, int(self.sao_planes != "chroma")); w.u(1, int(self.sao_planes != "luma"))   # slice_sao_luma_flag / slice_sao_chroma_flag
        if slice_type != 2:
            w.u(1, 1)                                                      # num_ref_idx_active_override_flag
            w.ue(nref - 1)
            if slice_type == 0:
                w.ue(nref - 1)
                w.u(1, 0)                                                  # mvd_l1_zero_flag
            if self.tmvp and not idr:
                col_l0 = 1
                if slice_type == 0:
                    col_l0 = int(self.rng.integers(0, 2))
                    w.u(1, col_l0)                                         # collocated_from_l0_flag
                if nref > 1:
                    w.ue(int(self.rng.integers(0, nref)))                  # collocated_ref_idx
            if self.weighted:
                self.pred_weight_table(w)
            w.ue(5 - self.max_merge)                                       # five_minus_max_num_merge_cand
        w.se(self.qp - 26)                                                 # slice_qp_delta
        if self.sao or not self.no_dbk:                                    # hevc.c:990-994
            w.u(1, int(self.lf_across_slices))                             # slice_loop_filter_across_slices_enabled
        self.c = Cabac(self.init_rows[2 - slice_type], self.qp)
        self.substreams = []
        self.slice_data(ctb_start, ctb_end)
        self.substreams.append(self.c.bits)
        data = bytearray()
        ends = []
        for bits in self.substreams:                                       # every substream ends byte aligned (9.3.2.5 / 7.3.8.1)
            bits = bits + [0] * (-len(bits) % 8)
            wb = BitWriter(); wb.bits = bits
            data += wb.bytes()
            ends.append(len(data))
        if self.wpp or self.tiles:
            # entry points count the bytes of the NAL unit INCLUDING emulation prevention bytes (7.4.7.1); the header
            # ends in a non-zero byte (alignment bit), so the zero run restarts at the first byte of the slice data
            pos, zeros, n = [0], 0, 0
            for b in data:
                if zeros >= 2 and b <= 3:
                    n += 1; zeros = 0
                n += 1
                zeros = zeros + 1 if b == 0 else 0
                pos.append(n)
            sizes = [pos[e] - pos[st] for st, e in zip([0] + ends[:-1], ends)]
            w.ue(len(sizes) - 1)                                           # num_entry_point_offsets
            if len(sizes) > 1:
                w.ue(31)                                                   # offset_len_minus1
                for sz in sizes[:-1]:
                    w.u(32, sz - 1)                                        # entry_point_offset_minus1
        w.bits.append(1)                                                   # byte_alignment()
        while len(w.bits) % 8:
            w.bits.append(0)
        return nal(19 if idr else 1, w.bytes() + bytes(data))              # IDR_W_RADL / TRAIL_R

    def pred_weight_table(self, w):
        r = self.rng
        w.ue(int(r.integers(0, 8)))                                        # luma_log2_weight_denom
        w.se(0)                                                            # delta_chroma_log2_weight_denom
        for l in range(2 if self.slice_type == 0 else 1):
            n = self.nrefs[l]
            lf = [int(r.random() < 0.7) for _ in range(n)]
            cf = [int(r.random() < 0.7) for _ in range(n)]
            for f in lf:
                w.u(1, f)
            for f in cf:
                w.u(1, f)
            for i in range(n):
                if lf[i]:
                    w.se(int(r.integers(-20, 21))); w.se(int(r.integers(-10, 11)))
                if cf[i]:
                    for _ in range(2):
                        w.se(int(r.integers(-20, 21))); w.se(int(r.integers(-20, 21)))

    def slice_data(self, ctb_start=0, ctb_end=None):
        n = self.cw * self.ch
        ctb_end = n if ctb_end is None else ctb_end
        saved = None
        # CTB order: raster, or tile scan (6.5.1) with uniformly spaced tiles; tile_x0 / tile_y0 = first CTB column / row of the
        # tile a CTB belongs to (neighbours outside the tile are unavailable, 6.4.1)
        if self.tiles:
            ncol, nrow = self.tiles
            cb = [(i * self.cw) // ncol for i in range(ncol + 1)]
            rb = [(j * self.ch) // nrow for j in range(nrow + 1)]
            order = [(x, y, cb[i], rb[j], cb[i + 1]) for j in range(nrow) for i in range(ncol) for y in range(rb[j], rb[j + 1]) for x in range(cb[i], cb[i + 1])]
        else:
            order = [(a % self.cw, a // self.cw, 0, 0, self.cw) for a in range(n)]
        for a in range(ctb_start, ctb_end):
            self.rx, self.ry, self.tile_x0, self.tile_y0, tile_x1 = order[a]
            tw = tile_x1 - self.tile_x0                                    # width of the tile (of the picture without tiles) in CTBs
            tile_start = self.tiles and (self.rx, self.ry) == (self.tile_x0, self.tile_y0)
            if tile_start and a:
                # first CTB of a tile: new substream, the arithmetic coder and the contexts start afresh (9.3.1)
                self.substreams.append(self.c.bits)
                self.c = Cabac(self.init_rows[2 - self.slice_type], self.qp)
            elif self.wpp and self.rx == self.tile_x0 and a:
                # new substream (a CTB row of the picture, or of the tile): arithmetic coder restarts, contexts come from the state
                # stored after the 2nd CTB of the row above (9.3.1: synchronization; a row one CTB wide re-initialises instead,
                # hevc_cabac.c:647-650)
                self.substreams.append(self.c.bits)
                fresh = Cabac(self.init_rows[2 - self.slice_type], self.qp)
                if tw > 1:
                    fresh.state = [list(st) for st in saved]
                self.c = fresh
            if self.sao:
                self.sao_syntax()
            self.quadtree(self.rx << self.ctb_log2, self.ry << self.ctb_log2, self.ctb_log2, 0)
            self.c.terminate(1 if a == ctb_end - 1 else 0)                 # end_of_slice_segment_flag
            row_end = False
            if self.wpp:
                if self.rx == self.tile_x0 + 1 or tw == 1:
                    saved = [list(st) for st in self.c.state]              # storage process after the 2nd CTB of a row (hevc_cabac.c:552-560)
                if self.rx == tile_x1 - 1 and a != ctb_end - 1:
                    self.c.terminate(1)                                    # end_of_subset_one_bit, then byte_alignment()
                    row_end = True
            if self.tiles and not row_end and a != ctb_end - 1 and order[a + 1][:2] == order[a + 1][2:4]:
                self.c.terminate(1)                                        # last CTB of a tile: end_of_subset_one_bit

    def left_ok(self, x0):
        """is the block to the left of luma column x0 available (same tile; one slice per picture)?  lc->ctb_left_flag || x0b"""
        return (x0 & ((1 << self.ctb_log2) - 1)) != 0 or self.ctb_left_ok()

    def up_ok(self, y0):
        return (y0 & ((1 << self.ctb_log2) - 1)) != 0 or self.ctb_up_ok()

    def ctb_left_ok(self):
        """lc->ctb_left_flag (hls_decode_neighbour, hevc.c): the CTB to the left exists, in this tile and in this slice"""
        return self.rx > self.tile_x0 and self.ry * self.cw + self.rx - 1 >= self.slice_start

    def ctb_up_ok(self):
        return self.ry > self.tile_y0 and (self.ry - 1) * self.cw + self.rx >= self.slice_start

    def sao_syntax(self):
        c, r, o = self.c, self.rng, self.off
        if self.ctb_left_ok():
            m = int(r.random() < 0.2)
            c.encode(o["sao_merge_flag"], m)
            if m:
                return
        if self.ctb_up_ok():
            m = int(r.random() < 0.2)
            c.encode(o["sao_merge_flag"], m)
            if m:
                return
        for cidx in range(2):                                              # Cr shares type / class with Cb
            if (cidx == 0 and self.sao_planes == "chroma") or (cidx == 1 and self.sao_planes == "luma"):
                continue                                                   # hevc.c:1133-1136: not applied, nothing coded
            t = int(r.choice([0, 1, 2], p=[0.3, 0.3, 0.4]))
            c.encode(o["sao_type_idx"], int(t != 0))
            if t:
                c.bypass(0 if t == 1 else 1)
            planes = [0] if cidx == 0 else [1, 2]
            if not t:
                continue
            for p in planes:
                maxv = (1 << (min(self.bd, 10) - 5)) - 1
                absv = [int(r.integers(0, maxv + 1)) for _ in range(4)]
                for v in absv:
                    for k in range(v):
                        c.bypass(1)
                    if v < maxv:
                        c.bypass(0)
                if t == 1:
                    for v in absv:
                        if v:
                            c.bypass(int(r.integers(0, 2)))
                    c.bypass_bits(5, int(r.integers(0, 32)))
                elif p != 2:
                    c.bypass_bits(2, int(r.integers(0, 4)))

    def quadtree(self, x0, y0, log2, depth):
        c, o = self.c, self.off
        size = 1 << log2
        if self.qpd and log2 >= min(self.ctb_log2, 5):
            self.qp_coded = 0                                               # new quantisation group (hevc.c:2525-2529)
        if x0 + size <= self.W and y0 + size <= self.H and log2 > self.min_cb_log2:
            inc = 0
            if self.left_ok(x0):
                inc += int(self.ct_depth[y0 >> 3, (x0 >> 3) - 1] > depth)
            if self.up_ok(y0):
                inc += int(self.ct_depth[(y0 >> 3) - 1, x0 >> 3] > depth)
            split = int(self.rng.random() < {6: 0.9, 5: 0.65, 4: 0.45}[log2] * (1 - 0.45 * self.calm))
            c.encode(o["split_coding_unit_flag"] + inc, split)
        else:
            split = int(log2 > self.min_cb_log2)
        if split:
            h = size >> 1
            for dx, dy in ((0, 0), (h, 0), (0, h), (h, h)):
                if x0 + dx < self.W and y0 + dy < self.H:
                    self.quadtree(x0 + dx, y0 + dy, log2 - 1, depth + 1)
        else:
            self.coding_unit(x0, y0, log2, depth)

    def mpm_candidates(self, x0, y0):
        ctb = 1 << self.ctb_log2
        left = self.ipm[y0 >> 2, (x0 >> 2) - 1] if self.left_ok(x0) else 1
        up = self.ipm[(y0 >> 2) - 1, x0 >> 2] if (y0 > 0 and (y0 - 1) >= (y0 // ctb) * ctb) else 1
        if left == up:
            if left < 2:
                return [0, 1, 26]
            return [left, 2 + ((left - 2 - 1 + 32) & 31), 2 + ((left - 2 + 1) & 31)]
        cand = [left, up]
        if 0 not in cand:
            cand.append(0)
        elif 1 not in cand:
            cand.append(1)
        else:
            cand.append(26)
        return cand

    def mvd(self):
        c, o, r = self.c, self.off, self.rng
        v = [int(r.choice([0, 1, 2, 3, 5, 9, 17, 40], p=[0.3, 0.2, 0.15, 0.1, 0.1, 0.07, 0.05, 0.03])) for _ in range(2)]
        for a in v:
            c.encode(o["abs_mvd_greater0_flag"], int(a > 0))
        for a in v:
            if a:
                c.encode(o["abs_mvd_greater1_flag"] + 1, int(a > 1))
        for a in v:
            if a > 1:                                                      # abs_mvd_minus2, EG1
                t, k = a - 2, 1
                while t >= (1 << k):
                    c.bypass(1)
                    t -= 1 << k
                    k += 1
                c.bypass(0)
                c.bypass_bits(k, t)
            if a:
                c.bypass(int(r.integers(0, 2)))                            # mvd_sign_flag

    def prediction_unit(self, w, h, depth, skipped):
        """syntax of one PU; returns merge_flag"""
        c, o, r = self.c, self.off, self.rng

        def merge_idx():
            if self.max_merge > 1:
                idx = int(r.integers(0, self.max_merge))
                c.encode(o["merge_idx"], int(idx > 0))
                if idx > 0:
                    for k in range(1, self.max_merge - 1):
                        c.bypass(int(idx > k))
                        if idx <= k:
                            break
        self.cnt["pu"] += 1
        if skipped:
            merge_idx()
            return 1
        merge = int(r.random() < 0.35)
        c.encode(o["merge_flag"], merge)
        if merge:
            merge_idx()
            return 1
        idc = 0                                                            # PRED_L0
        if self.slice_type == 0:
            if w + h == 12:
                idc = int(r.integers(0, 2))
                c.encode(o["inter_pred_idc"] + 4, idc)
            else:
                bi = int(r.random() < 0.55)
                c.encode(o["inter_pred_idc"] + depth, bi)
                if bi:
                    idc = 2
                else:
                    idc = int(r.integers(0, 2))
                    c.encode(o["inter_pred_idc"] + 4, idc)
        for l in range(2):
            if (l == 0 and idc == 1) or (l == 1 and idc == 0):
                continue
            n = self.nrefs[l]
            ref = int(r.integers(0, n))
            mx = n - 1
            i = 0
            while i < min(mx, 2):                                          # ref_idx_lX: two context bins, then bypass
                c.encode(o["ref_idx_l0"] + i, int(ref > i))
                if ref <= i:
                    break
                i += 1
            if i == 2 and ref >= 2:
                while i < mx:
                    c.bypass(int(ref > i))
                    if ref <= i:
                        break
                    i += 1
            self.mvd()
            c.encode(o["mvp_lx_flag"], int(r.integers(0, 2)))
        return 0

    def coding_unit(self, x0, y0, log2, depth):
        c, o, r = self.c, self.off, self.rng
        size = 1 << log2
        self.cu_bypass = 0
        if self.tqb > 0:                                                    # cu_transquant_bypass_flag (hevc.c:2371-2374): the residual is
            self.cu_bypass = int(r.random() < self.tqb)                    # added untransformed, deblocking / SAO leave the CU alone
            c.encode(o["cu_transquant_bypass_flag"], self.cu_bypass)
        if self.slice_type != 2:
            inc = 0
            if self.left_ok(x0):
                inc += int(self.skip[y0 >> 3, (x0 >> 3) - 1] != 0)
            if self.up_ok(y0):
                inc += int(self.skip[(y0 >> 3) - 1, x0 >> 3] != 0)
            skipped = int(r.random() < 0.25 + 0.5 * self.calm)
            c.encode(o["skip_flag"] + inc, skipped)
            self.skip[y0 >> 3:(y0 + size) >> 3, x0 >> 3:(x0 + size) >> 3] = skipped
            self.ct_depth[y0 >> 3:(y0 + size) >> 3, x0 >> 3:(x0 + size) >> 3] = depth
            if skipped:
                self.prediction_unit(size, size, depth, True)
                self.ipm[y0 >> 2:(y0 + size) >> 2, x0 >> 2:(x0 + size) >> 2] = 1
                return
            intra = int(r.random() < 0.2 - 0.15 * self.calm)
            c.encode(o["pred_mode"], intra)
            if not intra:
                self.ipm[y0 >> 2:(y0 + size) >> 2, x0 >> 2:(x0 + size) >> 2] = 1
                u = r.random()
                part = 0 if u < 0.6 else (1 if u < 0.8 else 2)             # 2Nx2N, 2NxN, Nx2N (no inter NxN at 8x8)
                c.encode(o["part_mode"], int(part == 0))
                pus = {0: [(size, size)], 1: [(size, size // 2)] * 2, 2: [(size // 2, size)] * 2}[part]
                if part:
                    c.encode(o["part_mode"] + 1, int(part == 1))
                    if self.amp and log2 > self.min_cb_log2:                # hevc_cabac.c:863-875
                        asym = int(r.integers(0, 3))                       # 0 = symmetric, 1 = small part first (nU / nL), 2 = small part last (nD / nR)
                        c.encode(o["part_mode"] + 3, int(asym == 0))
                        if asym:
                            c.bypass(int(asym == 2))
                            q = size // 4
                            a, b = (q, size - q) if asym == 1 else (size - q, q)
                            pus = [(size, a), (size, b)] if part == 1 else [(a, size), (b, size)]
                merge = 0
                for (pw_, ph_) in pus:
                    merge = self.prediction_unit(pw_, ph_, depth, False)
                root = 1
                if not (part == 0 and merge):
                    root = int(r.random() < 0.7 - 0.35 * self.calm)
                    c.encode(o["no_residual_data_flag"], root)
                if root:
                    self.inter = True
                    self.transform_tree(x0, y0, log2, 0, 0, 0, [1], 1, [0, 0], 2, 1)
                    self.inter = False
                return
        nxn = 0
        if log2 == self.min_cb_log2:
            nxn = int(r.random() < 0.35)
            c.encode(o["part_mode"], 1 - nxn)                              # bin 1 = PART_2Nx2N
        if self.pcm > 0 and not nxn and 3 <= log2 <= 5:
            # pcm_flag is a terminate bin (hevc.c:2406-2411); when set: the arithmetic codeword is flushed, the stream is byte
            # aligned, the samples follow raw (luma, Cb, Cr; hls_pcm_sample, hevc.c:1587-1623), and the arithmetic engine --
            # not the contexts -- starts afresh (9.3.2.5)
            is_pcm = int(r.random() < self.pcm)
            c.terminate(is_pcm)
            if is_pcm:
                c.bits += [0] * (-len(c.bits) % 8)                         # pcm_alignment_zero_bit
                for npix in (size * size, (size >> 1) ** 2, (size >> 1) ** 2):
                    for v in r.integers(0, 1 << self.bd, npix):
                        c.bits += [(int(v) >> k) & 1 for k in range(self.bd - 1, -1, -1)]
                c.low, c.range, c.outstanding, c.first = 0, 510, 0, True
                self.ipm[y0 >> 2:(y0 + size) >> 2, x0 >> 2:(x0 + size) >> 2] = 1          # INTRA_DC for the neighbours' candidates
                self.ct_depth[y0 >> 3:(y0 + size) >> 3, x0 >> 3:(x0 + size) >> 3] = depth
                return
        parts = [(0, 0), (4, 0), (0, 4), (4, 4)] if nxn else [(0, 0)]
        pb = size >> nxn
        prev = [int(r.random() < 0.6) for _ in parts]
        for f in prev:
            c.encode(o["prev_intra_luma_pred_mode"], f)
        modes = []
        for (dx, dy), f in zip(parts, prev):
            cand = self.mpm_candidates(x0 + dx, y0 + dy)
            if f:
                idx = int(r.integers(0, 3))
                c.bypass(int(idx > 0))
                if idx > 0:
                    c.bypass(int(idx > 1))
                mode = cand[idx]
            else:
                rem = int(r.integers(0, 32))
                c.bypass_bits(5, rem)
                mode = rem
                for cv in sorted(cand):
                    if mode >= cv:
                        mode += 1
            modes.append(int(mode))
            self.ipm[(y0 + dy) >> 2:(y0 + dy + pb) >> 2, (x0 + dx) >> 2:(x0 + dx + pb) >> 2] = mode
        table = [0, 26, 10, 1]
        modes_c, cms = [], []
        for m in (modes if self.cfi == 3 else modes[:1]):                   # 4:4:4: one intra_chroma_pred_mode per luma block (hevc.c:2270-2283)
            cm = int(r.integers(0, 5))                                     # intra_chroma_pred_mode (4 = derived from luma)
            c.encode(o["intra_chroma_pred_mode"], int(cm != 4))
            if cm != 4:
                c.bypass_bits(2, cm)
            modes_c.append(m if cm == 4 else (34 if m == table[cm] else table[cm]))
            cms.append(cm)
        mode_c = modes_c[0]
        if self.cfi == 2:
            mode_c = self.tab_mode_idx[mode_c]                              # 4:2:2: process of 8.4.3, table read from hevc.c:2252
        self.modes_c, self.cms, self.cm_tu = modes_c, cms, cms[0]
        self.ct_depth[y0 >> 3:(y0 + size) >> 3, x0 >> 3:(x0 + size) >> 3] = depth
        self.transform_tree(x0, y0, log2, 0, 0, nxn, modes, mode_c, [0, 0], self.max_th_depth_intra + nxn, modes[0])

    def transform_tree(self, x0, y0, log2, tdepth, blk, nxn, modes, mode_c, parent_cbf_c, max_depth, mode):
        c, o, r = self.c, self.off, self.rng
        if nxn and tdepth == 1:
            mode = modes[blk]                                               # lc->tu.intra_pred_mode of this quadrant (hevc.c:1452)
            if self.cfi == 3:
                mode_c = self.modes_c[blk]                                  # ... and its own chroma mode at 4:4:4 (hevc.c:1463-1465)
                self.cm_tu = self.cms[blk]
        if log2 <= self.max_tb_log2 and log2 > self.min_tb_log2 and tdepth < max_depth and not (nxn and tdepth == 0):
            split = int(r.random() < 0.3)
            c.encode(o["split_transform_flag"] + 5 - log2, split)
        else:
            split = int(log2 > self.max_tb_log2 or (nxn and tdepth == 0))
        # cbf_cb / cbf_cr (hevc.c:1491-1513): one flag per component, two at 4:2:2 (upper / lower square) unless the node splits
        # further above 8x8; a node is only asked when its parent's first flag was set
        nblk = 2 if self.cfi == 2 else 1
        if tdepth == 0 and not isinstance(parent_cbf_c[0], list):
            parent_cbf_c = [[0, 0], [0, 0]]
        cbf_c = [list(parent_cbf_c[0]), list(parent_cbf_c[1])]
        if log2 > 2 or self.cfi == 3:                                       # hevc.c:1493
            for k in range(2):
                if tdepth == 0 or parent_cbf_c[k][0]:
                    cbf_c[k][0] = int(r.random() < 0.5 - 0.3 * self.calm)
                    c.encode(o["cbf_cb, cbf_cr"] + tdepth, cbf_c[k][0])
                    if self.cfi == 2 and (not split or log2 == 3):
                        cbf_c[k][1] = int(r.random() < 0.5 - 0.3 * self.calm)
                        c.encode(o["cbf_cb, cbf_cr"] + tdepth, cbf_c[k][1])
        if split:
            h = 1 << (log2 - 1)
            for i, (dx, dy) in enumerate(((0, 0), (h, 0), (0, h), (h, h))):
                self.transform_tree(x0 + dx, y0 + dy, log2 - 1, tdepth + 1, i, nxn, modes, mode_c, cbf_c, max_depth, mode)
            return
        inter = getattr(self, "inter", False)
        if inter and tdepth == 0 and not any(cbf_c[0][:nblk] + cbf_c[1][:nblk]):
            cbf_luma = 1                                                    # inferred (7.3.8.8)
        else:
            cbf_luma = int(r.random() < 0.7 - 0.3 * self.calm)
            c.encode(o["cbf_luma"] + (1 if tdepth == 0 else 0), cbf_luma)

        if self.qpd and not self.qp_coded and (cbf_luma or cbf_c[0][0] or cbf_c[1][0] or (self.cfi == 2 and (cbf_c[0][1] or cbf_c[1][1]))):
            d = int(r.integers(-4, 5))                                      # cu_qp_delta_abs: prefix only (< 5), hevc_cabac.c:731-755
            for i in range(abs(d)):
                c.encode(o["cu_qp_delta"] + (1 if i else 0), 1)
            c.encode(o["cu_qp_delta"] + (1 if d else 0), 0)
            if d:
                c.bypass(int(d < 0))                                        # cu_qp_delta_sign_flag
            self.qp_coded = 1

        def scan_of(m, lg):
            if lg < 4 and not inter:
                if 6 <= m <= 14:
                    return 2
                if 22 <= m <= 30:
                    return 1
            return 0
        chroma_here = log2 > 2 or blk == 3 or self.cfi == 3                 # 4x4 luma: the chroma of the 8x8 parent comes with block 3 (not at 4:4:4)
        flags = cbf_c if (log2 > 2 or self.cfi == 3) else parent_cbf_c
        if not inter:
            self.cnt["intra_pred"] += 1 + (2 * nblk if chroma_here else 0)
        self.cnt["transform_add"] += cbf_luma + (sum(flags[0][:nblk]) + sum(flags[1][:nblk]) if chroma_here else 0)
        if cbf_luma:
            self.residual(log2, scan_of(mode, log2) if log2 < 4 else 0, 0)
        if chroma_here:
            log2_c = log2 if self.cfi == 3 else (log2 - 1 if log2 > 2 else 2)
            # cross-component prediction (hevc.c:1295-1300): chroma residual += (res_scale_val * luma residual) >> 3
            cross = bool(self.ccp and cbf_luma and (inter or self.cm_tu == 4))
            for k in range(2):                                              # Cb blocks, then Cr blocks (hevc.c:1302-1362)
                if cross:
                    v = int(r.choice([0, 1, 2, 3, 4], p=[0.2, 0.2, 0.2, 0.2, 0.2]))          # log2_res_scale_abs_plus1 (hevc_cabac.c:1056-1063)
                    for i in range(v):
                        c.encode(o["log2_res_scale_abs"] + 4 * k + i, 1)
                    if v < 4:
                        c.encode(o["log2_res_scale_abs"] + 4 * k + v, 0)
                    if v:
                        c.encode(o["res_scale_sign_flag"] + k, int(r.random() < 0.5))
                for i in range(nblk):
                    if flags[k][i]:
                        self.residual(log2_c, scan_of(mode_c, log2) if log2 < 4 else 0, k + 1)
                    elif cross:
                        self.cnt["transform_add"] += 1                       # the scaled luma residual alone is added (hevc.c:1314-1329)

    def residual(self, log2, scan_idx, cidx):
        c, o, r = self.c, self.off, self.rng
        n = 1 << log2
        # random sparse levels, low frequencies more likely
        lev = np.zeros((n, n), np.int64)
        yy, xx = np.mgrid[0:n, 0:n]
        mask = r.random((n, n)) < np.exp(-(xx + yy) / (r.uniform(0.7, 0.7 + n / 4.0) * (1 - 0.7 * self.calm)))
        mags = np.maximum(1, np.rint(np.abs(r.laplace(0, 2.5, (n, n))))).astype(np.int64)
        big = r.random((n, n)) < 0.03
        mags = np.where(big, mags * int(r.integers(5, 60)), mags)
        lev = np.where(mask, mags * np.where(r.random((n, n)) < 0.5, -1, 1), 0)
        if not lev.any():
            lev[0, 0] = int(r.choice([-2, -1, 1, 3]))
        if self.tskip > 0 and log2 == 2 and not self.cu_bypass:            # transform_skip_flag (hevc_cabac.c:1443-1446): first element of
            c.encode(o["transform_skip_flag[][]"] + (1 if cidx else 0), int(r.random() < self.tskip))   # residual_coding()
        sb_order, pos_order = scan_tables(log2, scan_idx)
        # scan position list (sub-block index i, position n) in forward order
        def coord(i, k):
            return (sb_order[i][0] << 2) + pos_order[k][0], (sb_order[i][1] << 2) + pos_order[k][1]
        last_i = last_k = -1
        for i in range(len(sb_order)):
            for k in range(16):
                x, y = coord(i, k)
                if lev[y, x]:
                    last_i, last_k = i, k
        lx, ly = coord(last_i, last_k)
        if scan_idx == 2:
            lx, ly = ly, lx                                                # coded swapped for the vertical scan
        # last_sig_coeff prefix / suffix
        def prefix_of(v):
            if v < 4:
                return v, 0, 0
            k = v.bit_length() - 1                                          # 1 << k <= v
            p = 2 * k + (1 if v >= (3 << (k - 1)) else 0)
            base = (1 << ((p >> 1) - 1)) * (2 + (p & 1))
            return p, v - base, (p >> 1) - 1
        if cidx == 0:
            ctx_off, ctx_shift = 3 * (log2 - 2) + ((log2 - 1) >> 2), (log2 + 1) >> 2
        else:
            ctx_off, ctx_shift = 15, log2 - 2
        maxp = (log2 << 1) - 1
        px, sx, nsx = prefix_of(lx)
        py, sy, nsy = prefix_of(ly)
        for name, p in (("last_significant_coeff_x_prefix", px), ("last_significant_coeff_y_prefix", py)):
            for i in range(p):
                c.encode(o[name] + (i >> ctx_shift) + ctx_off, 1)
            if p < maxp:
                c.encode(o[name] + (p >> ctx_shift) + ctx_off, 0)
        if px > 3:
            c.bypass_bits(nsx, sx)
        if py > 3:
            c.bypass_bits(nsy, sy)
        nsb = 1 << (log2 - 2)
        csbf = np.zeros((nsb + 1, nsb + 1), np.int32)
        greater1_ctx = 1
        for i in range(last_i, -1, -1):
            xs, ys = sb_order[i]
            sig = [(k, coord(i, k)) for k in range(16)]
            nz = [k for k, (x, y) in sig if lev[y, x]]
            infer_sb = i == last_i or i == 0
            if not infer_sb:
                ctxcg = min(int(csbf[ys, xs + 1]) + int(csbf[ys + 1, xs]), 1) + (2 if cidx else 0)
                c.encode(o["significant_coeff_group_flag"] + ctxcg, int(bool(nz)))
                csbf[ys, xs] = int(bool(nz))
            else:
                csbf[ys, xs] = 1
            if not csbf[ys, xs]:
                continue
            prev_sig = int(csbf[ys, xs + 1]) + 2 * int(csbf[ys + 1, xs])
            start = last_k - 1 if i == last_i else 15
            coded = [last_k] if i == last_i else []
            implicit = (not infer_sb)                                      # sub-block flag was coded as 1: last position may be inferred
            for k in range(start, -1, -1):
                xp, yp = pos_order[k]
                s = int(lev[(ys << 2) + yp, (xs << 2) + xp] != 0)
                if k == 0 and implicit and not coded:
                    assert s == 1
                    coded.append(0)
                    break
                # sigCtx (9.3.4.2.5)
                if log2 == 2:
                    sc = SIG_CTX_4x4[(yp << 2) + xp]
                elif xs == 0 and ys == 0 and k == 0 and (xp + yp) == 0:
                    sc = 0
                else:
                    if prev_sig == 0:
                        sc = 2 if xp + yp == 0 else (1 if xp + yp < 3 else 0)
                    elif prev_sig == 1:
                        sc = 2 if yp == 0 else (1 if yp == 1 else 0)
                    elif prev_sig == 2:
                        sc = 2 if xp == 0 else (1 if xp == 1 else 0)
                    else:
                        sc = 2
                    if cidx == 0:
                        if xs > 0 or ys > 0:
                            sc += 3
                        sc += (9 if scan_idx == 0 else 15) if log2 == 3 else 21
                    else:
                        sc += 9 if log2 == 3 else 12
                c.encode(o["significant_coeff_flag"] + sc + (27 if cidx else 0), s)
                if s:
                    coded.append(k)
            if not coded:
                continue
            # levels of this sub-block, in coding order (high scan position first)
            ctx_set = 2 if (i > 0 and cidx == 0) else 0
            if i != last_i and greater1_ctx == 0:
                ctx_set += 1
            greater1_ctx = 1
            vals = []
            for k in coded:
                xp, yp = pos_order[k]
                vals.append(int(lev[(ys << 2) + yp, (xs << 2) + xp]))
            g1, first_g1 = [], -1
            for m, v in enumerate(vals[:8]):
                f = int(abs(v) > 1)
                c.encode(o["coeff_abs_level_greater1_flag"] + (ctx_set << 2) + greater1_ctx + (16 if cidx else 0), f)
                g1.append(f)
                if f:
                    greater1_ctx = 0
                    if first_g1 < 0:
                        first_g1 = m
                elif 0 < greater1_ctx < 3:
                    greater1_ctx += 1
            g2 = 0
            if first_g1 >= 0:
                g2 = int(abs(vals[first_g1]) > 2)
                c.encode(o["coeff_abs_level_greater2_flag"] + ctx_set + (4 if cidx else 0), g2)
            for v in vals:
                c.bypass(int(v < 0))
            rice = 0
            for m, v in enumerate(vals):
                base = 1 + (g1[m] if m < 8 else 0) + (g2 if m == first_g1 else 0)
                thresh = (3 if m == first_g1 else 2) if m < 8 else 1
                if base == thresh:
                    rem = abs(v) - base
                    self.remaining(rem, rice)
                    if abs(v) > (3 << rice):
                        rice = min(rice + 1, 4)

    def remaining(self, v, rice):
        c = self.c
        if v < (3 << rice):
            p = v >> rice
            for _ in range(p):
                c.bypass(1)
            c.bypass(0)
            c.bypass_bits(rice, v & ((1 << rice) - 1))
        else:
            p = 0
            while (((1 << (p + 1)) + 2) << rice) <= v:
                p += 1
            for _ in range(p + 3):
                c.bypass(1)
            c.bypass(0)
            c.bypass_bits(p + rice, v - (((1 << p) + 2) << rice))

    def stream(self, frames, pattern="I"):
        """pattern: picture types in decode order after the leading IDR, cycled, e.g. "PB"; "I" = all IDR;
        "RA" = random access: hierarchical-B GOPs of 4 (decode order I0 P4 B2 B1 B3 P8 B6 B5 B7 ..., output in POC order);
        "RA8" = hierarchical-B GOPs of 8 with an I picture every 32 (BASELINE.json configs 2-4)"""
        if pattern in ("RA", "RA8"):
            self.plan = [dict(poc=0, type=2, neg=[], pos=[])]
            if pattern == "RA":
                self.reorder = 2
                a = 4
                while len(self.plan) < frames:
                    self.plan += [dict(poc=a, type=1, neg=[a - 4], pos=[]),
                                  dict(poc=a - 2, type=0, neg=[a - 4], pos=[a]),
                                  dict(poc=a - 3, type=0, neg=[a - 4], pos=[a - 2, a]),
                                  dict(poc=a - 1, type=0, neg=[a - 2], pos=[a])]
                    a += 4
            else:
                # BASELINE.json configs 2-4: hierarchical-B GOP 8 (decode order A8 B4 B2 B1 B3 B6 B5 B7), intra period 32 (the
                # anchor at POC % 32 == 0 is an I picture, open GOP: the B pictures in front of it still reference the previous
                # anchor).  Every picture's RPS lists what must stay in the DPB; its lists use the two nearest on either side.
                self.reorder = 3
                a = 8
                while len(self.plan) < frames:
                    self.plan += [dict(poc=a, type=2 if a % 32 == 0 else 1, neg=[a - 8], pos=[]),
                                  dict(poc=a - 4, type=0, neg=[a - 8], pos=[a]),
                                  dict(poc=a - 6, type=0, neg=[a - 8], pos=[a - 4, a]),
                                  dict(poc=a - 7, type=0, neg=[a - 8], pos=[a - 6, a - 4, a]),
                                  dict(poc=a - 5, type=0, neg=[a - 6], pos=[a - 4, a]),
                                  dict(poc=a - 2, type=0, neg=[a - 4], pos=[a]),
                                  dict(poc=a - 3, type=0, neg=[a - 4], pos=[a - 2, a]),
                                  dict(poc=a - 1, type=0, neg=[a - 2], pos=[a])]
                    a += 8
            self.plan = self.plan[:frames]
            out = self.vps() + self.sps() + self.pps()
            for k, pl in enumerate(self.plan):
                out += self.slice_nal(k, pl["type"])
            return out
        out = self.vps() + self.sps() + self.pps()
        for k in range(frames):
            if pattern == "I":
                out += self.slice_nal(0, 2)
            else:
                t = "I" if k == 0 else pattern[(k - 1) % len(pattern)]
                out += self.slice_nal(k, {"I": 2, "P": 1, "B": 0}[t])
        return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--width", type=int, default=832)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--bit-depth", type=int, default=8)
    ap.add_argument("--frames", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--qp", type=int, default=30)
    ap.add_argument("--no-sao", action="store_true")
    ap.add_argument("--pattern", default="I", help='"RA" = random access (hierarchical-B GOP 4), "RA8" = GOP 8 with intra period 32; else picture types after the IDR, e.g. "PB" (low-delay, 2 references)')
    ap.add_argument("--weighted", action="store_true")
    ap.add_argument("--cip", action="store_true", help="constrained_intra_pred_flag")
    ap.add_argument("--tqb", type=float, default=0.0, help="share of CUs coded with cu_transquant_bypass_flag")
    ap.add_argument("--pcm", type=float, default=0.0, help="share of 2Nx2N intra CUs coded as PCM")
    ap.add_argument("--pcm-lf-off", action="store_true", help="pcm_loop_filter_disabled_flag")
    ap.add_argument("--cfi", type=int, default=1, help="chroma_format_idc: 1 = 4:2:0, 2 = 4:2:2, 3 = 4:4:4")
    ap.add_argument("--slices", type=int, default=1, help="independent slices per picture (each starts a CTB row)")
    ap.add_argument("--no-lf-across-slices", action="store_true", help="slice_loop_filter_across_slices_enabled_flag = 0")
    ap.add_argument("--tskip", type=float, default=0.0, help="share of 4x4 TUs coded with transform_skip_flag")
    ap.add_argument("--tiles", default="", help="COLSxROWS uniformly spaced tiles, e.g. 3x2")
    ap.add_argument("--no-lf-across-tiles", action="store_true", help="loop_filter_across_tiles_enabled_flag = 0")
    ap.add_argument("--dbk-offsets", default="0,0", help="pps_beta_offset_div2,pps_tc_offset_div2")
    ap.add_argument("--chroma-qp-offsets", default="0,0", help="pps_cb_qp_offset,pps_cr_qp_offset")
    ap.add_argument("--sao-planes", default="both", choices=["both", "luma", "chroma"], help="which slice_sao_*_flag is set")
    ap.add_argument("--no-dbk", action="store_true", help="pps_deblocking_filter_disabled_flag")
    ap.add_argument("--tmvp", action="store_true", help="temporal motion vector prediction")
    ap.add_argument("--qpd", action="store_true", help="cu_qp_delta_enabled_flag: a QP delta per 32x32 quantisation group")
    ap.add_argument("--amp", action="store_true", help="amp_enabled_flag: asymmetric motion partitions")
    ap.add_argument("--ccp", action="store_true", help="cross_component_prediction_enabled_flag (needs --cfi 3)")
    ap.add_argument("--calm", type=float, default=0.0, help="0 = dense random content (default) .. 1 = lightly coded (more skip, larger CUs, sparse residuals)")
    ap.add_argument("--conf-win", default="", help="L,R,T,B: conformance window offsets in luma samples (multiples of the chroma subsampling)")
    ap.add_argument("--wpp", action="store_true", help="entropy_coding_sync_enabled_flag: one substream per CTB row + entry points")
    a = ap.parse_args()
    verify_tables_against_reference()
    g = StreamGen(a.width, a.height, a.bit_depth, a.seed, a.qp, sao=not a.no_sao, weighted=a.weighted, wpp=a.wpp, cip=a.cip, tqb=a.tqb, tskip=a.tskip, pcm=a.pcm, pcm_lf_off=a.pcm_lf_off, slices=a.slices, lf_across_slices=not a.no_lf_across_slices, cfi=a.cfi, calm=a.calm, ccp=a.ccp, amp=a.amp, qpd=a.qpd, tmvp=a.tmvp, no_dbk=a.no_dbk, sao_planes=a.sao_planes, dbk_offsets=tuple(int(v) for v in a.dbk_offsets.split(",")), chroma_qp_offsets=tuple(int(v) for v in a.chroma_qp_offsets.split(",")),
                  tiles=tuple(int(v) for v in a.tiles.split("x")) if a.tiles else None, lf_across_tiles=not a.no_lf_across_tiles)
    if a.conf_win:
        g.conf_win = tuple(int(v) for v in a.conf_win.split(","))
        sw, sh = (1 if a.cfi == 3 else 2), (2 if a.cfi == 1 else 1)
        assert len(g.conf_win) == 4 and all(v >= 0 for v in g.conf_win) and not (g.conf_win[0] | g.conf_win[1]) % sw and not (g.conf_win[2] | g.conf_win[3]) % sh
    data = g.stream(a.frames, a.pattern)
    open(a.out, "wb").write(data)
    print(f"wrote {a.out}: {len(data)} bytes, {a.frames} pictures {a.width}x{a.height} {a.bit_depth}-bit")
    for k, st in enumerate(g.stats):
        print(f"  picture {k}: intra_pred {st['intra_pred']} transform_add {st['transform_add']} prediction units {st['pu']}")


if __name__ == "__main__":
    main()
