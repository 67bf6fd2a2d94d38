/*
 * b200hevc_worklist.h — wire format of the per-frame packed work list ("blob v1").
 *
 * The host side of the decoder (openHEVC's CABAC parse / MV / BS derivation, which
 * stays on the CPU) does not execute pixel kernels any more: every call it makes
 * through the HEVCDSPContext / HEVCPredContext function tables
 * (reference: libavcodec/hevcdsp.h:44-124, libavcodec/hevcpred.h:31-41) is
 * *recorded* as one fixed-size record below.  One blob describes one picture and
 * is uploaded with a single cudaMemcpyAsync; one kernel per stage consumes it.
 *
 * Plain C, no CUDA / torch types: shared by the CUDA engine, the recorder,
 * the CPU oracle (oracle/hevc_oracle.c) and mirrored by numpy dtypes in
 * openhevc_b200/worklist.py.
 */
#ifndef B200HEVC_WORKLIST_H
#define B200HEVC_WORKLIST_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_BLOB_MAGIC   0x4C573242u /* "B2WL" */
#define B200_BLOB_VERSION 3u

/* blob sections; every section start is 256-byte aligned inside the blob */
enum {
    B200_SEC_COEFF = 0,   /* int16 pool: dequantised coefficients (sparse pairs or dense blocks) / PCM samples; count = #int16 */
    B200_SEC_TU4,         /* B200TuRec, 4x4 blocks   (transform_add[0] call sites)                  */
    B200_SEC_TU8,         /* B200TuRec, 8x8                                                        */
    B200_SEC_TU16,        /* B200TuRec, 16x16                                                      */
    B200_SEC_TU32,        /* B200TuRec, 32x32                                                      */
    B200_SEC_INTRA,       /* B200IntraRec in decode order (intra_pred[] call sites)                */
    B200_SEC_MC,          /* B200McRec, one per <=256-sample tile of a put_hevc_{q,e}pel* call     */
    B200_SEC_DBK,         /* uint16 edge-parameter grids, layout B200DbkLayout (count = #uint16)   */
    B200_SEC_SAO,         /* B200SaoRec grid [3][ctb_count] (count = 3*ctb_count) or 0 = no SAO    */
    B200_SEC_COUNT
};

typedef struct B200Section {
    uint32_t off;    /* byte offset from blob start */
    uint32_t count;  /* number of elements          */
} B200Section;

typedef struct B200BlobHeader {
    uint32_t magic;
    uint32_t version;
    uint32_t total_bytes;
    int32_t  poc;
    uint16_t width, height;      /* luma samples (sps->width / sps->height)                    */
    uint8_t  chroma_format_idc;  /* 1 = 4:2:0, 2 = 4:2:2, 3 = 4:4:4                            */
    uint8_t  bit_depth;          /* 8..12                                                      */
    uint8_t  log2_ctb_size;      /* 4..6                                                       */
    uint8_t  cur_slot;           /* DPB slot that receives this picture                        */
    uint32_t flags;              /* B200_FRAME_*                                               */
    B200Section sec[B200_SEC_COUNT];
    uint8_t  ref_slot[16];       /* DPB slot of each entry of the picture's reference table (from the RPS /
                                    RefPicList, hevc_refs.c); B200McRec.ref0/ref1 index this table            */
    uint8_t  n_ref;
    uint8_t  pad[3];
    uint32_t mc_big_count;       /* B200_SEC_MC is ordered: records [0, mc_big_count) are tiles of any legal shape (one warp
                                    each), the rest are tiles of <= 8x8 samples (four per warp), grouped by
                                    B200_MC_SMALL_KEY so that the tiles sharing a warp take the same branches            */
    B200Section cip;             /* constrained_intra_pred pictures only (else count = 0): uint32 words, B200CipHeader followed by
                                    one bit per min-PU, row-major, bit set = the PU is intra coded (MvField.pred_flag == PF_INTRA,
                                    hevc.h:1032-1041, read by hevcpred_template.c:39-40).  Carved out of the reserved words of blob v3:
                                    older blobs read as "no CIP"                                                                      */
    B200Section tqb;             /* pictures of streams with transquant_bypass / pcm_loop_filter_disabled AND SAO (else count = 0): uint32
                                    words, B200CipHeader followed by one bit per min-PU, bit set = s->is_pcm[] != 0 (PCM with the loop filter
                                    off, or cu_transquant_bypass).  After SAO those PUs get their deblocked samples back
                                    (restore_tqb_pixels, hevc_filter.c:163-193 -- with its two quirks, see k_sao.cuh)                        */
    B200Section ccp;             /* 4:4:4 pictures of streams with cross_component_prediction_enabled_flag (else count = 0): B200CcpRec[count],
                                    executed between the residual stage and the intra stage                                            */
    B200Section dbd;             /* deblocking parameters derived ON THE DEVICE (SURVEY.md 8f N2; else count = 0): uint32 words, a
                                    B200DbdHeader followed by the arrays it names.  A picture carries either the DBK grids (the
                                    reference's own per-edge calls, recorded) or this section (its inputs: transform-tree leaves,
                                    QP map, per-CTB offsets; motion and cbf come from the MC / TU records), never both -- except in
                                    check mode (B200_DBD_CHECK), where the device compares what it derived with the recorded grids */
    B200Section reserved_section; /* off and count must both be zero (b200_frame_upload rejects the blob otherwise); holds the place of
                                    the fields behind it */
    uint32_t mc_tile_count[5];   /* all zero: the records of B200_SEC_MC are TILES (<= 256 samples, ordered as mc_big_count says).  Else they are
                                    whole PREDICTION BLOCKS (w, h <= 64) in decode order and the DEVICE splits them (k_mc_expand): [0] tiles of
                                    any shape, [1 + B200_MC_SMALL_KEY] tiles of <= 8x8 samples; B200McRec.pad = index of the block's first
                                    tile inside its bucket (24 bits, little endian); all tiles of one record fall into one bucket */
    uint32_t reserved[64 - 28 - 2 * B200_SEC_COUNT];
} B200BlobHeader;               /* 256 bytes */

/* ---- on-device derivation of the deblocking parameters (hevc_filter.c:345-581 control half, :584-941) --------------------
 * What the reference computes on the host between the parse and the filter calls -- boundary strengths from the motion field
 * and the coded-block flags (ff_hevc_deblocking_boundary_strengths), then tc / beta per edge from the QP map and the slice
 * offsets (deblocking_filter_CTB) -- from inputs that are already in the blob (MC records: motion; luma TU records: cbf) plus:
 *   leaves   one uint32 per ff_hevc_deblocking_boundary_strengths() call (hevc.c:1578, 1607, 2400, 2484):
 *            bits 0..11 x0 >> 2, 12..23 y0 >> 2, 24..26 log2_size - 2 (transform blocks 4x4 .. coding blocks 64x64), bit 28 the top edge
 *            takes part (hevc_filter.c:832-839 evaluated on the host: slice / tile boundary rules), bit 29 the left edge (:870-877)
 *   qp       int8 per min coding block (s->qp_y_tab), row-major
 *   ctb      2 x int8 per CTB: beta_offset, tc_offset (s->deblock[], hevc.c:2677-2678)
 *   pcm      uint8 per min PU (s->is_pcm), only when flags & B200_DBDF_PCM (pcm loop filter off / transquant bypass: no_p / no_q) */
#define B200_DBD_LEAF(x0, y0, log2, top, left) \
    ((uint32_t)((x0) >> 2) | ((uint32_t)((y0) >> 2) << 12) | ((uint32_t)((log2) - 2) << 24) | ((uint32_t)((top) != 0) << 28) | ((uint32_t)((left) != 0) << 29))
#define B200_DBDF_PCM 1u
typedef struct B200DbdHeader {   /* 16 words */
    uint32_t flags;              /* B200_DBDF_* */
    uint32_t log2_min_cb_size, min_cb_width, min_cb_height;     /* geometry of qp[] */
    uint32_t log2_min_pu_size, min_pu_width, min_pu_height;     /* geometry of pcm[] */
    int32_t  cb_qp_offset, cr_qp_offset;                        /* pps, chroma_tc() hevc_filter.c:62-88 */
    uint32_t n_leaf;
    uint32_t off_leaf, off_qp, off_ctb, off_pcm;                /* byte offsets from the start of the section, 16-byte aligned */
    uint32_t reserved[2];
} B200DbdHeader;

typedef struct B200CipHeader {   /* first 4 words of the CIP section */
    uint32_t log2_min_pu_size;   /* sps->log2_min_pu_size */
    uint32_t min_pu_width;       /* sps->min_pu_width  (bitmap row length in bits) */
    uint32_t min_pu_height;
    uint32_t reserved;
} B200CipHeader;
#define B200_CIP_WORDS(pw, ph) (4u + (((uint32_t)(pw) * (uint32_t)(ph) + 31u) >> 5))

#define B200_MC_IS_SMALL(w, h) ((w) <= 8 && (h) <= 8)
/* How a prediction block of w x h samples is cut into tiles (recorder.cpp b200_rec_mc on the host, k_mc_expand on the device -- the
 * one definition): columns of <= 16 samples when the block is taller than 8 rows (the squarer tile has the smaller filter halo),
 * else <= 32; rows of <= 16 (tile width <= 16) or <= 8. */
#define B200_MC_TILE_WMAX(h) ((h) > 8 ? 16 : 32)
#define B200_MC_TILE_HMAX(tw) ((tw) > 16 ? 8 : 16)
#define B200_MC_SMALL_KEY(flags) ((((flags) & B200_MCF_CHROMA) ? 2 : 0) | (((flags) & B200_MCF_BI) ? 1 : 0))   /* 0..3 */

#define B200_FRAME_HAS_DEBLOCK 1u
#define B200_FRAME_HAS_SAO     2u
#define B200_FRAME_TQB         8u   /* B200BlobHeader.tqb is present; B200SaoRec.tqb marks the CTBs that contain such PUs */
#define B200_FRAME_CCP         16u  /* B200BlobHeader.ccp is present */
#define B200_FRAME_CIP         4u   /* pps->constrained_intra_pred_flag: B200IntraRec.flags hold the availability BEFORE the
                                       CIP rules; the device applies hevcpred_template.c:116-163 and :185-249 with the bitmap */

/* ---- residual stage (K2) ------------------------------------------------------------- */
enum {
    B200_TU_IDCT   = 0, /* hevcdsp.idct[log2-2](coeffs, col_limit)   hevc_cabac.c:1934 */
    B200_TU_DC     = 1, /* hevcdsp.idct_dc[log2-2](coeffs)           hevc_cabac.c:1925 */
    B200_TU_DST    = 2, /* hevcdsp.idct_4x4_luma(coeffs)             hevc_cabac.c:1921 */
    B200_TU_SKIP   = 3, /* hevcdsp.transform_skip(coeffs, log2)      hevc_cabac.c:1885 */
    B200_TU_BYPASS = 4, /* cu_transquant_bypass: coeffs are the residual  hevc_cabac.c:1868 */
    B200_TU_PCM    = 5  /* hevcdsp.put_pcm: pool holds final samples (already << (BD-pcm_bd)), stored not added */
};
#define B200_TUF_RDPCM      1u /* followed by hevcdsp.transform_rdpcm()      hevc_cabac.c:1873,1892 */
#define B200_TUF_RDPCM_VERT 2u /* rdpcm mode 1 (running sum down the columns)                      */
/* Either rdpcm flag is legal on B200_TU_SKIP and B200_TU_BYPASS only, as in the reference.  The device applies the vertical
   running sum between its two transform stages and would apply it to PCM samples, so any other kind with an rdpcm flag is
   rejected (k_validate; b200_rec_tu returns B200_EINVAL). */
#define B200_TUF_PARK       4u /* intra TU: leave the residual in the pool (K3 adds it after prediction) */

typedef struct B200TuRec {       /* 16 bytes */
    uint16_t x, y;               /* top-left sample in its plane                                  */
    uint8_t  plane;              /* 0 Y, 1 Cb, 2 Cr                                               */
    uint8_t  log2;               /* 2..5; PCM: log2 of the (square) block in this plane, 1..6 lives in the TU4 list with w/h in col_limit */
    uint8_t  kind;               /* B200_TU_*                                                     */
    uint8_t  flags;              /* B200_TUF_*                                                    */
    uint8_t  col_limit;          /* IDCT only (hevc_cabac.c:1927-1933)                            */
    uint8_t  pad;
    uint16_t nnz;                /* sparse transport: number of (position, value) int16 pairs; B200_TU_DENSE = dense NxN block */
    uint32_t coeff_off;          /* int16 index of this TU's data in the COEFF pool.  PARK TUs: the first two int16 are
                                    the (lo, hi) halves of the TU's index in the parked-residual pool, data follows  */
} B200TuRec;
#define B200_TU_DENSE 0xFFFFu

/* ---- intra stage (K3) ------------------------------------------------------------------ */
#define B200_INF_UP_LEFT     1u  /* cand_up_left      (after z-scan / CIP checks, hevcpred_template.c:100-104) */
#define B200_INF_UP          2u
#define B200_INF_UP_RIGHT    4u
#define B200_INF_LEFT        8u
#define B200_INF_BOTTOM_LEFT 16u
#define B200_INF_FILTER      32u /* !intra_smoothing_disabled && (c_idx==0 || chroma_array_type==3)  :288 */
#define B200_INF_STRONG      64u /* sps_strong_intra_smoothing_enable_flag                           :296 */

/* ---- cross-component prediction (range extensions, 4:4:4; hevc.c:1186-1197, 1295-1360, hevc_cabac.c:1942-1948) ----------
 * chroma residual += (res_scale_val * luma residual) >> 3, in int16 like the reference's coefficient arrays.  The reference
 * computes it on the host from the luma block it has just transformed in place; with the transforms on the device the
 * luma residual only exists there, so the recorder has the residual stage PARK it (a second, unlinked record of the luma TU)
 * next to the chroma block's own residual (when it has coefficients), and this record combines them.                      */
#define B200_CCPF_HAS_C   1u /* the chroma block has its own residual, parked at off_c                                 */
#define B200_CCPF_TO_PARK 2u /* intra TU: the result goes to parked[off_out] (B200IntraRec.resid_off), else it is added to the picture */
typedef struct B200CcpRec {      /* 32 bytes */
    uint16_t x, y;               /* block origin in its plane                                     */
    uint8_t  plane;              /* 1 = Cb, 2 = Cr                                                */
    uint8_t  log2;               /* 2..5                                                          */
    int8_t   scale;              /* lc->tu.res_scale_val: +-1, +-2, +-4, +-8                      */
    uint8_t  flags;              /* B200_CCPF_*                                                   */
    uint32_t off_y;              /* parked luma residual, int16 units                             */
    uint32_t off_c;              /* parked chroma residual (B200_CCPF_HAS_C)                      */
    uint32_t off_out;            /* destination in the parked pool (B200_CCPF_TO_PARK)            */
    uint32_t pad[3];
} B200CcpRec;

typedef struct B200IntraRec {    /* 16 bytes */
    uint16_t x, y;               /* top-left sample in its plane */
    uint8_t  plane;              /* c_idx */
    uint8_t  log2;               /* 2..5 */
    uint8_t  mode;               /* 0 planar, 1 DC, 2..34 angular */
    uint8_t  flags;              /* B200_INF_* */
    uint8_t  top_right_size;     /* samples really inside the picture, hevcpred_template.c:108-109 */
    uint8_t  bottom_left_size;   /* hevcpred_template.c:106-107 */
    uint8_t  pad[2];
    uint32_t resid_off;          /* int16 index of the parked residual in COEFF, 0xFFFFFFFF = cbf 0 */
} B200IntraRec;
#define B200_NO_RESID 0xFFFFFFFFu

/* ---- inter stage (K1) -------------------------------------------------------------------- */
#define B200_MCF_BI       1u
#define B200_MCF_WEIGHTED 2u
#define B200_MCF_CHROMA   4u     /* 4-tap epel filters, fractions in 1/8 units */

typedef struct B200McRec {       /* 32 bytes */
    uint16_t x, y;               /* destination top-left sample in its plane */
    uint8_t  w, h;               /* tile size, w*h <= 256 after recorder splitting, w<=32 */
    uint8_t  plane;
    uint8_t  flags;              /* B200_MCF_* */
    int16_t  sx0, sy0;           /* integer source position in ref0's plane (may lie outside: samples clamp, videodsp_template.c:26-100) */
    int16_t  sx1, sy1;
    uint8_t  ref0, ref1;         /* indices into B200BlobHeader.ref_slot[] */
    uint8_t  frac0, frac1;       /* mx | my << 4 */
    int16_t  w0, w1;             /* weights  (hevc.c:1677-1683, 1763-1773) */
    int16_t  o0, o1;             /* offsets, un-scaled as passed to the *_w table functions */
    uint8_t  denom;
    uint8_t  pad[3];
} B200McRec;

/* ---- deblocking (K4) ----------------------------------------------------------------------
 * One uint16 per 4-sample edge segment, dense grids (0 = edge not filtered):
 *   bits 0..5  tc   (8-bit scale, as in the tc[] argument)      bits 6..12 beta (8-bit scale)
 *   bit 13 no_p   bit 14 no_q   bit 15 present
 * Vertical-edge grid of a plane  : index (y>>2) * ew + (x>>3),   ew = (pw+7)>>3, rows (ph+3)>>2
 * Horizontal-edge grid of a plane: index (y>>3) * sw + (x>>2),   sw = (pw+3)>>2, rows (ph+7)>>3
 * x,y,pw,ph are in samples of that plane.  Section order: Y-vert, Y-horz, Cb-vert, Cb-horz, Cr-vert, Cr-horz,
 * each grid start rounded up to 64 uint16.  (hevc_filter.c:345-581 call sites.) */
#define B200_DBK_TC(e)    ((e) & 63)
#define B200_DBK_BETA(e)  (((e) >> 6) & 127)
#define B200_DBK_NOP(e)   (((e) >> 13) & 1)
#define B200_DBK_NOQ(e)   (((e) >> 14) & 1)
#define B200_DBK_PRESENT  0x8000u
#define B200_DBK_PACK(tc, beta, nop, noq) \
    ((uint16_t)(B200_DBK_PRESENT | ((tc) & 63) | (((beta) & 127) << 6) | (((nop) & 1) << 13) | (((noq) & 1) << 14)))

typedef struct B200DbkLayout {   /* derived from the picture geometry, never stored */
    uint32_t off[3][2];          /* [plane][0 vert,1 horz] start index in uint16 units */
    uint32_t stride[3][2];       /* grid row stride */
    uint32_t rows[3][2];
    uint32_t total;              /* total uint16 count */
} B200DbkLayout;

/* ---- SAO (K5) ---------------------------------------------------------------------------- */
enum { B200_SAO_NONE = 0, B200_SAO_BAND = 1, B200_SAO_EDGE = 2 };

typedef struct B200SaoRec {      /* 16 bytes; grid index = plane * ctb_count + ctb_addr_rs */
    uint8_t  type;               /* B200_SAO_* (sao->type_idx at call time)                          */
    uint8_t  param;              /* band_position (band) or eo_class (edge)                           */
    uint8_t  borders;            /* bit0 left, bit1 top, bit2 right, bit3 bottom picture border      */
    uint8_t  edges;              /* bit0-1 vert_edge[2], bit2-3 horiz_edge[2], bit4-7 diag_edge[4]; only variant 1 */
    uint8_t  variant;            /* 0 = sao_edge_filter[0], 1 = sao_edge_filter[1] (restore)          */
    uint8_t  tqb;                /* 1 = the CTB contains PUs of B200BlobHeader.tqb (set by the recorder)  */
    int16_t  offset_val[5];      /* sao->offset_val[c_idx][0..4]                                      */
} B200SaoRec;

#ifdef __cplusplus
static_assert(sizeof(B200BlobHeader) == 256 && sizeof(B200TuRec) == 16 && sizeof(B200IntraRec) == 16 &&
              sizeof(B200McRec) == 32 && sizeof(B200SaoRec) == 16, "blob v1 layout");
#else
_Static_assert(sizeof(B200BlobHeader) == 256 && sizeof(B200TuRec) == 16 && sizeof(B200IntraRec) == 16 &&
               sizeof(B200McRec) == 32 && sizeof(B200SaoRec) == 16, "blob v1 layout");
#endif

/* data of a TU inside the pool; *park_off receives the parked-pool index of PARK TUs */
static inline const int16_t *b200_tu_data(const B200TuRec *t, const int16_t *pool, uint32_t *park_off)
{
    const int16_t *p = pool + t->coeff_off;
    if (t->flags & B200_TUF_PARK) { *park_off = (uint32_t)(uint16_t)p[0] | ((uint32_t)(uint16_t)p[1] << 16); p += 2; }
    return p;
}
/* dense NxN coefficients of a TU (what lc->tu.coeffs held at transform_add time) */
static inline void b200_tu_expand(const B200TuRec *t, const int16_t *data, int16_t *dense)
{
    const int n2 = 1 << (2 * t->log2);
    if (t->nnz == B200_TU_DENSE) { for (int i = 0; i < n2; i++) dense[i] = data[i]; return; }
    for (int i = 0; i < n2; i++) dense[i] = 0;
    for (int e = 0; e < t->nnz; e++) dense[(uint16_t)data[2 * e] & (n2 - 1)] = data[2 * e + 1];
}

static inline uint32_t b200_align_u32(uint32_t v, uint32_t a) { return (v + a - 1) / a * a; }

static inline void b200_plane_dims(int width, int height, int chroma_format_idc, int plane, int *pw, int *ph)
{
    int hs = plane && chroma_format_idc != 3, vs = plane && chroma_format_idc == 1;
    *pw = width >> hs;
    *ph = height >> vs;
}

static inline void b200_dbk_layout(int width, int height, int chroma_format_idc, B200DbkLayout *L)
{
    uint32_t o = 0;
    for (int p = 0; p < 3; p++) {
        int pw, ph;
        b200_plane_dims(width, height, chroma_format_idc, p, &pw, &ph);
        L->stride[p][0] = (uint32_t)(pw + 7) >> 3; L->rows[p][0] = (uint32_t)(ph + 3) >> 2;
        L->stride[p][1] = (uint32_t)(pw + 3) >> 2; L->rows[p][1] = (uint32_t)(ph + 7) >> 3;
        for (int d = 0; d < 2; d++) {
            L->off[p][d] = o;
            o = b200_align_u32(o + L->stride[p][d] * L->rows[p][d], 64);
        }
    }
    L->total = o;
}

#ifdef __cplusplus
}
#endif
#endif /* B200HEVC_WORKLIST_H */
