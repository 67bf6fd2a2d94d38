/*
 * b200hevc.h — C ABI of libb200hevc.so, the H100 (sm_90a) back end for openHEVC's
 * per-CTU pixel-reconstruction path.
 *
 * Layering (see DESIGN.md):
 *   reference call sites (hevc.c / hevc_cabac.c / hevc_filter.c, unchanged)
 *     -> table slots installed by ff_hevcdsp_init_b200() & co. (include/b200hevc_tables.h; the
 *        same mechanism as ff_hevcdsp_init_x86, reference libavcodec/hevcdsp.c:1326-1327)
 *     -> recorder  b200_rec_*()        : appends one record per table call to the frame's blob
 *     -> engine    b200_frame_submit() : one pinned cudaMemcpyAsync + one kernel per stage
 *
 * Everything here is plain C: pointers, sizes, ints.  No CUDA / torch types.
 * All functions returning int return 0 on success or a negative B200_E* code; the text of the
 * last error of a context is available from b200_last_error().  Nothing here falls back to the
 * CPU: without a CUDA device b200_ctx_create() fails.
 */
#ifndef B200HEVC_H
#define B200HEVC_H

#include <stddef.h>
#include <stdint.h>
#include "b200hevc_worklist.h"

#ifdef __cplusplus
extern "C" {
#endif

#define B200_EINVAL   (-1)  /* bad argument / malformed blob        */
#define B200_ECUDA    (-2)  /* CUDA runtime error (latched)         */
#define B200_ENOMEM   (-3)
#define B200_ESTATE   (-4)  /* call sequence error                  */
#define B200_ENOTSUP  (-5)  /* feature outside the implemented path */

typedef struct B200Ctx B200Ctx;
typedef struct B200Rec B200Rec;

/* Threading contract.  A B200Ctx is driven by ONE submitting thread at a time: every call that takes a B200Ctx and is not
 * listed below mutates un-locked context state (slot hazards, arenas, lanes) and must come from that thread, pictures in
 * decode order (the table-level shim runs a dedicated submission thread for exactly this reason).  Callable from ANY
 * thread, concurrently with the submitting thread: b200_upload_wait, b200_readback_wait, b200_export_wait,
 * b200_export_event (they touch an immutable event handle only), b200_yuv_to_rgb (no context), b200_last_error, the b200_host_* functions and every b200_rec_* function (a B200Rec belongs to the thread
 * that records into it).  b200_ctx_create / b200_ctx_destroy are serialised internally. */

typedef struct B200Config {
    int32_t device;             /* CUDA device ordinal                                               */
    int32_t width, height;      /* luma samples: sps->width / sps->height (libavcodec/hevc.h)        */
    int32_t chroma_format_idc;  /* 1 = 4:2:0, 2 = 4:2:2, 3 = 4:4:4                                   */
    int32_t bit_depth;          /* 8..12 (luma == chroma, as the reference requires hevc_ps.c:1654)   */
    int32_t log2_ctb_size;      /* 4..6                                                              */
    int32_t n_slots;            /* device-resident DPB slots (reference: HEVCFrame DPB[32], hevc.h:1207) */
    int32_t n_arenas;           /* blobs in flight (upload of frame k+1 overlaps kernels of frame k)  */
    uint64_t max_blob_bytes;    /* capacity of one device arena; 0 = worst case for the geometry     */
    void    *ext_frame_mem;     /* optional caller-owned device memory for the DPB (e.g. a torch      */
    uint64_t ext_frame_bytes;   /*   tensor, so that torch.distributed can broadcast slots), else NULL/0 */
    int32_t n_lanes;            /* pictures executing concurrently (compute streams); 0 = default (8), max 16; env B200_LANES overrides */
    int32_t reserved0;
} B200Config;

/* ---- context --------------------------------------------------------------------------------- */
int         b200_ctx_create(const B200Config *cfg, B200Ctx **out);
void        b200_ctx_destroy(B200Ctx *ctx);
const char *b200_last_error(const B200Ctx *ctx);          /* ctx may be NULL: error of the failed create */
uint64_t    b200_dpb_bytes(const B200Config *cfg);         /* device bytes needed for cfg->n_slots slots   */
uint64_t    b200_slot_bytes(const B200Ctx *ctx);           /* bytes of one slot (3 planes, pitched)        */
void       *b200_slot_devptr(const B200Ctx *ctx, int slot, int plane, uint64_t *pitch_bytes);
void       *b200_stream(const B200Ctx *ctx);               /* cudaStream_t of compute lane 0 (slot uploads / fills run here)  */
int         b200_join(B200Ctx *ctx);                       /* b200_stream() waits for every picture submitted so far, on all
                                                              lanes: an event recorded on it afterwards covers them all      */
/* Caller-owned streams touching a DPB slot (NCCL broadcast of a reference picture, a display kernel ...): bracket the
 * work with begin/end.  begin makes `stream` wait for the slot's last writer (and, for write != 0, its pending
 * readers); end publishes the access so that later pictures / read-backs order themselves after it. */
int         b200_slot_begin_access(B200Ctx *ctx, int slot, void *stream, int write);
int         b200_slot_end_access(B200Ctx *ctx, int slot, void *stream, int write);

/* ---- pinned host memory for blobs / frames ---------------------------------------------------- */
void *b200_host_alloc(uint64_t bytes);
void  b200_host_free(void *p);
int   b200_host_register(void *p, uint64_t bytes);         /* page-lock memory the caller allocated (cudaHostRegister) */
int   b200_host_unregister(void *p);

/* ---- per-frame execution ---------------------------------------------------------------------- */
/* Upload `blob` (include/b200hevc_worklist.h) into arena `arena` on the copy stream (asynchronous when the blob
 * lives in b200_host_alloc memory).  Waits (stream-side) until the arena's previous frame has finished. */
int b200_frame_upload(B200Ctx *ctx, const void *blob, uint64_t nbytes, int arena);
/* Run K1..K5 for the blob resident in `arena`: reconstructs the picture into DPB slot hdr.cur_slot. */
int b200_frame_execute(B200Ctx *ctx, int arena);
/* Same, with the DPB placement overridden: cur_slot < 0 / ref_slots == NULL keep the header's values.  Lets a
 * resident work list be replayed against a rotating DPB (GOP-periodic streams, frame-parallel multi-GPU). */
int b200_frame_execute_ex(B200Ctx *ctx, int arena, int cur_slot, const uint8_t *ref_slots, int n_ref);
/* upload + execute, arenas used round-robin: the call the recorder's frame_end makes (hevc.c:3446). */
int b200_frame_submit(B200Ctx *ctx, const void *blob, uint64_t nbytes);
/* Same; *upload_token names the upload so that the owner of `blob` -- possibly another thread -- can wait until the blob
 * has left host memory (b200_upload_wait) before it writes the next picture into the same memory. */
int b200_frame_submit_ex(B200Ctx *ctx, const void *blob, uint64_t nbytes, uint32_t *upload_token);
int b200_upload_wait(B200Ctx *ctx, uint32_t upload_token);   /* any thread */

/* Planes are exchanged in the reference's AVFrame layout: planar, uint8 samples for 8-bit,
 * little-endian uint16 above; strides in bytes.  (libavcodec/hevc_ps.c:1666-1688) */
int b200_slot_upload(B200Ctx *ctx, int slot, const void *const planes[3], const int64_t strides[3]);
int b200_slot_readback(B200Ctx *ctx, int slot, void *const planes[3], const int64_t strides[3]); /* async after the slot's last writer */
/* read-back another thread will wait for (the decoder's output path, hevc_refs.c:182-307: a picture leaves the decoder long
 * after it was decoded): asynchronous like b200_slot_readback, *token names its completion for b200_readback_wait */
int b200_slot_readback_async(B200Ctx *ctx, int slot, void *const planes[3], const int64_t strides[3], uint32_t *token);
int b200_readback_wait(B200Ctx *ctx, uint32_t token);        /* any thread; host blocks until that read-back has landed */
/* ---- device-resident output ----------------------------------------------------------------------
 * b200_slot_export_async copies one DPB slot into caller-owned DEVICE memory, in the same AVFrame layout (uint8 samples at 8
 * bit, uint16 above), optionally cropped.  The copy is a reader of the slot like a read-back: it starts after the slot's last
 * writer, and a later picture that writes the slot waits for it.  *token names its completion: b200_export_wait blocks the
 * host, b200_export_event returns the cudaEvent_t (as void *) that a consumer's stream can wait on instead.  Tokens are
 * recycled after 64 further exports; both calls may come from any thread. */
typedef struct B200Export {
    void    *planes[3];         /* device destinations: Y, Cb, Cr                                                            */
    int64_t  pitches[3];        /* bytes per row                                                                            */
    int32_t  crop_x, crop_y;    /* crop window in luma samples; chroma offsets follow the chroma format, so x / width must   */
    int32_t  crop_w, crop_h;    /*   be even unless 4:4:4 and y / height even for 4:2:0.  crop_w == crop_h == 0: whole picture */
    void    *after_event;       /* optional cudaEvent_t: the copy starts after it (e.g. the destination's previous consumer)  */
} B200Export;
int   b200_slot_export_async(B200Ctx *ctx, int slot, const B200Export *e, uint32_t *token);
int   b200_export_wait(B200Ctx *ctx, uint32_t token);         /* any thread; host blocks until that export has landed */
void *b200_export_event(B200Ctx *ctx, uint32_t token);        /* any thread; cudaEvent_t of that export, NULL for a bad token */

/* YUV (AVFrame layout, device memory: a DPB slot, an export target, ...) -> planar RGB (CHW, contiguous) in caller device
 * memory, as uint8 or as float32 in [0, 1], on `stream` (a cudaStream_t; NULL = the legacy default stream).  The matrix and
 * the range are the caller's: the decoder does not read the VUI colour description.  Chroma is upsampled by nearest sample.
 * The fixed-point definition of the arithmetic is in openhevc_b200/csrc/k_yuv_rgb.cuh.  B200_ENOTSUP for a matrix, chroma
 * format or bit depth outside the list below. */
typedef struct B200RgbArgs {
    const void *planes[3];      /* device Y, Cb, Cr                                                                          */
    int64_t     pitches[3];     /* bytes per row                                                                             */
    int32_t     width, height;  /* luma samples of the planes                                                                */
    int32_t     chroma_format_idc;  /* 1 = 4:2:0, 2 = 4:2:2, 3 = 4:4:4                                                       */
    int32_t     bit_depth;      /* 8..12                                                                                     */
    int32_t     crop_x, crop_y, crop_w, crop_h;   /* luma samples, any offsets and sizes; crop_w == crop_h == 0: whole picture  */
    int32_t     matrix;         /* matrix_coefficients: 1 = BT.709, 5 or 6 = BT.601, 9 = BT.2020 non-constant luminance       */
    int32_t     full_range;     /* 0 = limited (video) range, 1 = full range                                                 */
    int32_t     out_float;      /* 0 = uint8, 1 = float32                                                                    */
    int32_t     reserved0;
    void       *out;            /* 3 x crop_h x crop_w samples: R, G, B planes                                               */
} B200RgbArgs;
int b200_yuv_to_rgb(const B200RgbArgs *a, void *stream);

int b200_poll_errors(B200Ctx *ctx);                          /* device-side error latches (rejected work list, intra dependency time-out)
                                                                WITHOUT synchronising: 0 or the error b200_sync would report */
int b200_slot_wait_readback(B200Ctx *ctx, int slot);         /* host blocks until the slot's last read-back has landed (not for the whole queue) */
int b200_slot_fill(B200Ctx *ctx, int slot, int value);    /* generate_missing_ref, hevc_refs.c:538-606 */
int b200_wait_uploads(B200Ctx *ctx);                       /* wait until submitted blobs have left host memory (not for the kernels) */
int b200_sync(B200Ctx *ctx);                               /* wait for everything, surface latched errors */

/* ---- measurement ------------------------------------------------------------------------------ */
enum { B200_ST_MC = 0, B200_ST_RESIDUAL, B200_ST_INTRA, B200_ST_DEBLOCK, B200_ST_SAO, B200_ST_TOTAL, B200_ST_COUNT };
int      b200_set_profiling(B200Ctx *ctx, int on);         /* CUDA events around every stage            */
int      b200_get_stage_ms(B200Ctx *ctx, float ms[B200_ST_COUNT]); /* of the last executed frame (syncs) */
uint64_t b200_launch_count(const B200Ctx *ctx);            /* kernels launched by this context so far   */

/* ---- recorder: host side, builds one blob per picture ------------------------------------------
 * One B200Rec per decoding thread context and picture in flight.  b200_rec_* mirror the table
 * slots one to one; coordinates are in samples of `plane`. */
int  b200_rec_create(const B200Config *cfg, B200Rec **out);
void b200_rec_destroy(B200Rec *r);
int  b200_rec_begin(B200Rec *r, int cur_slot, int poc);                   /* hevc_frame_start, hevc.c:3197 */
/* the picture's reference table: DPB slot of every frame the RefPicLists can address (hevc_refs.c ff_hevc_slice_rpl);
 * B200McRec.ref0/ref1 passed to b200_rec_mc() index it */
int  b200_rec_set_refs(B200Rec *r, const uint8_t *slots, int n);
/* transform_add[log2-2](dst, coeffs, stride) preceded by kind/flags recorded from idct*/
int  b200_rec_tu(B200Rec *r, int plane, int x, int y, int log2, int kind, int flags, int col_limit,
                 const int16_t *coeffs, int intra_linked);
int  b200_rec_pcm(B200Rec *r, int plane, int x, int y, int log2, const int16_t *samples);
int  b200_rec_intra(B200Rec *r, int plane, int x, int y, int log2, int mode, int flags,
                    int top_right_size, int bottom_left_size);
/* one put_hevc_{q,e}pel_{uni,uni_w} call, or a put_hevc_*pel + put_hevc_*pel_bi[_w] pair (split into tiles here) */
int  b200_rec_mc(B200Rec *r, const B200McRec *whole_block /* w,h up to 64 */);
int  b200_rec_deblock(B200Rec *r, int plane, int vertical, int x, int y, int beta, const int tc[2],
                      const uint8_t no_p[2], const uint8_t no_q[2]);
int  b200_rec_sao(B200Rec *r, int plane, int x, int y, const B200SaoRec *params);
/* pps->constrained_intra_pred_flag pictures: which min-PUs are intra coded (one byte per PU, row-major, non-zero = intra:
 * MvField.pred_flag == PF_INTRA of s->ref->tab_mvf, hevc.h:1032-1041), once all CTBs are parsed.  B200IntraRec.flags of
 * such a picture are the availability BEFORE the constrained-intra rule (hevcpred_template.c:116-163) */
int  b200_rec_set_cip(B200Rec *r, int log2_min_pu_size, int min_pu_width, int min_pu_height, const uint8_t *is_intra);
/* streams with transquant_bypass_enable_flag / pcm_loop_filter_disabled AND SAO: s->is_pcm[] (one byte per min-PU, non-zero
 * = PCM-without-loop-filter or transquant-bypass PU), once all CTBs are parsed; the device gives those PUs their deblocked
 * samples back after SAO, exactly as restore_tqb_pixels does (hevc_filter.c:163-193) */
int  b200_rec_set_tqb(B200Rec *r, int log2_min_pu_size, int min_pu_width, int min_pu_height, const uint8_t *is_pcm);
/* cross-component prediction (4:4:4, hevc.c:1295-1360): b200_rec_tu_parked records a transform block whose residual is only
 * PARKED (not added to the picture, not linked to an intra record) and returns where; b200_rec_ccp records
 * "block of `plane` += (scale * parked luma residual) >> 3 [+ its own parked residual]" -- added to the picture after the
 * residual stage, or handed to the intra stage when the block is intra predicted (decided like b200_rec_tu does). */
int  b200_rec_tu_parked(B200Rec *r, int plane, int x, int y, int log2, int kind, int flags, int col_limit, const int16_t *coeffs,
                        uint32_t *park_off);
int  b200_rec_ccp(B200Rec *r, int plane, int x, int y, int log2, int scale, uint32_t off_y, int has_c, uint32_t off_c);
/* Deblocking parameters derived on the device (SURVEY.md 8f N2; B200DbdHeader in b200hevc_worklist.h): instead of the
 * reference's per-edge filter calls (b200_rec_deblock) the picture carries their inputs.  b200_rec_bs_leaf = one call of
 * ff_hevc_deblocking_boundary_strengths() (hevc_filter.c:805; top / left: that edge of the block takes part, :832-839 /
 * :870-877 evaluated by the caller); b200_rec_set_dbd, once all CTBs are parsed, hands over s->qp_y_tab, s->deblock[] and
 * -- for streams with PCM-loop-filter-off / transquant-bypass blocks -- s->is_pcm (else NULL). */
typedef struct B200DbdInput {
    int32_t log2_min_cb_size, min_cb_width, min_cb_height; const int8_t *qp_y;       /* s->qp_y_tab */
    int32_t log2_min_pu_size, min_pu_width, min_pu_height; const uint8_t *is_pcm;    /* s->is_pcm or NULL */
    const int8_t *ctb_offsets;                                                       /* s->deblock[]: beta_offset, tc_offset per CTB */
    int32_t cb_qp_offset, cr_qp_offset;                                              /* pps */
} B200DbdInput;
int  b200_rec_bs_leaf(B200Rec *r, int x0, int y0, int log2_size, int top, int left);
int  b200_rec_set_dbd(B200Rec *r, const B200DbdInput *in);
/* host helper shared by the recorder and by external blob builders: permutation (perm[new] = old) that sorts decode-order
 * intra records by dependency level (stable); returns the number of levels (>= 0) or a negative error */
int  b200_intra_level_order(const B200IntraRec *recs, uint32_t n, int width, int height, int chroma_format_idc, uint32_t *perm);
/* finish: returns the blob (pinned memory owned by the recorder, valid until the next begin) */
int b200_rec_merge(B200Rec *dst, B200Rec *src);           /* fold the lists of a worker thread of the SAME picture into dst (WPP / tiles / slices) */
int  b200_rec_finish(B200Rec *r, const void **blob, uint64_t *nbytes);

#ifdef __cplusplus
}
#endif
#endif /* B200HEVC_H */
