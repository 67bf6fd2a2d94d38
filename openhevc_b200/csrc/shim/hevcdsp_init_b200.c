/*
 * hevcdsp_init_b200.c — the drop-in boundary: re-populates openHEVC's own function tables with
 * recorders that feed libb200hevc.so.  The B200 analogue of libavcodec/x86/hevcdsp_init.c:
 *
 *   ff_hevcdsp_init_b200(HEVCDSPContext *, bit_depth)   <- hook after hevcdsp.c:1326-1327
 *   ff_hevcpred_init_b200(HEVCPredContext *, bit_depth) <- hook after hevcpred.c:84
 *   ff_videodsp_init_b200(VideoDSPContext *, bpc)       <- hook after videodsp.c:51-58
 *   b200_frame_begin / b200_frame_end / b200_frame_readback <- hevc.c:3245 / 3446 / 4145 (INTEGRATION.md)
 *
 * Every installed function has exactly the signature of the slot it replaces (hevcdsp.h:45-105,
 * hevcpred.h:32-40, videodsp.h:66-70) and never touches pixels: it maps the pointers it is given
 * back to (DPB slot, plane, x, y) through the planes registered at frame begin and appends one record.
 * Compiled against the reference's headers where they lie (-I/root/reference); it contains no
 * reference code.  Threading (SURVEY.md §8b): recorder state is thread-local.  Frame threads (-f 1): every thread owns
 * the picture it decodes, pictures are submitted to the GPU in decode order through a ticket.  Slice / WPP / tile worker
 * threads of ONE picture (-f 2, execute2 jobs, hevc.c:3082): a worker attaches itself to the picture in progress on its
 * first table call, records into its own B200Rec, and b200_frame_end folds the workers into the owner's recorder
 * (b200_rec_merge).  Frame and slice threads combined (-f 4): several pictures are in progress and a table call carries no
 * context, so the execute2 jobs say which picture they belong to (b200_worker_begin).  One decoder instance per process.
 *
 * Pictures reach the device through ONE submission thread (the engine's threading contract, include/b200hevc.h): a decoding
 * thread that has parsed its picture hands the finished work list over (a queue ordered by the ticket taken at
 * b200_frame_begin, i.e. decode order) and goes on with its next packet at once; the submission thread uploads, launches and
 * issues the read-back of the picture into its (pinned, b200_frame_buffer_alloc) host frame.  Nobody waits for the device
 * until the picture LEAVES the decoder: b200_output_wait, hooked where hevc_decode_frame hands a frame to its caller.
 */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "libavcodec/hevc.h"
#include "libavcodec/hevcdsp.h"
#include "libavcodec/hevcpred.h"
#include "libavcodec/videodsp.h"
#include "libavcodec/get_bits.h"
#include "b200hevc.h"
#include "b200hevc_tables.h"
#include <dlfcn.h>
#include <time.h>
static inline uint64_t now_ns(void) { struct timespec t; clock_gettime(CLOCK_MONOTONIC, &t); return (uint64_t)t.tv_sec * 1000000000ull + (uint64_t)t.tv_nsec; }

#define MAX_REG 33
#define MAX_WORKERS 64
#define MAX_ACTIVE 64
#define MAX_JOBS 64
#define MAX_RB 128

typedef struct RegPlane { const uint8_t *base; ptrdiff_t linesize, size; uint64_t inv; int slot, plane, w, h; } RegPlane;

#include <pthread.h>

/* One per decoder instance (an avcodec context the application opened; with frame threads all its thread copies): shared by
 * every decoding thread of that decoder -- the device context, the geometry, and the ticket that keeps pictures in decode
 * order on the GPU (frame threads reach b200_frame_end out of order; hevc_frame_start is called in decode order).  A thread
 * reaches the instance it is working for through its ShimThread (`G` below). */
#define MAX_INST 8
typedef struct Instance {
    const void *key;                    /* instance_key() of the decoder that owns this entry, NULL = free */
    B200Ctx *ctx;
    B200Config cfg;
    int bd, B, cfi;
    int pw[3], ph[3];
    pthread_mutex_t mu;
    pthread_cond_t cv;
    unsigned next_ticket, turn;
    unsigned gen;                       /* bumped when the context is re-created for a new geometry */
    struct ShimThread *active[MAX_ACTIVE];   /* owners of the pictures between b200_frame_begin and b200_frame_end */
    int n_active;
    /* B200_SHIM_DUMP=<dir>: record only.  Every picture's work list is written to <dir>/pic_NNNNN.blob (decode order) and
     * nothing is sent to a GPU -- no device is needed, the decoder's output pictures stay untouched.  tests/ replay the dumps
     * through the CPU oracle and compare with the unmodified decoder: the recorder + wire format + oracle, end to end. */
    const char *dump_dir;
    int dump_no, configured, env_read;
    int in_flight;                      /* pictures begun whose packet has not ended yet (b200_frame_begin .. b200_frame_readback) */
    /* the submission thread: jobs by ticket (a decoding thread owns at most two tickets, MAX_JOBS covers 32 threads) */
    struct Job *jobq[MAX_JOBS];
    pthread_t sub_thread;
    pthread_cond_t cv_sub;
    int sub_running, sub_stop;
    int err_code; char errmsg[256];     /* latched by the submission thread, returned by the next b200_frame_begin / _end */
    /* read-backs in flight, keyed by the host frame's luma buffer [data0, end) (b200_output_wait): an output frame with a
     * conformance window points inside it (ff_hevc_output_frame moves the data pointers by the window's offsets) */
    struct { const uint8_t *data0, *end; uint32_t token; int state; unsigned seq; } rb[MAX_RB];
    unsigned rb_seq;
    uint64_t n_pictures, h2d_bytes, d2h_bytes;   /* B200_SHIM_REPORT=1: totals on stderr when the process ends */
    uint64_t ns_ctx, ns_rec, ns_pool, n_pool, bytes_pool, ns_first_submit;   /* ... and where the start-up time went */
} Instance;
static Instance g_insts[MAX_INST] = { [0 ... MAX_INST - 1] = { .mu = PTHREAD_MUTEX_INITIALIZER, .cv = PTHREAD_COND_INITIALIZER, .cv_sub = PTHREAD_COND_INITIALIZER } };
static pthread_mutex_t g_insts_mu = PTHREAD_MUTEX_INITIALIZER;      /* guards the keys */
static unsigned g_gen_counter;          /* context generations are unique across instances (a thread's recorders follow (instance, generation)) */

/* one picture on its way to the device (lives in the ShimThread that recorded it: two per thread, used alternately, so that
 * a thread can parse its next picture while the previous one's work list is still being uploaded) */
typedef struct Job {
    unsigned ticket;
    int kind;                           /* JOB_SKIP: the ticket only (abandoned / failed picture); JOB_PICTURE */
    const void *blob; uint64_t nbytes;
    uint8_t fill_slot[16]; int n_fill;  /* grey reference pictures this picture needs (generate_missing_ref), in front of it */
    int slot; void *planes[3]; int64_t strides[3]; int rb; unsigned rb_seq;   /* read-back into the host frame: entry of G.rb (and its generation) or -1 */
    int pending, done;                  /* pending: handed to the submission thread, its memory must not be reused before done */
    uint32_t upload_token; int uploaded;
} Job;
enum { JOB_SKIP = 0, JOB_PICTURE = 1 };

/* per thread: the owner of a picture (the thread that runs hevc_frame_start .. the end of decode_nal_unit for it; with
 * frame threads one per picture in flight, pthread_frame.c) or a slice / WPP worker attached to an owner's picture */
struct Job;
typedef struct ShimThread {
    Instance *inst;                     /* the decoder instance this block belongs to: a thread has one block per instance it works for */
    struct ShimThread *next_mine;       /* the same thread's block for another instance */
    B200Rec *rec;                       /* the recorder of the picture in progress: recs[cur] (workers: recs[0]) */
    B200Rec *recs[2];
    struct Job *jobs;                   /* [3], allocated with the first recorder */
    int rb_at; unsigned rb_seq;         /* entry of G.rb announced at b200_frame_begin for the picture in progress, or -1 */
    int cur;
    unsigned rec_gen;
    unsigned ticket;
    RegPlane reg[MAX_REG * 3];
    int n_reg, reg_hit, reg_hit2;
    const uint8_t *cur_base[3]; ptrdiff_t cur_ls[3], cur_size[3]; uint64_t cur_inv[3]; int cur_slot;
    uint8_t ref_slot[16]; int n_ref;
    /* pending in-place transform on the per-thread coefficient scratch (hevc.h:1063) */
    const int16_t *pend_ptr; int pend_kind, pend_flags, pend_col_limit;
    /* first list of a bi-predicted block: put_hevc_*pel() into the caller's tmp[] (hevc.c:1761) */
    const int16_t *first_tmp; B200McRec first;
    /* emulated_edge_mc results, keyed by destination buffer (lc->edge_emu_buffer / edge_emu_buffer2) */
    struct { const uint8_t *buf; ptrdiff_t ls; int slot, plane, x, y; } emu[2];
    int emu_next;
    int err; char errmsg[256];
    int in_frame;                                        /* 0 no picture, 1 owner of the picture in progress, 2 attached worker */
    int poc;
    unsigned frame_seq;                                  /* owner: bumped by every b200_frame_begin */
    struct ShimThread *workers[MAX_WORKERS]; int n_workers;   /* owner: workers that recorded part of this picture */
    struct ShimThread *att; unsigned att_seq;            /* worker: the owner it is attached to */
    int n_tu, n_intra, n_pu, n_dbk, n_sao, frame_no;   /* B200_SHIM_STATS=1: table calls per picture (stderr) */
    /* cross-component prediction (4:4:4 range extension): the owner's decoder context, this thread's local context (found by
     * the coefficient pointer), and the luma transform block the chroma blocks of the same TU refer to */
    HEVCContext *s; int ccp; HEVCLocalContext *lc;
    int counted;                                         /* this thread's picture is part of G.in_flight */
    int pic_cip, pic_tqb;                                /* the picture in progress needs the PU-type / is_pcm hand-over at its end */
    int dbd;                                             /* deblocking parameters of the picture in progress: 0 recorded from the host's filter calls, 1 derived on the device, 2 both (check) */
    struct { int x, y, log2, kind, flags, cl, parked; uint32_t park; } last_y;
    uint8_t fill_slot[16]; int n_fill;                  /* generate_missing_ref (hevc_refs.c:538): grey references this picture needs */
} ShimThread;
/* One heap block per thread, reached through an 8-byte initial-exec TLS pointer: a plain `static __thread ShimThread` in a
 * shared library costs a __tls_get_addr call per table call (2.4% of the hooked decoder's CPU time plus the PLT), and the
 * struct itself is too large for the static TLS surplus if libOpenHevc is dlopen()ed.  Blocks of threads that exited are
 * recycled, never freed: workers keep pointers to their owner's block (att), and frame_seq must stay monotonic. */
static __thread struct ShimThread *g_self __attribute__((tls_model("initial-exec")));      /* this thread's block for the instance it is working for */
static __thread struct ShimThread *g_mine __attribute__((tls_model("initial-exec")));      /* all blocks of this thread (next_mine) */
static pthread_key_t g_key;
static pthread_once_t g_key_once = PTHREAD_ONCE_INIT;
static pthread_mutex_t g_pool_mu = PTHREAD_MUTEX_INITIALIZER;
static ShimThread *g_pool[256]; static int g_pool_n;
static ShimThread g_oom = { .inst = &g_insts[0], .err = B200_ENOMEM, .errmsg = "out of memory (per-thread state of the B200 shim)" };

static void shim_thread_exit(void *p)
{
    pthread_mutex_lock(&g_pool_mu);
    for (ShimThread *t = p, *next; t; t = next) {
        next = t->next_mine;
        if (t == &g_oom) continue;
        t->in_frame = 0; t->next_mine = NULL;
        if (g_pool_n < 256) g_pool[g_pool_n++] = t;     /* else: leaked, 256 blocks of exited threads are already parked */
    }
    pthread_mutex_unlock(&g_pool_mu);
}
static void shim_key_make(void) { pthread_key_create(&g_key, shim_thread_exit); }
/* this thread's block for instance I (created on first use) becomes the current one */
static __attribute__((noinline)) ShimThread *shim_block_for(Instance *I)
{
    for (ShimThread *t = g_mine; t; t = t->next_mine) if (t->inst == I) return g_self = t;
    pthread_once(&g_key_once, shim_key_make);
    pthread_mutex_lock(&g_pool_mu);
    ShimThread *t = g_pool_n ? g_pool[--g_pool_n] : NULL;
    pthread_mutex_unlock(&g_pool_mu);
    if (t) { t->err = 0; t->n_fill = 0; t->n_workers = 0; t->att = NULL; }
    else t = calloc(1, sizeof(*t));
    if (!t) return g_self = &g_oom;
    t->inst = I;
    t->next_mine = g_mine; g_mine = t;
    pthread_setspecific(g_key, t);
    return g_self = t;
}
static __attribute__((noinline)) ShimThread *shim_self_slow(void) { return shim_block_for(&g_insts[0]); }
static inline ShimThread *shim_self(void)
{
    ShimThread *t = g_self;
    return __builtin_expect(t != NULL, 1) ? t : shim_self_slow();
}
#define g (*shim_self())
#define G (*g.inst)

static void fail(int code, const char *msg)
{
    if (!g.err) { g.err = code; snprintf(g.errmsg, sizeof(g.errmsg), "%s", msg); }
}
const char *b200_shim_error(void) { return g.err ? g.errmsg : (G.ctx ? b200_last_error(G.ctx) : ""); }

/* ---- decoder instances ---------------------------------------------------------------------------------------------
 * Which decoder does a context belong to?  Unthreaded and slice-threaded decoders: the AVCodecContext.  Frame threads decode on
 * COPIES of the context (pthread_frame.c:758-800), which all belong to the application's one decoder: a copy's
 * internal->thread_ctx_frame is its PerThreadContext, whose first member is the FrameThreadContext they share
 * (pthread_frame.c:56-57).  Callers that drive the tables without an AVCodecContext (oracle/replay_ref.c) are their own key. */
#include "libavcodec/internal.h"
static const void *instance_key(const HEVCContext *s)
{
    const AVCodecContext *a = s->avctx;
    if (!a) return s;
    /* (the copy of thread 0 is not marked is_copy, pthread_frame.c:797-812; the application's own context never decodes) */
    if ((a->active_thread_type & FF_THREAD_FRAME) && a->internal && a->internal->thread_ctx_frame) return *(void *const *)a->internal->thread_ctx_frame;
    return a;
}
/* the calling thread works for the decoder of `s` from here on (every hook that is handed a context starts with this) */
static int use_instance(const HEVCContext *s)
{
    const void *key = instance_key(s);
    ShimThread *t = shim_self();
    if (__atomic_load_n(&t->inst->key, __ATOMIC_RELAXED) == key) return 0;
    Instance *I = NULL;
    pthread_mutex_lock(&g_insts_mu);
    for (int i = 0; i < MAX_INST && !I; i++) if (g_insts[i].key == key) I = &g_insts[i];
    for (int i = 0; i < MAX_INST && !I; i++) if (!g_insts[i].key) { I = &g_insts[i]; __atomic_store_n(&I->key, key, __ATOMIC_RELAXED); }
    pthread_mutex_unlock(&g_insts_mu);
    if (!I) { fail(B200_ENOTSUP, "more than 8 decoders open in this process"); return B200_ENOTSUP; }
    shim_block_for(I);
    return 0;
}

static int thread_recorder(int k);
/* A table call on a thread that owns no picture: a slice / WPP / tile worker (execute2 job).  Attach it to the picture
 * in progress: own recorder, own reference table, a copy of the owner's plane registry. */
static int attach_to(const HEVCContext *owner)     /* owner: the context b200_frame_begin was called with, or NULL = "the one picture in progress" */
{
    pthread_mutex_lock(&G.mu);
    int rc = 0;
    ShimThread *o = NULL;
    if (owner) { for (int i = 0; i < G.n_active; i++) if (G.active[i]->s == owner) o = G.active[i]; }
    else if (G.n_active == 1) o = G.active[0];
    if (!o) {
        fail(B200_ENOTSUP, owner || !G.n_active ? "table call outside b200_frame_begin / b200_frame_end"
                                                : "table call from a worker thread with several pictures in progress (frame + slice threads combined) "
                                                  "and no b200_worker_begin hook in the decoder");
        /* nobody would collect this thread's error (it is on no picture's worker list): the whole decoder hears of it */
        if (!G.err_code) { G.err_code = g.err; snprintf(G.errmsg, sizeof(G.errmsg), "%s", g.errmsg); }
        rc = -1;
    } else {
        if (thread_recorder(0)) { fail(B200_ENOMEM, "b200_rec_create failed (worker)"); rc = -1; }
        if (!rc && o->n_workers == MAX_WORKERS) { fail(B200_ENOTSUP, "too many worker threads"); rc = -1; }
        if (!rc) {
            memcpy(g.reg, o->reg, sizeof(g.reg)); g.n_reg = o->n_reg;
            for (int p = 0; p < 3; p++) { g.cur_base[p] = o->cur_base[p]; g.cur_ls[p] = o->cur_ls[p]; g.cur_size[p] = o->cur_size[p]; g.cur_inv[p] = o->cur_inv[p]; }
            g.cur_slot = o->cur_slot; g.poc = o->poc;
            g.s = o->s; g.ccp = o->ccp; g.lc = NULL; g.last_y.log2 = 0; g.dbd = o->dbd;
            g.n_ref = 0; g.pend_ptr = NULL; g.first_tmp = NULL; g.emu[0].buf = g.emu[1].buf = NULL;
            g.n_tu = g.n_intra = g.n_pu = g.n_dbk = g.n_sao = 0;
            if (b200_rec_begin(g.rec, g.cur_slot, g.poc)) { fail(B200_ESTATE, "b200_rec_begin failed (worker)"); rc = -1; }
            else { o->workers[o->n_workers++] = &g; g.att = o; g.att_seq = o->frame_seq; g.in_frame = 2; }
        }
    }
    pthread_mutex_unlock(&G.mu);
    return rc;
}
static inline int attached(void)
{
    if (g.in_frame == 1) return 1;
    if (g.err) return 0;
    if (g.in_frame == 2 && g.att->in_frame == 1 && g.att->frame_seq == g.att_seq) return 1;
    return attach_to(NULL) == 0;
}
/* First statement of the decoder's execute2 jobs (hls_decode_entry_wpp / _tiles / _wpp_in_tiles, hevc.c:2751-2931), called with
 * the context the job belongs to (avctx->priv_data): the worker thread records for THAT picture.  With this hook frame threads
 * whose pictures are decoded by slice threads (-f 4, pthread.c:57-71) work: several pictures are in progress at once and a table
 * call alone cannot tell which one it belongs to.  Without it (-f 2 only) a worker attaches itself on its first table call. */
int b200_worker_begin(HEVCContext *owner)
{
    if (use_instance(owner)) return g.err;
    ShimThread *t = &g;
    if (t->in_frame == 1 && t->s == owner) return 0;                       /* the owner thread runs a job itself */
    if (t->err) return t->err;
    if (t->in_frame == 2 && t->att->s == owner && t->att->in_frame == 1 && t->att->frame_seq == t->att_seq) return 0;
    if (t->in_frame == 1) { fail(B200_ESTATE, "b200_worker_begin on a thread that owns another picture"); return t->err; }
    t->in_frame = 0;
    return attach_to(owner) ? t->err : 0;
}

/* ---- pointer -> (slot, plane, x, y) ---------------------------------------------------------------- */
/* offset / linesize without a division (several hundred thousand calls per 4K picture): inv = floor(2^48 / ls) + 1 is exact
 * for off * ls < 2^48, i.e. any plane below 4 GB with a line below 64 KB; inv == 0 (odd geometry) falls back to dividing */
static inline uint64_t row_inverse(ptrdiff_t ls) { return ls > 0 && ls < 65536 ? (1ull << 48) / (uint64_t)ls + 1 : 0; }
static inline uint32_t row_of(uint32_t off, uint32_t ls, uint64_t inv)
{
    return inv ? (uint32_t)(((unsigned __int128)off * inv) >> 48) : off / ls;
}

static int locate_cur(const uint8_t *p, int *plane, int *x, int *y)
{
    if (!attached()) return -1;
    ShimThread *t = &g;
    for (int c = 0; c < 3; c++) {
        const ptrdiff_t off = p - t->cur_base[c];
        if (off >= 0 && off < t->cur_size[c]) {
            const uint32_t o = (uint32_t)off, ls = (uint32_t)t->cur_ls[c], row = row_of(o, ls, t->cur_inv[c]);
            *plane = c; *y = (int)row; *x = (int)((o - row * ls) >> (G.B - 1));
            return 0;
        }
    }
    fail(B200_EINVAL, "destination pointer is not inside the current picture");
    return -1;
}

static int locate_ref(const uint8_t *p, int plane_hint, int *slot, int *x, int *y)
{
    if (!attached()) return -1;
    ShimThread *t = &g;
    for (int e = 0; e < 2; e++)          /* source inside an edge-emulation buffer? (hevc.c:1673) */
        if (t->emu[e].buf && p >= t->emu[e].buf && p < t->emu[e].buf + t->emu[e].ls * (MAX_PB_SIZE + 7)) {
            ptrdiff_t off = p - t->emu[e].buf;
            *slot = t->emu[e].slot; *y = t->emu[e].y + (int)(off / t->emu[e].ls); *x = t->emu[e].x + (int)(off % t->emu[e].ls) / G.B;
            return t->emu[e].plane;
        }
    /* The two reference pictures hit last come first (planes are registered three per picture, Y Cb Cr): a block's calls go
     * luma L0, luma L1, Cb L0, Cb L1, Cr L0, Cr L1, and neighbouring blocks mostly use the same one or two pictures. */
    for (int k = -6; k < t->n_reg; k++) {
        const int i = k < -3 ? t->reg_hit + (k + 6) : k < 0 ? t->reg_hit2 + (k + 3) : k;
        if (i < 0 || i >= t->n_reg) continue;
        const RegPlane *r = &t->reg[i];
        ptrdiff_t off = p - r->base;
        if (off >= 0 && off < r->size && (plane_hint < 0 || r->plane == plane_hint)) {
            const uint32_t o = (uint32_t)off, ls = (uint32_t)r->linesize, row = row_of(o, ls, r->inv);
            *slot = r->slot; *y = (int)row; *x = (int)((o - row * ls) >> (G.B - 1));
            const int first = i - r->plane;                      /* index of the picture's luma plane */
            if (first != t->reg_hit) { t->reg_hit2 = t->reg_hit; t->reg_hit = first; }
            return r->plane;
        }
    }
    fail(B200_EINVAL, "source pointer is not inside a registered reference picture");
    return -1;
}

static int ref_index(int slot)
{
    for (int i = 0; i < g.n_ref; i++) if (g.ref_slot[i] == slot) return i;
    if (g.n_ref == 16) { fail(B200_ENOTSUP, "more than 16 reference pictures"); return 0; }
    g.ref_slot[g.n_ref] = (uint8_t)slot;
    return g.n_ref++;
}

/* ---- residual slots --------------------------------------------------------------------------------- */
static void rec_idct(int16_t *c, int col_limit) { g.pend_ptr = c; g.pend_kind = B200_TU_IDCT; g.pend_flags = 0; g.pend_col_limit = col_limit; }
static void rec_idct_dc(int16_t *c) { g.pend_ptr = c; g.pend_kind = B200_TU_DC; g.pend_flags = 0; g.pend_col_limit = 0; }
static void rec_idct_4x4_luma(int16_t *c) { g.pend_ptr = c; g.pend_kind = B200_TU_DST; g.pend_flags = 0; g.pend_col_limit = 0; }
static void rec_transform_skip(int16_t *c, int16_t log2_size) { (void)log2_size; g.pend_ptr = c; g.pend_kind = B200_TU_SKIP; g.pend_flags = 0; g.pend_col_limit = 0; }
static void rec_transform_rdpcm(int16_t *c, int16_t log2_size, int mode)
{
    (void)log2_size;
    if (g.pend_ptr != c) { g.pend_ptr = c; g.pend_kind = B200_TU_BYPASS; g.pend_col_limit = 0; }
    g.pend_flags = B200_TUF_RDPCM | (mode ? B200_TUF_RDPCM_VERT : 0);
}
/* Cross-component prediction (hevc.c:1295-1360, hevc_cabac.c:1942-1948).  Between the chroma block's idct() call and its
 * transform_add() call the reference adds (res_scale_val * luma residual) >> 3 to the chroma coefficients ON THE HOST, reading
 * the luma block it has transformed in place -- which, with the transforms recorded instead of executed, still holds the
 * dequantised luma COEFFICIENTS.  The term it added is therefore known exactly (same arrays, same arithmetic) and is taken
 * out again; the device gets the chroma block as the decoder parsed it, the luma block a second time (parked only), and a
 * record that combines the two residuals there.  The local context (res_scale_val, cross_pf, the luma array) is found through
 * the coefficient pointer: the tables carry no context argument. */
static HEVCLocalContext *local_context_of(const int16_t *coeffs)
{
    ShimThread *t = &g;
    if (t->lc && coeffs >= t->lc->tu.coeffs[0] && coeffs < t->lc->tu.coeffs[0] + 2 * MAX_TB_SIZE * MAX_TB_SIZE) return t->lc;
    HEVCContext *s = t->s;
    for (int i = -1; s && i < MAX_NB_THREADS; i++) {
        HEVCLocalContext *lc = i < 0 ? s->HEVClc : s->HEVClcList[i];
        if (lc && coeffs >= lc->tu.coeffs[0] && coeffs < lc->tu.coeffs[0] + 2 * MAX_TB_SIZE * MAX_TB_SIZE) return t->lc = lc;
    }
    return NULL;
}
static int rec_cross_component(int plane, int x, int y, int log2, int16_t *coeffs, int kind, int flags, int cl, int pending)
{
    ShimThread *t = &g;
    HEVCLocalContext *lc = local_context_of(coeffs);
    if (!lc) { fail(B200_EINVAL, "cross_component_prediction: coefficient block outside every local context"); return -1; }
    if (!lc->tu.cross_pf || !lc->tu.res_scale_val) return 0;                 /* nothing was added on the host */
    if (t->last_y.log2 != log2 || t->last_y.x != x || t->last_y.y != y) { fail(B200_ESTATE, "cross_component_prediction without the luma block of the same TU"); return -1; }
    const int16_t *cy = lc->tu.coeffs[0];
    const int scale = lc->tu.res_scale_val, nn = 1 << (2 * log2);
    int16_t own[MAX_TB_SIZE * MAX_TB_SIZE];
    int has_c = pending;
    for (int i = 0; i < nn; i++) {
        own[i] = (int16_t)(coeffs[i] - ((scale * cy[i]) >> 3));
        has_c |= own[i] != 0;
    }
    int rc = 0;
    uint32_t off_c = 0;
    if (!t->last_y.parked) {
        rc = b200_rec_tu_parked(t->rec, 0, x, y, log2, t->last_y.kind, t->last_y.flags, t->last_y.cl, cy, &t->last_y.park);
        t->last_y.parked = 1;
    }
    if (!rc && has_c) rc = b200_rec_tu_parked(t->rec, plane, x, y, log2, kind, flags, cl, own, &off_c);
    if (!rc) rc = b200_rec_ccp(t->rec, plane, x, y, log2, scale, t->last_y.park, has_c, off_c);
    if (rc) { fail(rc, "recording a cross-component prediction block failed"); return -1; }
    return 1;
}

static void rec_transform_add(uint8_t *dst, int16_t *coeffs, ptrdiff_t stride, int log2)
{
    int plane, x, y;
    (void)stride;
    if (locate_cur(dst, &plane, &x, &y)) return;
    int kind = B200_TU_BYPASS, flags = 0, cl = 0;
    const int pending = g.pend_ptr == coeffs;
    if (pending) { kind = g.pend_kind; flags = g.pend_flags; cl = g.pend_col_limit; }
    g.pend_ptr = NULL;
    g.n_tu++;
    if (g.ccp) {
        if (plane == 0) { g.last_y.x = x; g.last_y.y = y; g.last_y.log2 = log2; g.last_y.kind = kind; g.last_y.flags = flags; g.last_y.cl = cl; g.last_y.parked = 0; }
        else if (rec_cross_component(plane, x, y, log2, coeffs, kind, flags, cl, pending)) return;
    }
    int rc = b200_rec_tu(g.rec, plane, x, y, log2, kind, flags, cl, coeffs, -1);
    if (rc) fail(rc, "b200_rec_tu failed");
}
static void rec_add4(uint8_t *d, int16_t *c, ptrdiff_t s) { rec_transform_add(d, c, s, 2); }
static void rec_add8(uint8_t *d, int16_t *c, ptrdiff_t s) { rec_transform_add(d, c, s, 3); }
static void rec_add16(uint8_t *d, int16_t *c, ptrdiff_t s) { rec_transform_add(d, c, s, 4); }
static void rec_add32(uint8_t *d, int16_t *c, ptrdiff_t s) { rec_transform_add(d, c, s, 5); }

static void rec_put_pcm(uint8_t *dst, ptrdiff_t stride, int width, int height, GetBitContext *gb, int pcm_bit_depth)
{
    int plane, x, y;
    int16_t smp[32 * 32];
    (void)stride;
    if (locate_cur(dst, &plane, &x, &y)) return;
    if (width > 32 || height > 64) { fail(B200_ENOTSUP, "pcm block too large"); return; }
    /* square blocks per plane; 4:2:2 chroma (w x 2w) is recorded as two squares */
    for (int part = 0; part < height / width; part++) {
        for (int i = 0; i < width * width; i++) smp[i] = (int16_t)(get_bits(gb, pcm_bit_depth) << (G.bd - pcm_bit_depth));
        int log2 = 0;
        while ((1 << log2) < width) log2++;
        if (log2 < 2) { fail(B200_ENOTSUP, "pcm block smaller than 4x4"); return; }
        int rc = b200_rec_pcm(g.rec, plane, x, y + part * width, log2, smp);
        if (rc) fail(rc, "b200_rec_pcm failed");
    }
}

/* ---- inter prediction slots --------------------------------------------------------------------------- */
static int mc_fill(B200McRec *m, int list, const uint8_t *src, int mx, int my, int chroma_hint)
{
    int slot, sx, sy;
    int plane = locate_ref(src, -1, &slot, &sx, &sy);
    if (plane < 0) return -1;
    (void)chroma_hint;
    const int ri = ref_index(slot);
    /* The origin travels as int16.  A legal motion vector reaches 2^13 samples beyond a picture of at most 2^14, so this clamp
     * never acts on a legal stream -- and must not: the device reads the block's motion vector back from source position
     * and fraction (k_dbd.cuh).  Samples outside the picture clamp one by one on the device (videodsp_template.c:26-100). */
    if (sx < -16384) sx = -16384; if (sx > 32767) sx = 32767;
    if (sy < -16384) sy = -16384; if (sy > 32767) sy = 32767;
    if (list == 0) { m->ref0 = (uint8_t)ri; m->sx0 = (int16_t)sx; m->sy0 = (int16_t)sy; m->frac0 = (uint8_t)(mx | (my << 4)); }
    else           { m->ref1 = (uint8_t)ri; m->sx1 = (int16_t)sx; m->sy1 = (int16_t)sy; m->frac1 = (uint8_t)(mx | (my << 4)); }
    return plane;
}

static void mc_first(int16_t *dst, uint8_t *src, int height, intptr_t mx, intptr_t my, int width, int chroma)
{
    memset(&g.first, 0, sizeof(g.first));
    g.first.w = (uint8_t)width; g.first.h = (uint8_t)height;
    g.first.flags = (uint8_t)(B200_MCF_BI | (chroma ? B200_MCF_CHROMA : 0));
    if (mc_fill(&g.first, 0, src, (int)mx, (int)my, chroma) < 0) return;
    g.first_tmp = dst;
}
static void mc_emit(B200McRec *m, uint8_t *dst)
{
    int plane, x, y;
    if (locate_cur(dst, &plane, &x, &y)) return;
    m->plane = (uint8_t)plane; m->x = (uint16_t)x; m->y = (uint16_t)y;
    g.n_pu++;
    int rc = b200_rec_mc(g.rec, m);
    if (rc) fail(rc, "b200_rec_mc failed");
}
static void mc_uni(uint8_t *dst, uint8_t *src, int height, int mx, int my, int width, int chroma, int weighted, int denom, int wx, int ox)
{
    B200McRec m;
    memset(&m, 0, sizeof(m));
    m.w = (uint8_t)width; m.h = (uint8_t)height;
    m.flags = (uint8_t)((chroma ? B200_MCF_CHROMA : 0) | (weighted ? B200_MCF_WEIGHTED : 0));
    m.denom = (uint8_t)denom; m.w0 = (int16_t)wx; m.o0 = (int16_t)ox;
    if (mc_fill(&m, 0, src, mx, my, chroma) < 0) return;
    mc_emit(&m, dst);
}
static void mc_bi(uint8_t *dst, uint8_t *src, int16_t *src2, int height, int mx, int my, int width, int chroma, int weighted,
                  int denom, int wx0, int wx1, int ox0, int ox1)
{
    if (src2 != g.first_tmp) { fail(B200_ESTATE, "put_hevc_*_bi without the matching first-list call"); return; }
    B200McRec m = g.first;
    g.first_tmp = NULL;
    if (m.w != width || m.h != height) { fail(B200_ESTATE, "bi-prediction block size mismatch"); return; }
    m.flags |= weighted ? B200_MCF_WEIGHTED : 0;
    m.denom = (uint8_t)denom; m.w0 = (int16_t)wx0; m.w1 = (int16_t)wx1; m.o0 = (int16_t)ox0; m.o1 = (int16_t)ox1;
    if (mc_fill(&m, 1, src, mx, my, chroma) < 0) return;
    mc_emit(&m, dst);
}

#define MC_FAMILY(T, CH) \
static void rec_##T(int16_t *dst, ptrdiff_t ds, uint8_t *src, ptrdiff_t ss, int h, intptr_t mx, intptr_t my, int w) \
{ (void)ds; (void)ss; mc_first(dst, src, h, mx, my, w, CH); } \
static void rec_##T##_uni(uint8_t *dst, ptrdiff_t ds, uint8_t *src, ptrdiff_t ss, int h, intptr_t mx, intptr_t my, int w) \
{ (void)ds; (void)ss; mc_uni(dst, src, h, (int)mx, (int)my, w, CH, 0, 0, 0, 0); } \
static void rec_##T##_uni_w(uint8_t *dst, ptrdiff_t ds, uint8_t *src, ptrdiff_t ss, int h, int denom, int wx, int ox, intptr_t mx, intptr_t my, int w) \
{ (void)ds; (void)ss; mc_uni(dst, src, h, (int)mx, (int)my, w, CH, 1, denom, wx, ox); } \
static void rec_##T##_bi(uint8_t *dst, ptrdiff_t ds, uint8_t *src, ptrdiff_t ss, int16_t *src2, ptrdiff_t s2, int h, intptr_t mx, intptr_t my, int w) \
{ (void)ds; (void)ss; (void)s2; mc_bi(dst, src, src2, h, (int)mx, (int)my, w, CH, 0, 0, 0, 0, 0, 0); } \
static void rec_##T##_bi_w(uint8_t *dst, ptrdiff_t ds, uint8_t *src, ptrdiff_t ss, int16_t *src2, ptrdiff_t s2, int h, int denom, int wx0, int wx1, int ox0, int ox1, intptr_t mx, intptr_t my, int w) \
{ (void)ds; (void)ss; (void)s2; mc_bi(dst, src, src2, h, (int)mx, (int)my, w, CH, 1, denom, wx0, wx1, ox0, ox1); }
MC_FAMILY(qpel, 0)
MC_FAMILY(epel, 1)

/* vdsp.emulated_edge_mc: remember where the window really comes from; nothing is copied (the device clamps) */
static void rec_emulated_edge_mc(uint8_t *buf, const uint8_t *src, ptrdiff_t buf_linesize, ptrdiff_t src_linesize,
                                 int block_w, int block_h, int src_x, int src_y, int w, int h)
{
    (void)block_w; (void)block_h; (void)w; (void)h;
    if (!attached()) return;
    const uint8_t *base = src - ((ptrdiff_t)src_y * src_linesize + (ptrdiff_t)src_x * G.B);
    for (int i = 0; i < g.n_reg; i++)
        if (g.reg[i].base == base && g.reg[i].linesize == src_linesize) {
            int e = (g.emu[0].buf == buf) ? 0 : (g.emu[1].buf == buf) ? 1 : (g.emu_next++ & 1);
            g.emu[e].buf = buf; g.emu[e].ls = buf_linesize; g.emu[e].slot = g.reg[i].slot; g.emu[e].plane = g.reg[i].plane;
            g.emu[e].x = src_x; g.emu[e].y = src_y;
            return;
        }
    fail(B200_EINVAL, "emulated_edge_mc source does not belong to a registered reference picture");
}

/* ---- deblocking slots ------------------------------------------------------------------------------------ */
static void rec_dbk(uint8_t *pix, int vertical, int beta, int *tc, uint8_t *no_p, uint8_t *no_q)
{
    int plane, x, y;
    if (locate_cur(pix, &plane, &x, &y)) return;
    g.n_dbk++;
    int rc = b200_rec_deblock(g.rec, plane, vertical, x, y, beta, tc, no_p, no_q);
    if (rc) fail(rc, "b200_rec_deblock failed");
}
static void rec_h_luma(uint8_t *p, ptrdiff_t s, int beta, int *tc, uint8_t *np, uint8_t *nq) { (void)s; rec_dbk(p, 0, beta, tc, np, nq); }
static void rec_v_luma(uint8_t *p, ptrdiff_t s, int beta, int *tc, uint8_t *np, uint8_t *nq) { (void)s; rec_dbk(p, 1, beta, tc, np, nq); }
static void rec_h_chroma(uint8_t *p, ptrdiff_t s, int *tc, uint8_t *np, uint8_t *nq) { (void)s; rec_dbk(p, 0, 0, tc, np, nq); }
static void rec_v_chroma(uint8_t *p, ptrdiff_t s, int *tc, uint8_t *np, uint8_t *nq) { (void)s; rec_dbk(p, 1, 0, tc, np, nq); }

/* ---- SAO slots (dst = picture, src = the host's sao_frame copy, which the device does not need) ---------- */
static void rec_sao(uint8_t *dst, SAOParams *sao, int *borders, int c_idx, int type, int variant, uint8_t *ve, uint8_t *he, uint8_t *de)
{
    int plane, x, y;
    if (locate_cur(dst, &plane, &x, &y)) return;
    B200SaoRec r;
    memset(&r, 0, sizeof(r));
    r.type = (uint8_t)type;
    r.param = type == B200_SAO_BAND ? sao->band_position[c_idx] : sao->eo_class[c_idx];
    r.borders = (uint8_t)((borders[0] ? 1 : 0) | (borders[1] ? 2 : 0) | (borders[2] ? 4 : 0) | (borders[3] ? 8 : 0));
    if (variant) r.edges = (uint8_t)((ve[0] ? 1 : 0) | (ve[1] ? 2 : 0) | (he[0] ? 4 : 0) | (he[1] ? 8 : 0) | (de[0] ? 16 : 0) | (de[1] ? 32 : 0) | (de[2] ? 64 : 0) | (de[3] ? 128 : 0));
    r.variant = (uint8_t)variant;
    for (int k = 0; k < 5; k++) r.offset_val[k] = sao->offset_val[c_idx][k];
    g.n_sao++;
    int rc = b200_rec_sao(g.rec, plane, x, y, &r);
    if (rc) fail(rc, "b200_rec_sao failed");
}
static void rec_sao_band(uint8_t *dst, uint8_t *src, ptrdiff_t sd, ptrdiff_t ss, SAOParams *sao, int *borders, int w, int h, int c_idx)
{ (void)src; (void)sd; (void)ss; (void)w; (void)h; rec_sao(dst, sao, borders, c_idx, B200_SAO_BAND, 0, NULL, NULL, NULL); }
static void rec_sao_edge0(uint8_t *dst, uint8_t *src, ptrdiff_t sd, ptrdiff_t ss, SAOParams *sao, int *borders, int w, int h, int c_idx, uint8_t *ve, uint8_t *he, uint8_t *de)
{ (void)src; (void)sd; (void)ss; (void)w; (void)h; rec_sao(dst, sao, borders, c_idx, B200_SAO_EDGE, 0, ve, he, de); }
static void rec_sao_edge1(uint8_t *dst, uint8_t *src, ptrdiff_t sd, ptrdiff_t ss, SAOParams *sao, int *borders, int w, int h, int c_idx, uint8_t *ve, uint8_t *he, uint8_t *de)
{ (void)src; (void)sd; (void)ss; (void)w; (void)h; rec_sao(dst, sao, borders, c_idx, B200_SAO_EDGE, 1, ve, he, de); }

/* ---- intra slot: the availability derivation of hevcpred_template.c:82-109, then one record ------------------ */
static void rec_intra(HEVCContext *s, int x0, int y0, int log2_size, int c_idx)
{
    HEVCLocalContext *lc = s->HEVClc;
    const HEVCSPS *sps = s->sps;
    if (!attached()) return;
    const int hshift = sps->hshift[c_idx], vshift = sps->vshift[c_idx];
    const int size = 1 << log2_size;
    const int size_l_h = size << hshift, size_l_v = size << vshift;
    const int tbs_h = size_l_h >> sps->log2_min_tb_size, tbs_v = size_l_v >> sps->log2_min_tb_size;
    const int x_tb = (x0 >> sps->log2_min_tb_size) & sps->tb_mask, y_tb = (y0 >> sps->log2_min_tb_size) & sps->tb_mask;
    const int zstride = sps->tb_mask + 2;
    const int *zs = s->pps->min_tb_addr_zs;
    const int cur = zs[y_tb * zstride + x_tb];
    const int bl = lc->na.cand_bottom_left && cur > zs[((y_tb + tbs_v) & sps->tb_mask) * zstride + x_tb - 1];
    const int ur = lc->na.cand_up_right && cur > zs[(y_tb - 1) * zstride + ((x_tb + tbs_h) & sps->tb_mask)];
    int bls = (FFMIN(y0 + 2 * size_l_v, sps->height) - (y0 + size_l_v)) >> vshift;
    int trs = (FFMIN(x0 + 2 * size_l_h, sps->width) - (x0 + size_l_h)) >> hshift;
    int flags = (lc->na.cand_up_left ? B200_INF_UP_LEFT : 0) | (lc->na.cand_up ? B200_INF_UP : 0) | (ur ? B200_INF_UP_RIGHT : 0) |
                (lc->na.cand_left ? B200_INF_LEFT : 0) | (bl ? B200_INF_BOTTOM_LEFT : 0);
    if (!sps->spsRext.intra_smoothing_disabled_flag && (c_idx == 0 || sps->chroma_array_type == 3)) flags |= B200_INF_FILTER;
    if (sps->sps_strong_intra_smoothing_enable_flag) flags |= B200_INF_STRONG;
    if (ur && trs <= 0) { flags &= ~B200_INF_UP_RIGHT; if (!(flags & B200_INF_UP)) fail(B200_ENOTSUP, "up-right available with no sample inside the picture"); }
    if (bl && bls <= 0) { flags &= ~B200_INF_BOTTOM_LEFT; if (!(flags & B200_INF_LEFT)) fail(B200_ENOTSUP, "bottom-left available with no sample inside the picture"); }
    const int mode = c_idx ? lc->tu.intra_pred_mode_c : lc->tu.intra_pred_mode;
    g.n_intra++;
    int rc = b200_rec_intra(g.rec, c_idx, x0 >> hshift, y0 >> vshift, log2_size, mode, flags, trs, bls);
    if (rc) fail(rc, "b200_rec_intra failed");
}
static void rec_intra_2(HEVCContext *s, int x0, int y0, int c) { rec_intra(s, x0, y0, 2, c); }
static void rec_intra_3(HEVCContext *s, int x0, int y0, int c) { rec_intra(s, x0, y0, 3, c); }
static void rec_intra_4(HEVCContext *s, int x0, int y0, int c) { rec_intra(s, x0, y0, 4, c); }
static void rec_intra_5(HEVCContext *s, int x0, int y0, int c) { rec_intra(s, x0, y0, 5, c); }

/* ---- deblocking control on the device (SURVEY.md 8f N2) -------------------------------------------------------------------
 * Two guards in hevc_filter.c (INTEGRATION.md): b200_bs_on_device() as the first statement of
 * ff_hevc_deblocking_boundary_strengths() records the call as one word (position, size, and whether the block's top / left
 * edge takes part: the slice / tile boundary rules of :832-839 / :870-877 need the local context, so they are evaluated here)
 * and lets the function return; b200_deblock_on_device() does the same for deblocking_filter_CTB().  The device derives
 * boundary strengths, tc and beta from the picture's own records (k_dbd.cuh).  B200_DBD=0: off (the reference derives, its
 * filter calls are recorded); 2: both, and the device compares.  Pictures of tile streams decoded with several threads keep
 * the host path (tiles_filters recomputes the strengths at tile borders with its own rules, hevc.c:2967-3003). */
static int dbd_mode(void)
{
    static int mode = -1;                          /* every frame thread asks: relaxed atomics, the value is the same whoever writes it */
    int m = __atomic_load_n(&mode, __ATOMIC_RELAXED);
    if (m < 0) { const char *e = getenv("B200_DBD"); m = e ? atoi(e) : 1; if (m < 0 || m > 2) m = 0; __atomic_store_n(&mode, m, __ATOMIC_RELAXED); }
    return m;
}
int b200_bs_on_device(HEVCContext *s, int x0, int y0, int log2_size)
{
    if (!attached() || !g.dbd) return 0;
    const HEVCLocalContext *lc = s->HEVClc;
    const int ctb_mask = (1 << s->sps->log2_ctb_size) - 1;
    int top = 0, left = 0;
    if (y0 > 0 && (y0 & 7) == 0) {
        const int bd_slice = s->sh.slice_loop_filter_across_slices_enabled_flag || !(lc->slice_or_tiles_up_boundary & 1);
        const int bd_tiles = s->pps->loop_filter_across_tiles_enabled_flag || !(lc->slice_or_tiles_up_boundary & 2);
        top = (bd_slice && bd_tiles) || (y0 & ctb_mask);
    }
    if (x0 > 0 && (x0 & 7) == 0) {
        const int bd_slice = s->sh.slice_loop_filter_across_slices_enabled_flag || !(lc->slice_or_tiles_left_boundary & 1);
        const int bd_tiles = s->pps->loop_filter_across_tiles_enabled_flag || !(lc->slice_or_tiles_left_boundary & 2);
        left = (bd_slice && bd_tiles) || (x0 & ctb_mask);
    }
    int rc = b200_rec_bs_leaf(g.rec, x0, y0, log2_size, top, left);
    if (rc) fail(rc, "b200_rec_bs_leaf failed");
    return g.dbd == 1;
}
int b200_deblock_on_device(void)
{
    ShimThread *t = g_self;
    return t && (t->in_frame == 1 || (t->in_frame == 2 && t->att->in_frame == 1 && t->att->frame_seq == t->att_seq)) && t->dbd == 1;
}

/* ---- table installation ------------------------------------------------------------------------------------- */
/* The host copies of the picture are dead once the tables record instead of computing: the one place where the reference
 * still moves whole CTBs of them around (copy_CTB in sao_filter_CTB, hevc_filter.c:151-161, 269, 305; 6 % of the hooked
 * decoder's CPU time on a dense 4K stream, 24 % on a lightly coded one) may skip the work. */
static int g_tables_installed;          /* 0 -> 1 once, by whichever thread initialises its tables first */
int b200_host_pixels_unused(void) { return __atomic_load_n(&g_tables_installed, __ATOMIC_RELAXED); }

void ff_hevcdsp_init_b200(HEVCDSPContext *c, const int bit_depth)
{
    (void)bit_depth;
    __atomic_store_n(&g_tables_installed, 1, __ATOMIC_RELAXED);
    c->put_pcm = rec_put_pcm;
    c->transform_add[0] = rec_add4; c->transform_add[1] = rec_add8; c->transform_add[2] = rec_add16; c->transform_add[3] = rec_add32;
    c->transform_skip = rec_transform_skip;
    c->transform_rdpcm = rec_transform_rdpcm;
    c->idct_4x4_luma = rec_idct_4x4_luma;
    for (int i = 0; i < 4; i++) { c->idct[i] = rec_idct; c->idct_dc[i] = rec_idct_dc; }
    c->sao_band_filter = rec_sao_band;
    c->sao_edge_filter[0] = rec_sao_edge0; c->sao_edge_filter[1] = rec_sao_edge1;
    for (int i = 0; i < 10; i++)
        for (int j = 0; j < 2; j++)
            for (int k = 0; k < 2; k++) {
                c->put_hevc_qpel[i][j][k] = rec_qpel; c->put_hevc_qpel_uni[i][j][k] = rec_qpel_uni; c->put_hevc_qpel_uni_w[i][j][k] = rec_qpel_uni_w;
                c->put_hevc_qpel_bi[i][j][k] = rec_qpel_bi; c->put_hevc_qpel_bi_w[i][j][k] = rec_qpel_bi_w;
                c->put_hevc_epel[i][j][k] = rec_epel; c->put_hevc_epel_uni[i][j][k] = rec_epel_uni; c->put_hevc_epel_uni_w[i][j][k] = rec_epel_uni_w;
                c->put_hevc_epel_bi[i][j][k] = rec_epel_bi; c->put_hevc_epel_bi_w[i][j][k] = rec_epel_bi_w;
            }
    c->hevc_h_loop_filter_luma = rec_h_luma; c->hevc_v_loop_filter_luma = rec_v_luma;
    c->hevc_h_loop_filter_chroma = rec_h_chroma; c->hevc_v_loop_filter_chroma = rec_v_chroma;
    c->hevc_h_loop_filter_luma_c = rec_h_luma; c->hevc_v_loop_filter_luma_c = rec_v_luma;
    c->hevc_h_loop_filter_chroma_c = rec_h_chroma; c->hevc_v_loop_filter_chroma_c = rec_v_chroma;
}

void ff_hevcpred_init_b200(HEVCPredContext *c, const int bit_depth)
{
    (void)bit_depth;
    c->intra_pred[0] = rec_intra_2; c->intra_pred[1] = rec_intra_3; c->intra_pred[2] = rec_intra_4; c->intra_pred[3] = rec_intra_5;
    /* pred_planar / pred_dc / pred_angular are only reached through intra_pred: left untouched */
}

void ff_videodsp_init_b200(VideoDSPContext *c, int bpc)
{
    (void)bpc;
    c->emulated_edge_mc = rec_emulated_edge_mc;
}

/* ---- frame life cycle ----------------------------------------------------------------------------------------- */
/* recorder k (0 / 1) of the calling thread, created on first use and re-created when the geometry changed; becomes g.rec.
 * Called with G.mu held. */
static int thread_recorder(int k)
{
    ShimThread *t = &g;
    if (t->rec_gen != G.gen) {
        for (int i = 0; i < 2; i++) if (t->recs[i]) { b200_rec_destroy(t->recs[i]); t->recs[i] = NULL; }
        t->rec_gen = G.gen;
    }
    if (!t->jobs && !(t->jobs = calloc(3, sizeof(Job)))) return B200_ENOMEM;     /* [2]: the ticket-only job of ticket_skip */
    if (!t->recs[k]) {
        const uint64_t t0 = now_ns();
        int rc = b200_rec_create(&G.cfg, &t->recs[k]);
        G.ns_rec += now_ns() - t0;
        if (rc) return rc;
    }
    t->rec = t->recs[k];
    return 0;
}

static void latch_global(int code, const char *msg)         /* G.mu held */
{
    if (!G.err_code) { G.err_code = code; snprintf(G.errmsg, sizeof(G.errmsg), "%s", msg ? msg : "B200 back end failed"); }
}
static int global_error(void)                                /* a failure of the submission thread reaches every decoding thread */
{
    int e = __atomic_load_n(&G.err_code, __ATOMIC_ACQUIRE);
    if (e && !g.err) {
        pthread_mutex_lock(&G.mu);
        fail(G.err_code, G.errmsg);
        pthread_mutex_unlock(&G.mu);
    }
    return e;
}

/* ---- the submission thread: the only thread that drives the device context ---- */
static int process_job(Job *j, char *msg, size_t msg_n)
{
    int rc = 0;
    const int drop = G.dump_dir && !strcmp(G.dump_dir, "-");      /* "-": record and drop (host-side timing without a device) */
    for (int i = 0; i < j->n_fill && !rc; i++) {                  /* grey reference pictures, in decode order with everything else */
        const int grey = 1 << (G.bd - 1);
        if (drop) continue;
        if (G.dump_dir) {
            char path[1024];
            snprintf(path, sizeof(path), "%s/pic_%05d.fill", G.dump_dir, G.dump_no);
            FILE *f = fopen(path, "a");
            if (f) { fprintf(f, "%d %d\n", j->fill_slot[i], grey); fclose(f); } else rc = B200_EINVAL;
        } else rc = b200_slot_fill(G.ctx, j->fill_slot[i], grey);
    }
    if (rc) { snprintf(msg, msg_n, "grey reference fill failed: %s", G.ctx ? b200_last_error(G.ctx) : "dump"); return rc; }
    if (j->kind != JOB_PICTURE) return 0;
    if (drop) { G.dump_no++; return 0; }
    if (G.dump_dir) {
        char path[1024];
        snprintf(path, sizeof(path), "%s/pic_%05d.blob", G.dump_dir, G.dump_no++);
        FILE *f = fopen(path, "wb");
        if (!f || fwrite(j->blob, 1, (size_t)j->nbytes, f) != (size_t)j->nbytes) { rc = B200_EINVAL; snprintf(msg, msg_n, "B200_SHIM_DUMP: cannot write the work list"); }
        if (f) fclose(f);
        return rc;
    }
    rc = b200_frame_submit_ex(G.ctx, j->blob, j->nbytes, &j->upload_token);
    if (!rc) { j->uploaded = 1; G.n_pictures++; G.h2d_bytes += j->nbytes; if (j->rb >= 0) for (int p = 0; p < 3; p++) G.d2h_bytes += (uint64_t)G.pw[p] * G.ph[p] * G.B; }
    uint32_t token = 0;
    if (!rc && j->rb >= 0) rc = b200_slot_readback_async(G.ctx, j->slot, j->planes, j->strides, &token);
    if (!rc) rc = b200_poll_errors(G.ctx);
    if (rc) snprintf(msg, msg_n, "%s", b200_last_error(G.ctx));
    if (j->rb >= 0) {
        pthread_mutex_lock(&G.mu);
        if (G.rb[j->rb].seq == j->rb_seq && G.rb[j->rb].state == 1) {      /* else: the host buffer went to a newer picture meanwhile */
            G.rb[j->rb].token = token;
            G.rb[j->rb].state = rc ? 3 : 2;                       /* 2 issued, 3 failed: a waiter must not wait for it */
        }
        pthread_mutex_unlock(&G.mu);
    }
    return rc;
}

static void *submit_main(void *arg)
{
    shim_block_for((Instance *)arg);               /* G = the instance this thread was started for */
    pthread_mutex_lock(&G.mu);
    for (;;) {
        Job *j;
        while (!(j = G.jobq[G.turn % MAX_JOBS]) && !G.sub_stop) pthread_cond_wait(&G.cv_sub, &G.mu);
        if (!j) break;
        G.jobq[G.turn % MAX_JOBS] = NULL;
        pthread_mutex_unlock(&G.mu);
        char msg[256] = "";
        const int rc = process_job(j, msg, sizeof(msg));
        pthread_mutex_lock(&G.mu);
        if (rc) latch_global(rc, msg);
        j->done = 1;
        G.turn++;
        pthread_cond_broadcast(&G.cv);
    }
    pthread_mutex_unlock(&G.mu);
    return NULL;
}

/* the process ends (exit() or return from main) while work lists may still be queued: let them through -- record-only runs
 * (B200_SHIM_DUMP) write their files on the submission thread */
static void drain_at_exit(void)
{
    uint64_t tot[8] = { 0 };
    for (int i = 0; i < MAX_INST; i++) {
        Instance *I = &g_insts[i];
        pthread_mutex_lock(&I->mu);
        while (I->sub_running && I->turn != I->next_ticket && !I->err_code) pthread_cond_wait(&I->cv, &I->mu);
        pthread_mutex_unlock(&I->mu);
        const uint64_t v[8] = { I->n_pictures, I->h2d_bytes, I->d2h_bytes, I->ns_ctx, I->ns_rec, I->n_pool, I->bytes_pool, I->ns_pool };
        for (int k = 0; k < 8; k++) tot[k] += v[k];
    }
    if (getenv("B200_SHIM_REPORT"))
        fprintf(stderr, "b200 shim: pictures %llu h2d_bytes %llu d2h_bytes %llu\nb200 shim start-up: device context %.0f ms, recorders %.0f ms, pinned frame buffers %llu x (%.0f MB total) %.0f ms\n",
                (unsigned long long)tot[0], (unsigned long long)tot[1], (unsigned long long)tot[2],
                tot[3] * 1e-6, tot[4] * 1e-6, (unsigned long long)tot[5], tot[6] * 1e-6, tot[7] * 1e-6);
}

static void register_drain_at_exit(void) { atexit(drain_at_exit); }
static void enqueue(Job *j)                        /* j->ticket is this thread's ticket */
{
    pthread_mutex_lock(&G.mu);
    if (!G.sub_running) {
        static pthread_once_t registered = PTHREAD_ONCE_INIT;
        G.sub_stop = 0;
        if (pthread_create(&G.sub_thread, NULL, submit_main, &G)) latch_global(B200_ENOMEM, "cannot start the submission thread");
        else { G.sub_running = 1; pthread_once(&registered, register_drain_at_exit); }
    }
    j->pending = 1; j->done = 0;
    if (!G.sub_running) { j->done = 1; G.turn++; pthread_cond_broadcast(&G.cv); }      /* nobody will run it: keep the tickets moving */
    else { G.jobq[j->ticket % MAX_JOBS] = j; pthread_cond_signal(&G.cv_sub); }
    pthread_mutex_unlock(&G.mu);
}

/* the job's memory (recorder blob, Job itself) may be written again */
static void job_reclaim(Job *j)
{
    if (!j->pending) return;
    pthread_mutex_lock(&G.mu);
    while (!j->done) pthread_cond_wait(&G.cv, &G.mu);
    pthread_mutex_unlock(&G.mu);
    if (j->uploaded && G.ctx) b200_upload_wait(G.ctx, j->upload_token);
    j->pending = 0; j->uploaded = 0;
}

static void drain_queue(void)                      /* G.mu held: every ticket handed out so far has been through the submission thread */
{
    while (G.turn != G.next_ticket) pthread_cond_wait(&G.cv, &G.mu);
}

static int ensure_ctx(const HEVCContext *s)       /* called with G.mu held */
{
    const HEVCSPS *sps = s->sps;
    if (!G.env_read) { G.dump_dir = getenv("B200_SHIM_DUMP"); G.env_read = 1; }     /* once, under G.mu: read without it afterwards */
    if (!((G.ctx || (G.dump_dir && G.configured)) && G.cfg.width == sps->width && G.cfg.height == sps->height && G.cfg.bit_depth == sps->bit_depth &&
          G.cfg.chroma_format_idc == sps->chroma_format_idc && G.cfg.log2_ctb_size == (int)sps->log2_ctb_size)) {
        /* New geometry (a new SPS, hence an IRAP picture: nothing older is referenced any more).  With frame threads older pictures
         * may still be parsing on other threads against the old context, plane sizes and sample width: wait until their packets
         * have ended (they do not depend on this thread) and their work lists have gone through the submission thread, then switch. */
        while (G.in_flight > (g.counted ? 1 : 0)) pthread_cond_wait(&G.cv, &G.mu);      /* (this thread's own packet does not count) */
        drain_queue();
        G.gen = __atomic_add_fetch(&g_gen_counter, 1, __ATOMIC_RELAXED);
        if (G.ctx) { b200_sync(G.ctx); b200_ctx_destroy(G.ctx); G.ctx = NULL; }
        for (int i = 0; i < MAX_RB; i++) G.rb[i].state = 0;
        memset(&G.cfg, 0, sizeof(G.cfg));
        const char *dev = getenv("B200_DEVICE");
        G.cfg.device = dev ? atoi(dev) : 0;
        G.cfg.width = sps->width; G.cfg.height = sps->height; G.cfg.chroma_format_idc = sps->chroma_format_idc;
        G.cfg.bit_depth = sps->bit_depth; G.cfg.log2_ctb_size = sps->log2_ctb_size;
        G.cfg.n_slots = 32;                /* == FF_ARRAY_ELEMS(s->DPB), hevc.h:1207 */
        G.cfg.n_arenas = 8;
        if (!G.dump_dir) {
            const uint64_t t0 = now_ns();
            int rc = b200_ctx_create(&G.cfg, &G.ctx);
            G.ns_ctx += now_ns() - t0;
            if (rc) { fail(rc, b200_last_error(NULL)); return rc; }
        }
        G.configured = 1;
        G.bd = sps->bit_depth; G.B = G.bd > 8 ? 2 : 1; G.cfi = sps->chroma_format_idc;
        for (int p = 0; p < 3; p++) b200_plane_dims(sps->width, sps->height, G.cfi, p, &G.pw[p], &G.ph[p]);
    }
    return 0;
}

/* this thread's ticket is spent without a picture (abandoned picture whose frame is gone, or a failure before the hand-over) */
static void rb_cancel(void)                        /* no pixels will come for the announced read-back: release whoever waits for it */
{
    if (g.rb_at < 0) return;
    pthread_mutex_lock(&G.mu);
    if (G.rb[g.rb_at].seq == g.rb_seq && G.rb[g.rb_at].state == 1) { G.rb[g.rb_at].state = 3; pthread_cond_broadcast(&G.cv); }
    pthread_mutex_unlock(&G.mu);
    g.rb_at = -1;
}
static void ticket_skip(void)
{
    rb_cancel();
    Job *skip = &g.jobs[2];                        /* heap, like the other two: the submission thread may outlive this thread */
    job_reclaim(skip);
    memset(skip, 0, sizeof(*skip));
    skip->ticket = g.ticket; skip->kind = JOB_SKIP; skip->rb = -1;
    enqueue(skip);
}

static void deactivate(void)                       /* the picture is no longer open for worker threads */
{
    pthread_mutex_lock(&G.mu);
    g.in_frame = 0;
    for (int i = 0; i < G.n_active; i++)
        if (G.active[i] == &g) { G.active[i] = G.active[--G.n_active]; break; }
    pthread_mutex_unlock(&G.mu);
}

static void finish_abandoned(HEVCContext *s);
static void picture_flags(HEVCContext *s);
static int rb_insert(const uint8_t *data0, size_t luma_bytes);

int b200_frame_begin(HEVCContext *s)
{
    if (use_instance(s)) return g.err;
    /* a failure of one picture (unsupported tool, out of memory, a work list the device rejected) must not disable the decoder for
     * the rest of the process: a random-access point starts afresh.  CUDA errors are sticky and stay latched. */
    if (g.err && g.err != B200_ECUDA && IS_IRAP(s) && g.in_frame != 1) {
        pthread_mutex_lock(&G.mu);
        if (G.err_code != B200_ECUDA) G.err_code = 0;
        pthread_mutex_unlock(&G.mu);
        g.err = 0;
    }
    if (g.err) return g.err;
    if (g.in_frame == 1) finish_abandoned(s);                  /* previous picture of this thread was abandoned */
    if (g.err || global_error()) return g.err;
    g.in_frame = 0;
    g.rb_at = -1;
    picture_flags(s);
    /* cross-component prediction (4:4:4): host arithmetic between two table calls, undone and redone on the device (rec_cross_component) */
    g.s = s; g.lc = NULL; g.last_y.log2 = 0;
    g.ccp = s->sps->chroma_array_type == 3 && s->pps->cross_component_prediction_enabled_flag;
    /* (a caller that drives the tables without the decoder's own state -- oracle/replay_ref.c -- has no QP map: its filter calls are recorded) */
    g.dbd = ((s->pps->tiles_enabled_flag && s->threads_number != 1) || !s->qp_y_tab || !s->deblock) ? 0 : dbd_mode();
    /* the other of this thread's two recorders; its previous picture (two pictures back) has left host memory by now */
    g.cur ^= 1;
    if (g.jobs) job_reclaim(&g.jobs[g.cur]);
    pthread_mutex_lock(&G.mu);
    int erc = ensure_ctx(s);
    if (!erc && (erc = thread_recorder(g.cur))) fail(erc, "b200_rec_create failed");
    if (!erc) {
        g.ticket = G.next_ticket++;
        if (!g.counted) { G.in_flight++; g.counted = 1; }      /* once per packet, however many pictures it starts */
    }
    pthread_mutex_unlock(&G.mu);
    if (erc) return g.err;
    g.n_reg = 0;
    for (int i = 0; i < 32; i++) {
        AVFrame *f = s->DPB[i].frame;
        if (!f || !f->data[0]) continue;
        for (int p = 0; p < 3; p++) {
            RegPlane *r = &g.reg[g.n_reg++];
            r->base = f->data[p]; r->linesize = f->linesize[p]; r->slot = i; r->plane = p; r->w = G.pw[p]; r->h = G.ph[p];
            r->size = r->linesize * r->h; r->inv = row_inverse(r->linesize);
        }
    }
    g.cur_slot = (int)(s->ref - s->DPB);
    for (int p = 0; p < 3; p++) {
        g.cur_base[p] = s->frame->data[p]; g.cur_ls[p] = s->frame->linesize[p];
        g.cur_size[p] = g.cur_ls[p] * G.ph[p]; g.cur_inv[p] = row_inverse(g.cur_ls[p]);
    }
    g.n_ref = 0; g.pend_ptr = NULL; g.first_tmp = NULL; g.emu[0].buf = g.emu[1].buf = NULL;
    g.poc = s->poc; g.n_workers = 0;
    int rc = b200_rec_begin(g.rec, g.cur_slot, s->poc);
    if (rc) { fail(rc, "b200_rec_begin failed"); ticket_skip(); return rc; }
    pthread_mutex_lock(&G.mu);
    g.frame_seq++;
    g.in_frame = 1;
    if (G.n_active < MAX_ACTIVE) G.active[G.n_active++] = &g;
    /* announce the read-back NOW: the frame may be picked for output (bumping, by the thread of a later picture) while this
     * thread is still parsing it, and whoever hands it to the application must wait for pixels that are not even queued yet */
    g.rb_at = -1;
    if (!G.dump_dir && s->frame->data[0]) { g.rb_at = rb_insert(s->frame->data[0], (size_t)s->frame->linesize[0] * s->sps->height); if (g.rb_at >= 0) g.rb_seq = G.rb[g.rb_at].seq; }
    pthread_mutex_unlock(&G.mu);
    return 0;
}

/* a read-back into `data0`'s frame is on its way: remembered until the frame leaves the decoder (b200_output_wait).  G.mu held. */
static int rb_insert(const uint8_t *data0, size_t luma_bytes)
{
    int at = -1, oldest = -1;
    for (int i = 0; i < MAX_RB; i++) {
        if (G.rb[i].state && G.rb[i].data0 == data0) { at = i; break; }       /* the buffer was recycled without having been output */
        if (!G.rb[i].state) { if (at < 0) at = i; }
        else if (G.rb[i].state >= 2 && (oldest < 0 || (int)(G.rb[i].seq - G.rb[oldest].seq) < 0)) oldest = i;
    }
    if (at < 0) at = oldest;                       /* table full of pictures nobody asked for: forget the oldest one */
    if (at < 0) return -1;
    G.rb[at].data0 = data0; G.rb[at].end = data0 + luma_bytes; G.rb[at].state = 1; G.rb[at].seq = G.rb_seq++; G.rb[at].token = 0;
    return at;
}

static int frame_end_of(HEVCContext *s, HEVCFrame *ref)
{
    if (g.in_frame != 1) return g.err ? g.err : B200_ESTATE;
    deactivate();                                   /* all execute2 jobs of the picture have returned (hevc.c:3087) */
    int mrc = b200_rec_set_refs(g.rec, g.ref_slot, g.n_ref);
    for (int i = 0; i < g.n_workers; i++) {         /* fold the slice / WPP workers' lists into this recorder */
        ShimThread *w = g.workers[i];
        if (w->err) { fail(w->err, w->errmsg); w->err = 0; }
        if (!mrc) mrc = b200_rec_set_refs(w->rec, w->ref_slot, w->n_ref);
        if (!mrc) mrc = b200_rec_merge(g.rec, w->rec);
        g.n_tu += w->n_tu; g.n_intra += w->n_intra; g.n_pu += w->n_pu; g.n_dbk += w->n_dbk; g.n_sao += w->n_sao;
        w->in_frame = 0;
    }
    if (mrc) fail(mrc, "merging the worker threads' work lists failed");
    if (!g.err && g.pic_cip && ref && ref->tab_mvf) {
        /* the device applies the constrained-intra rules itself (hevcpred_template.c:116-249): hand it the PU types */
        const int pw = s->sps->min_pu_width, ph = s->sps->min_pu_height;
        uint8_t *map = malloc((size_t)pw * ph);
        if (!map) fail(B200_ENOMEM, "constrained_intra_pred map");
        else {
            for (int i = 0; i < pw * ph; i++) map[i] = ref->tab_mvf[i].pred_flag == PF_INTRA;
            int crc = b200_rec_set_cip(g.rec, s->sps->log2_min_pu_size, pw, ph, map);
            if (crc) fail(crc, "b200_rec_set_cip failed");
            free(map);
        }
    }
    if (!g.err && g.pic_tqb && s->is_pcm) {
        /* restore_tqb_pixels (hevc_filter.c:163-193) is pixel work outside the tables: the device redoes it from is_pcm[] */
        int crc = b200_rec_set_tqb(g.rec, s->sps->log2_min_pu_size, s->sps->min_pu_width, s->sps->min_pu_height, s->is_pcm);
        if (crc) fail(crc, "b200_rec_set_tqb failed");
    }
    if (!g.err && g.dbd) {
        /* deblocking parameters on the device: the QP map, the per-CTB slice offsets and (PCM loop filter off / bypass) is_pcm */
        B200DbdInput in;
        memset(&in, 0, sizeof(in));
        in.log2_min_cb_size = s->sps->log2_min_cb_size; in.min_cb_width = s->sps->min_cb_width; in.min_cb_height = s->sps->min_cb_height; in.qp_y = s->qp_y_tab;
        in.log2_min_pu_size = s->sps->log2_min_pu_size; in.min_pu_width = s->sps->min_pu_width; in.min_pu_height = s->sps->min_pu_height;
        const int pcmf = (s->sps->pcm_enabled_flag && s->sps->pcm.loop_filter_disable_flag) || s->pps->transquant_bypass_enable_flag;
        in.is_pcm = pcmf ? s->is_pcm : NULL;
        in.ctb_offsets = (const int8_t *)s->deblock;
        in.cb_qp_offset = s->pps->cb_qp_offset; in.cr_qp_offset = s->pps->cr_qp_offset;
        int drc = sizeof(DBParams) == 2 ? b200_rec_set_dbd(g.rec, &in) : B200_ENOTSUP;
        if (drc) fail(drc, "b200_rec_set_dbd failed");
    }
    if (g.err) { ticket_skip(); return g.err; }
    if (getenv("B200_SHIM_STATS"))
        fprintf(stderr, "b200 picture %d: intra_pred %d transform_add %d mc %d deblock %d sao %d\n", g.frame_no, g.n_intra, g.n_tu, g.n_pu, g.n_dbk, g.n_sao);
    g.frame_no++; g.n_tu = g.n_intra = g.n_pu = g.n_dbk = g.n_sao = 0;
    const void *blob; uint64_t n;
    int rc = b200_rec_finish(g.rec, &blob, &n);
    if (rc) { fail(rc, "b200_rec_finish failed"); ticket_skip(); return rc; }
    /* hand the picture to the submission thread: it enters the device queue in decode order (ticket), whatever order the
     * frame threads finish parsing in, and this thread is free for its next packet */
    Job *j = &g.jobs[g.cur];
    j->ticket = g.ticket; j->kind = JOB_PICTURE; j->blob = blob; j->nbytes = n;
    j->n_fill = g.n_fill; memcpy(j->fill_slot, g.fill_slot, sizeof(j->fill_slot)); g.n_fill = 0;
    j->uploaded = 0; j->rb = -1;
    AVFrame *hf = ref ? ref->frame : NULL;
    if (!G.dump_dir && hf && hf->data[0] && hf->data[0] == g.cur_base[0] && g.rb_at >= 0) {    /* the read-back into the picture's host frame is part of the job */
        j->slot = g.cur_slot;
        for (int p = 0; p < 3; p++) { j->planes[p] = hf->data[p]; j->strides[p] = hf->linesize[p]; }
        j->rb = g.rb_at; j->rb_seq = g.rb_seq;
    } else rb_cancel();
    g.rb_at = -1;
    enqueue(j);
    return global_error();
}
static void picture_flags(HEVCContext *s)
{
    g.pic_cip = s->pps->constrained_intra_pred_flag;
    g.pic_tqb = s->sps->sao_enabled && (s->pps->transquant_bypass_enable_flag || (s->sps->pcm.loop_filter_disable_flag && s->sps->pcm_enabled_flag));
}
int b200_frame_end(HEVCContext *s)
{
    if (use_instance(s)) return g.err;
    picture_flags(s);                               /* the parameter sets of the picture that ends (at b200_frame_begin of the NEXT one they may have changed) */
    return frame_end_of(s, s->ref);
}

/* A picture that was begun but never ended (corrupt slice data).  It is finished with what was recorded -- the part the
 * reference has reconstructed as well -- and copied into its host frame, which the decoder will still output. */
static void finish_abandoned(HEVCContext *s)
{
    HEVCFrame *old = g.cur_slot >= 0 && g.cur_slot < 32 ? &s->DPB[g.cur_slot] : NULL;
    if (!old || !old->frame || !old->frame->data[0] || old->frame->data[0] != g.cur_base[0]) {      /* the frame is gone: nothing to show */
        deactivate(); ticket_skip();
        return;
    }
    frame_end_of(s, old);
}

/* hevc_refs.c:538-606 generate_missing_ref: a reference the stream does not contain is replaced by a grey picture the host
 * fills with memset; the device slot must hold the same.  Called while the RPS of the NEXT picture of this thread is set up
 * (before its b200_frame_begin), executed in decode order in front of that picture. */
int b200_frame_fill(HEVCContext *s, HEVCFrame *frame)
{
    if (use_instance(s)) return g.err;
    if (g.err) return g.err;
    const int slot = (int)(frame - s->DPB);
    if (slot < 0 || slot >= 32) { fail(B200_EINVAL, "generate_missing_ref: frame is not in the DPB"); return g.err; }
    if (g.n_fill == 16) { fail(B200_ENOTSUP, "more than 16 missing reference pictures"); return g.err; }
    g.fill_slot[g.n_fill++] = (uint8_t)slot;
    return 0;
}

/* The frame is about to leave the decoder (hevc_decode_frame hands it to its caller) or to be read on the host (SEI
 * checksum): wait until the device picture has landed in it.  Frames the shim knows nothing about return at once. */
int b200_output_wait(HEVCContext *s, AVFrame *frame)
{
    if (s && use_instance(s)) return g.err;
    if (!frame || !frame->data[0] || G.dump_dir) return 0;
    pthread_mutex_lock(&G.mu);
    int at = -1;
    for (int i = 0; i < MAX_RB; i++)                /* the frame's luma pointer lies inside the buffer (cropped frames: past its start) */
        if (G.rb[i].state && G.rb[i].data0 <= frame->data[0] && frame->data[0] < G.rb[i].end) { at = i; break; }
    if (at < 0) { pthread_mutex_unlock(&G.mu); return 0; }
    const unsigned seq = G.rb[at].seq;
    while (G.rb[at].state == 1 && G.rb[at].seq == seq && !G.err_code) pthread_cond_wait(&G.cv, &G.mu);
    const int st = G.rb[at].seq == seq ? G.rb[at].state : 0;
    const uint32_t token = G.rb[at].token;
    if (G.rb[at].seq == seq) G.rb[at].state = 0;
    B200Ctx *ctx = G.ctx;
    pthread_mutex_unlock(&G.mu);
    int rc = 0;
    if (st == 2 && ctx) rc = b200_readback_wait(ctx, token);
    if (rc) fail(rc, "waiting for the read-back of an output picture failed");
    return rc ? rc : global_error();
}

static int packet_end(HEVCContext *s, AVFrame *frame);
int b200_frame_readback(HEVCContext *s, AVFrame *frame)
{
    if (use_instance(s)) return g.err;
    const int rc = packet_end(s, frame);
    if (g.counted) {                                /* this thread's picture no longer needs the context it was begun with */
        pthread_mutex_lock(&G.mu);
        g.counted = 0;
        G.in_flight--;
        pthread_cond_broadcast(&G.cv);
        pthread_mutex_unlock(&G.mu);
    }
    return rc;
}
static int packet_end(HEVCContext *s, AVFrame *frame)
{
    if (!frame) {
        /* The packet ended without a complete picture.  If one was begun, it was abandoned (corrupt slice data: hls_slice_data came
         * back short of the picture, hevc.c:3444-3446, and decode_nal_unit swallowed the error).  It is finished here with what was
         * recorded -- the part the reference has reconstructed as well: the decoder may still output the frame, and the pictures
         * behind it in decode order wait for its ticket.  Even after an error the ticket must not be lost.
         * (Packets are access units: a picture never continues in the next packet.) */
        if (g.in_frame == 1) {
            if (g.err || !s->ref) { deactivate(); ticket_skip(); }
            else {
                const int rc = b200_frame_end(s);
                if (rc) return rc;
                frame = s->ref->frame;
            }
        }
        if (!frame) return g.err;
    }
    if (g.err) return g.err;
    /* the read-back was issued with the picture; only a decoder that reads the pixels itself (SEI checksum, hevc.c:4146) waits here */
    if (s->decode_checksum_sei) return b200_output_wait(s, frame);
    return global_error();
}

/* reference pictures that exist only on the host (e.g. produced before the hook was active) */
int b200_frame_upload_ref(HEVCContext *s, AVFrame *frame)
{
    if (use_instance(s)) return g.err;
    pthread_mutex_lock(&G.mu);
    int rc = ensure_ctx(s);
    if (!rc && !G.dump_dir) {
        drain_queue();                               /* the submission thread is idle and stays so while G.mu is held */
        int slot = -1;
        for (int i = 0; i < 32; i++) if (s->DPB[i].frame && s->DPB[i].frame->data[0] == frame->data[0]) slot = i;
        if (slot < 0) { fail(B200_EINVAL, "upload of a frame that is not in the DPB"); rc = g.err; }
        else {
            const void *planes[3] = { frame->data[0], frame->data[1], frame->data[2] };
            int64_t strides[3] = { frame->linesize[0], frame->linesize[1], frame->linesize[2] };
            rc = b200_slot_upload(G.ctx, slot, planes, strides);
            if (!rc) rc = b200_sync(G.ctx);
            if (rc) fail(rc, b200_last_error(G.ctx));
        }
    }
    pthread_mutex_unlock(&G.mu);
    return rc ? g.err : 0;
}

/* ---- pinned host frames ------------------------------------------------------------------------------------------
 * Allocator for the decoder's frame pool (libavcodec/utils.c:558-561 passes av_buffer_allocz): the picture planes live in
 * page-locked memory, so the read-back of a picture is one asynchronous DMA at full PCIe rate instead of a staged,
 * synchronous copy.  Falls back to the stock allocator without a device.  libavutil is reached through dlsym: the shim
 * must load on its own (tests, tools) without the decoder library. */
typedef struct AVBufferRef *(*av_buffer_create_fn)(uint8_t *, int, void (*)(void *, uint8_t *), void *, int);
typedef struct AVBufferRef *(*av_buffer_allocz_fn)(int);
static void frame_buffer_free(void *opaque, uint8_t *data) { (void)opaque; b200_host_free(data); }
static struct { av_buffer_create_fn create; av_buffer_allocz_fn allocz; int use_pinned; } g_pool_fn;
static pthread_once_t g_pool_fn_once = PTHREAD_ONCE_INIT;
static void pool_fn_lookup(void)                   /* once: every frame thread's pool calls the allocator */
{
    g_pool_fn.create = (av_buffer_create_fn)dlsym(RTLD_DEFAULT, "av_buffer_create");
    g_pool_fn.allocz = (av_buffer_allocz_fn)dlsym(RTLD_DEFAULT, "av_buffer_allocz");
    g_pool_fn.use_pinned = !getenv("B200_SHIM_DUMP") && !(getenv("B200_PINNED_FRAMES") && !atoi(getenv("B200_PINNED_FRAMES")));
}
struct AVBufferRef *b200_frame_buffer_alloc(int size)
{
    pthread_once(&g_pool_fn_once, pool_fn_lookup);
    const av_buffer_create_fn create = g_pool_fn.create; const av_buffer_allocz_fn allocz = g_pool_fn.allocz;
    if (!create || !allocz) return NULL;
    const int use_pinned = g_pool_fn.use_pinned;
    const uint64_t t0 = now_ns();
    uint8_t *p = use_pinned && size > 0 ? b200_host_alloc((uint64_t)size) : NULL;
    if (!p) return allocz(size);
    memset(p, 0, (size_t)size);
    __atomic_fetch_add(&G.ns_pool, now_ns() - t0, __ATOMIC_RELAXED); __atomic_fetch_add(&G.n_pool, 1, __ATOMIC_RELAXED); __atomic_fetch_add(&G.bytes_pool, (uint64_t)size, __ATOMIC_RELAXED);
    struct AVBufferRef *r = create(p, size, frame_buffer_free, NULL, 0);
    if (!r) { b200_host_free(p); return NULL; }
    return r;
}

/* the device side of the calling thread's instance goes away: queue drained, submission thread joined, context destroyed.  G.mu held. */
static void instance_shutdown(void)
{
    if (G.sub_running) {
        drain_queue();
        G.sub_stop = 1;
        pthread_cond_broadcast(&G.cv_sub);
        pthread_mutex_unlock(&G.mu);
        pthread_join(G.sub_thread, NULL);
        pthread_mutex_lock(&G.mu);
        G.sub_running = 0;
    }
    if (G.ctx) { b200_sync(G.ctx); b200_ctx_destroy(G.ctx); }
    G.ctx = NULL; G.next_ticket = G.turn = 0; G.err_code = 0; G.configured = 0; G.n_active = 0; G.in_flight = 0;
    memset(&G.cfg, 0, sizeof(G.cfg));
    for (int i = 0; i < MAX_RB; i++) G.rb[i].state = 0;
}

/* hevc_decode_free (hevc.c:4187): the decoder is being closed.  With frame threads every copy and then the application's own
 * context come through here (pthread_frame.c:676, utils.c avcodec_close); the first call that still finds the instance gives the
 * device context, the submission thread and the entry back -- another decoder may open later in the same process. */
void b200_decoder_close(HEVCContext *s)
{
    const void *key = instance_key(s);
    Instance *I = NULL;
    pthread_mutex_lock(&g_insts_mu);
    for (int i = 0; i < MAX_INST && !I; i++) if (g_insts[i].key == key) I = &g_insts[i];
    pthread_mutex_unlock(&g_insts_mu);
    if (!I) return;
    ShimThread *prev = g_self;
    shim_block_for(I);
    pthread_mutex_lock(&G.mu);
    instance_shutdown();
    pthread_mutex_unlock(&G.mu);
    pthread_mutex_lock(&g_insts_mu);
    __atomic_store_n(&I->key, NULL, __ATOMIC_RELAXED);
    pthread_mutex_unlock(&g_insts_mu);
    if (prev) g_self = prev;
}

void b200_shim_close(void)                         /* every instance; for hosts that unload the library */
{
    ShimThread *prev = g_self;
    for (int i = 0; i < MAX_INST; i++) {
        shim_block_for(&g_insts[i]);
        pthread_mutex_lock(&G.mu);
        instance_shutdown();
        pthread_mutex_unlock(&G.mu);
        ShimThread *t = &g;
        for (int k = 0; k < 2; k++) if (t->recs[k]) { b200_rec_destroy(t->recs[k]); t->recs[k] = NULL; }      /* recorders of other threads die with the process */
        t->rec = NULL; t->in_frame = 0; t->err = 0; t->counted = 0;
        pthread_mutex_lock(&g_insts_mu);
        __atomic_store_n(&g_insts[i].key, NULL, __ATOMIC_RELAXED);
        pthread_mutex_unlock(&g_insts_mu);
    }
    if (prev) g_self = prev;
}
