// engine.cu — context, device-resident DPB, upload arenas and the per-frame stage pipeline
// behind the C ABI of include/b200hevc.h.
//
// Streams: `copy` carries the one pinned H2D upload per picture, `down` the read-backs, and
// pictures execute on `n_lanes` compute LANES (stream + private work picture, parked-residual
// pool, intra edge records).  Pictures are submitted in decode order and placed round-robin on the
// lanes; what orders them on the device is the data they touch, not the submission order:
// every DPB slot carries a "written" event and per-lane "read" events, a picture waits for the
// writers of its reference slots (RAW) and for the readers / previous writer of its own slot
// (WAR / WAW).  Pictures that do not depend on each other (the B pictures of one hierarchy
// level, an I picture and the tail of the previous GOP) therefore overlap, which hides the
// latency-bound intra wavefront (K3) behind the throughput-bound kernels of its neighbours.
// Arenas are multi-buffered: the upload of picture k+1 overlaps the kernels of picture k.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <stdarg.h>
#include <ctype.h>
#include <sched.h>
#include <unistd.h>
#include <sys/syscall.h>
#include <mutex>
#include <vector>
#include "../../include/b200hevc.h"
#include "common.cuh"
#include "k_yuv_rgb.cuh"

int launch_yuv_rgb(cudaStream_t st, const YuvRgbJob &j, int bd, int out_float);     // kernels.cu

#define MAX_SLOTS 64
#define MAX_ARENAS 16
#define MAX_LANES 16
#define RD_DOWN MAX_LANES            // reader index of the read-back stream
#define RD_EXT (MAX_LANES + 1)       // reader index of caller-owned streams (b200_slot_end_access)
#define RD_EXP (MAX_LANES + 2)       // reader index of the export stream (b200_slot_export_async)
#define N_RD (MAX_LANES + 3)
#define RB_RING 64

struct Arena {
    uint8_t *dev = nullptr;
    uint8_t *stage = nullptr;       // pinned staging for blobs that are not in pinned memory
    uint64_t stage_bytes = 0;
    B200CipHeader cip_hdr = {};     // host copy of the resident blob's CIP section header (constrained_intra_pred pictures)
    B200CipHeader tqb_hdr = {};     // ... and of its TQB section header (restore_tqb_pixels)
    B200DbdHeader dbd_hdr = {};     // ... and of its DBD section header (deblocking parameters derived on the device)
    B200BlobHeader hdr;             // host copy of the resident blob's header
    bool resident = false;
    cudaEvent_t ev_uploaded = nullptr;
    cudaEvent_t ev_done[MAX_LANES] = {};   // last execution of the resident blob on each lane
    uint32_t done_mask = 0;
};

struct Lane {
    cudaStream_t st = nullptr;
    uint8_t *work = nullptr;            // pre-SAO picture (reconstruct + deblock happen here when the picture has SAO)
    FrameDesc work_desc;
    uint2 *flags[3] = { nullptr, nullptr, nullptr };   // intra edge records, 16 B per 4x4 unit
    uint32_t *counter = nullptr;        // [0] K3 ticket, [1] validation gate of the picture in progress, [2] K3 time-out latch, [3] validation latch,
                                        // [6] tiles k_mc_expand wrote (kernels.cu)
    int16_t *parked = nullptr;          // residuals of intra TUs (K2 -> K3), indexed like the coefficient pool
    B200McRec *mc_tiles = nullptr;      // tile list k_mc_expand writes when the blob carries whole prediction blocks (B200BlobHeader.mc_tile_count)
    uint32_t mc_tag = 0;                // stamp of the tiles k_mc_expand wrote for the lane's latest such picture (24 bits, never 0)
    DbdMaps dbd = {};                   // scratch of the on-device deblocking derivation, allocated with the first picture that needs it
    size_t dbd_bytes = 0;
    cudaEvent_t tail = nullptr;         // end of the last picture of this lane
    bool used = false;
};

struct SlotState {
    cudaEvent_t done = nullptr;         // last write of the slot
    cudaEvent_t rd[N_RD] = {};          // last read per lane / read-back stream / external stream
    uint32_t readers = 0;               // which rd[] are pending since the last write
    int writer = -1;                    // lane of the last write (-1: none yet, -2: not a lane)
};

struct B200Ctx {
    B200Config cfg;
    int pw[3], ph[3], pitch[3];
    size_t plane_off[3], slot_bytes;
    uint8_t *dpb = nullptr;          // n_slots frames
    bool own_dpb = false;
    FrameDesc *dpb_desc_dev = nullptr;
    FrameDesc slot_desc[MAX_SLOTS];
    int flag_stride[3];
    Lane lane[MAX_LANES];
    int n_lanes = 1, next_lane = 0;
    SlotState slot[MAX_SLOTS];
    Arena arena[MAX_ARENAS];
    uint64_t arena_bytes = 0;
    uint64_t mc_tile_cap = 0;        // tiles a picture can expand to: the smallest blocks are 8x4 luma (32 samples) with their chroma
    int next_arena = 0;
    cudaStream_t st_copy = nullptr, st_compute = nullptr /* == lane[0].st */, st_down = nullptr;
    cudaEvent_t prof[B200_ST_COUNT + 1];
    bool profiling = false, prof_valid = false;
    uint64_t launches = 0;
    // read-backs whose completion other threads wait for (b200_readback_wait): a ring of events on the read-back stream
    cudaEvent_t rb_ev[RB_RING] = {};
    uint32_t rb_next = 0;
    // device-to-device exports (b200_slot_export_async): their own stream, so that they do not queue behind host read-backs
    cudaStream_t st_exp = nullptr;
    cudaEvent_t ex_ev[RB_RING] = {};
    uint32_t ex_next = 0;
    // device-side error latches mirrored in mapped host memory (one word per lane): readable without a synchronisation
    volatile uint32_t *err_host = nullptr;
    uint32_t *err_dev = nullptr;
    B200DbkLayout dbk;
    int ctb_w, ctb_h;
    char err[512];
    int err_code = 0;
    // B200_TRACE=<file>: timeline of the pictures as they really ran on the lanes (events at the stage boundaries of every
    // picture, written as CSV when the context is destroyed) -- the overlap between pictures is invisible to per-kernel tools
    struct TraceRec { cudaEvent_t ev[7]; int lane, arena, poc, n_ref; };
    std::vector<TraceRec> trace;
    const char *trace_path = nullptr;
};

static char g_create_err[512];
static std::mutex g_mu;

static int fail(B200Ctx *ctx, int code, const char *fmt, ...)
{
    char *dst = ctx ? ctx->err : g_create_err;
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(dst, 512, fmt, ap);
    va_end(ap);
    if (ctx && !ctx->err_code) ctx->err_code = code;
    return code;
}
#define CU(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return fail(ctx, B200_ECUDA, "%s: %s", #call, cudaGetErrorString(e_)); } while (0)

static void geometry(const B200Config *c, int pw[3], int ph[3], int pitch[3], size_t off[3], size_t *slot_bytes)
{
    const int B = c->bit_depth > 8 ? 2 : 1;
    size_t o = 0;
    for (int p = 0; p < 3; p++) {
        b200_plane_dims(c->width, c->height, c->chroma_format_idc, p, &pw[p], &ph[p]);
        pitch[p] = (pw[p] * B + 255) & ~255;
        off[p] = o;
        o += (size_t)pitch[p] * ph[p];
        o = (o + 1023) & ~(size_t)1023;
    }
    *slot_bytes = o;
}

extern "C" uint64_t b200_worst_blob_bytes(const B200Config *c);      // recorder.cpp: the one definition of the largest blob of a geometry

static bool config_ok(const B200Config *c)
{
    return c && c->width >= 16 && c->height >= 16 && c->width <= 16384 && c->height <= 16384 && !(c->width & 7) && !(c->height & 7) &&
           c->chroma_format_idc >= 1 && c->chroma_format_idc <= 3 && c->bit_depth >= 8 && c->bit_depth <= 12 &&
           c->log2_ctb_size >= 4 && c->log2_ctb_size <= 6 && c->n_slots >= 1 && c->n_slots <= MAX_SLOTS &&
           c->n_arenas >= 1 && c->n_arenas <= MAX_ARENAS;
}

extern "C" uint64_t b200_dpb_bytes(const B200Config *cfg)
{
    if (!config_ok(cfg)) return 0;
    int pw[3], ph[3], pitch[3];
    size_t off[3], sb;
    geometry(cfg, pw, ph, pitch, off, &sb);
    return (uint64_t)sb * cfg->n_slots;
}

extern "C" const char *b200_last_error(const B200Ctx *ctx) { return ctx ? ctx->err : g_create_err; }
extern "C" uint64_t b200_slot_bytes(const B200Ctx *ctx) { return ctx->slot_bytes; }
extern "C" void *b200_stream(const B200Ctx *ctx) { return ctx->st_compute; }
extern "C" uint64_t b200_launch_count(const B200Ctx *ctx) { return ctx->launches; }

extern "C" void *b200_slot_devptr(const B200Ctx *ctx, int slot, int plane, uint64_t *pitch_bytes)
{
    if (!ctx || slot < 0 || slot >= ctx->cfg.n_slots || plane < 0 || plane > 2) return nullptr;
    if (pitch_bytes) *pitch_bytes = ctx->pitch[plane];
    return ctx->slot_desc[slot].p[plane].base;
}

// Pinned staging memory on the NUMA node the GPU hangs off: on a two-socket host a buffer on the far node halves the
// PCIe rate both ways (every transfer crosses the socket interconnect).  Pages are placed at allocation time (the driver
// faults them in to pin them), so the calling thread is moved onto the GPU's node -- CPU affinity, plus a preferred-node
// memory policy where the container allows the syscall -- for the duration of the cudaHostAlloc only.  Best effort:
// any failure leaves the default placement.  B200_NUMA=0 disables it.
static int gpu_numa_node(int device, cpu_set_t *cpus)
{
    char bus[32] = { 0 }, path[128], buf[4096];
    if (cudaDeviceGetPCIBusId(bus, sizeof(bus), device) != cudaSuccess) { cudaGetLastError(); return -1; }
    for (char *c = bus; *c; c++) *c = (char)tolower(*c);
    snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bus);
    FILE *f = fopen(path, "r");
    int node = -1;
    if (f) { if (fscanf(f, "%d", &node) != 1) node = -1; fclose(f); }
    if (node < 0) return -1;
    snprintf(path, sizeof(path), "/sys/devices/system/node/node%d/cpulist", node);
    f = fopen(path, "r");
    if (!f) return -1;
    const bool ok = fgets(buf, sizeof(buf), f) != nullptr;
    fclose(f);
    if (!ok) return -1;
    CPU_ZERO(cpus);
    for (char *t = strtok(buf, ",\n"); t; t = strtok(nullptr, ",\n")) {       // "0-31,64-95"
        int a, b;
        const int n = sscanf(t, "%d-%d", &a, &b);
        if (n == 1) b = a;
        if (n >= 1) for (int c = a; c <= b && c < CPU_SETSIZE; c++) CPU_SET(c, cpus);
    }
    return node;
}

static cudaError_t host_alloc_near_gpu(void **p, size_t bytes)
{
    static const bool enabled = !getenv("B200_NUMA") || atoi(getenv("B200_NUMA"));
    int dev = 0;
    cpu_set_t local, saved;
    int node = -1;
    bool moved = false, policy = false;
    if (enabled && cudaGetDevice(&dev) == cudaSuccess && (node = gpu_numa_node(dev, &local)) >= 0 && node < 64) {
        if (sched_getaffinity(0, sizeof(saved), &saved) == 0) {
            cpu_set_t want;
            CPU_AND(&want, &local, &saved);                      // stay inside the cpuset the container was given
            if (CPU_COUNT(&want) > 0 && sched_setaffinity(0, sizeof(want), &want) == 0) moved = true;
        }
        unsigned long mask = 1ul << node;
        policy = syscall(SYS_set_mempolicy, 1 /* MPOL_PREFERRED */, &mask, 65ul) == 0;
    }
    const cudaError_t rc = cudaHostAlloc(p, bytes, cudaHostAllocDefault);
    if (policy) syscall(SYS_set_mempolicy, 0 /* MPOL_DEFAULT */, nullptr, 0ul);
    if (moved) sched_setaffinity(0, sizeof(saved), &saved);
    static const bool verbose = getenv("B200_VERBOSE") != nullptr;
    if (verbose) fprintf(stderr, "b200: pinned %zu bytes, GPU %d on NUMA node %d (affinity %s, mempolicy %s)\n", bytes, dev, node, moved ? "set" : "-", policy ? "set" : "-");
    return rc;
}

extern "C" void *b200_host_alloc(uint64_t bytes)
{
    void *p = nullptr;
    if (host_alloc_near_gpu(&p, bytes) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}
extern "C" void b200_host_free(void *p) { if (p) cudaFreeHost(p); }

extern "C" void b200_ctx_destroy(B200Ctx *ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->cfg.device);
    cudaDeviceSynchronize();
    if (ctx->trace_path && !ctx->trace.empty()) {
        FILE *f = fopen(ctx->trace_path, "w");
        if (f) {
            fprintf(f, "picture,lane,arena,poc,n_ref,start_us,mc_us,residual_us,intra_us,deblock_us,sao_us\n");
            for (size_t i = 0; i < ctx->trace.size(); i++) {
                const B200Ctx::TraceRec &t = ctx->trace[i];
                float t0 = 0, d[5] = { 0, 0, 0, 0, 0 };
                cudaEventElapsedTime(&t0, ctx->trace[0].ev[0], t.ev[0]);
                for (int k = 0; k < 5; k++) cudaEventElapsedTime(&d[k], t.ev[0], t.ev[k + 1]);
                fprintf(f, "%zu,%d,%d,%d,%d,%.1f,%.1f,%.1f,%.1f,%.1f,%.1f\n", i, t.lane, t.arena, t.poc, t.n_ref, 1e3 * t0, 1e3 * d[0], 1e3 * d[1], 1e3 * d[2], 1e3 * d[3], 1e3 * d[4]);
            }
            fclose(f);
        }
        cudaGetLastError();
    }
    for (auto &t : ctx->trace) for (int k = 0; k < 6; k++) if (t.ev[k]) cudaEventDestroy(t.ev[k]);
    for (int i = 0; i < MAX_ARENAS; i++) {
        if (ctx->arena[i].dev) cudaFree(ctx->arena[i].dev);
        if (ctx->arena[i].stage) cudaFreeHost(ctx->arena[i].stage);
        if (ctx->arena[i].ev_uploaded) cudaEventDestroy(ctx->arena[i].ev_uploaded);
        for (int l = 0; l < MAX_LANES; l++) if (ctx->arena[i].ev_done[l]) cudaEventDestroy(ctx->arena[i].ev_done[l]);
    }
    for (int i = 0; i < MAX_SLOTS; i++) {
        if (ctx->slot[i].done) cudaEventDestroy(ctx->slot[i].done);
        for (int l = 0; l < N_RD; l++) if (ctx->slot[i].rd[l]) cudaEventDestroy(ctx->slot[i].rd[l]);
    }
    for (int i = 0; i <= B200_ST_COUNT; i++) if (ctx->prof[i]) cudaEventDestroy(ctx->prof[i]);
    for (int i = 0; i < RB_RING; i++) if (ctx->rb_ev[i]) cudaEventDestroy(ctx->rb_ev[i]);
    for (int i = 0; i < RB_RING; i++) if (ctx->ex_ev[i]) cudaEventDestroy(ctx->ex_ev[i]);
    if (ctx->err_host) cudaFreeHost((void *)ctx->err_host);
    if (ctx->own_dpb && ctx->dpb) cudaFree(ctx->dpb);
    if (ctx->dpb_desc_dev) cudaFree(ctx->dpb_desc_dev);
    for (int l = 0; l < MAX_LANES; l++) {
        Lane &L = ctx->lane[l];
        if (L.work) cudaFree(L.work);
        for (int p = 0; p < 3; p++) if (L.flags[p]) cudaFree(L.flags[p]);
        if (L.counter) cudaFree(L.counter);
        if (L.parked) cudaFree(L.parked);
        if (L.dbd.mot) cudaFree(L.dbd.mot);
        if (L.mc_tiles) cudaFree(L.mc_tiles);
        if (L.tail) cudaEventDestroy(L.tail);
        if (L.st) cudaStreamDestroy(L.st);
    }
    if (ctx->st_copy) cudaStreamDestroy(ctx->st_copy);
    if (ctx->st_down) cudaStreamDestroy(ctx->st_down);
    if (ctx->st_exp) cudaStreamDestroy(ctx->st_exp);
    delete ctx;
}

static int ctx_init(B200Ctx *ctx)
{
    const B200Config &c = ctx->cfg;
    CU(cudaSetDevice(c.device));
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, c.device));
    if (prop.major != 9 || prop.minor != 0) return fail(ctx, B200_ENOTSUP, "device %d is sm_%d%d; this library carries sm_90a code only", c.device, prop.major, prop.minor);
    geometry(&c, ctx->pw, ctx->ph, ctx->pitch, ctx->plane_off, &ctx->slot_bytes);
    const uint64_t need = (uint64_t)ctx->slot_bytes * c.n_slots;
    if (c.ext_frame_mem) {
        if (c.ext_frame_bytes < need) return fail(ctx, B200_EINVAL, "ext_frame_bytes %llu < required %llu", (unsigned long long)c.ext_frame_bytes, (unsigned long long)need);
        if ((uintptr_t)c.ext_frame_mem & 255) return fail(ctx, B200_EINVAL, "ext_frame_mem must be 256-byte aligned");
        ctx->dpb = (uint8_t *)c.ext_frame_mem;
    } else {
        CU(cudaMalloc(&ctx->dpb, need));
        ctx->own_dpb = true;
        CU(cudaMemset(ctx->dpb, 0, need));
    }
    auto describe = [&](FrameDesc &fd, uint8_t *base) {
        for (int p = 0; p < 3; p++) {
            PlaneDesc &d = fd.p[p];
            d.base = base + ctx->plane_off[p]; d.pitch = ctx->pitch[p]; d.w = ctx->pw[p]; d.h = ctx->ph[p];
        }
    };
    for (int s = 0; s < c.n_slots; s++) describe(ctx->slot_desc[s], ctx->dpb + (size_t)s * ctx->slot_bytes);
    CU(cudaMalloc(&ctx->dpb_desc_dev, sizeof(FrameDesc) * c.n_slots));
    CU(cudaMemcpy(ctx->dpb_desc_dev, ctx->slot_desc, sizeof(FrameDesc) * c.n_slots, cudaMemcpyHostToDevice));
    ctx->arena_bytes = c.max_blob_bytes ? c.max_blob_bytes : b200_worst_blob_bytes(&c);
    ctx->arena_bytes = (ctx->arena_bytes + 4095) & ~(uint64_t)4095;
    ctx->mc_tile_cap = 3ull * ((uint64_t)ctx->pw[0] * ctx->ph[0] / 32) + 4096;
    ctx->n_lanes = c.n_lanes > 0 ? c.n_lanes : 8;
    if (const char *e = getenv("B200_LANES")) if (atoi(e) > 0) ctx->n_lanes = atoi(e);
    if (ctx->n_lanes > MAX_LANES) ctx->n_lanes = MAX_LANES;
    ctx->trace_path = getenv("B200_TRACE");
    if (ctx->trace_path && strstr(ctx->trace_path, "%d")) {           // one file per device when several ranks share the environment
        static char per_dev[MAX_LANES][512];
        snprintf(per_dev[c.device % MAX_LANES], 512, ctx->trace_path, c.device);
        ctx->trace_path = per_dev[c.device % MAX_LANES];
    }
    if (ctx->trace_path) ctx->trace.reserve(4096);      // TraceRec pointers stay valid while a picture is being submitted
    for (int p = 0; p < 3; p++) ctx->flag_stride[p] = (ctx->pw[p] + 3) / 4 + 1;
    {   // one error word per lane in mapped host memory: kernels store to it on their (rare) error paths, the host polls it
        void *eh = nullptr, *ed = nullptr;
        CU(cudaHostAlloc(&eh, 256, cudaHostAllocMapped));
        memset(eh, 0, 256);
        ctx->err_host = (volatile uint32_t *)eh;
        CU(cudaHostGetDevicePointer(&ed, eh, 0));
        ctx->err_dev = (uint32_t *)ed;
    }
    for (int i = 0; i < RB_RING; i++) CU(cudaEventCreateWithFlags(&ctx->rb_ev[i], cudaEventDisableTiming));
    for (int i = 0; i < RB_RING; i++) CU(cudaEventCreateWithFlags(&ctx->ex_ev[i], cudaEventDisableTiming));
    for (int l = 0; l < ctx->n_lanes; l++) {
        Lane &L = ctx->lane[l];
        CU(cudaStreamCreateWithFlags(&L.st, cudaStreamNonBlocking));
        CU(cudaMalloc(&L.work, ctx->slot_bytes));
        CU(cudaMemset(L.work, 0, ctx->slot_bytes));
        describe(L.work_desc, L.work);
        for (int p = 0; p < 3; p++) {
            const size_t n = (size_t)ctx->flag_stride[p] * ((ctx->ph[p] + 3) / 4 + 1);
            CU(cudaMalloc(&L.flags[p], n * 16));
            CU(cudaMemset(L.flags[p], 0, n * 16));
        }
        CU(cudaMalloc(&L.counter, 256));
        CU(cudaMemset(L.counter, 0, 256));
        {   // counter[4..5]: device address of this lane's mapped host error word
            const unsigned long long hp = (unsigned long long)(uintptr_t)(ctx->err_dev + l);
            CU(cudaMemcpy(L.counter + 4, &hp, sizeof(hp), cudaMemcpyHostToDevice));
        }
        CU(cudaMalloc(&L.parked, ctx->arena_bytes));
        CU(cudaEventCreateWithFlags(&L.tail, cudaEventDisableTiming));
    }
    ctx->st_compute = ctx->lane[0].st;
    CU(cudaStreamCreateWithFlags(&ctx->st_copy, cudaStreamNonBlocking));
    CU(cudaStreamCreateWithFlags(&ctx->st_down, cudaStreamNonBlocking));
    CU(cudaStreamCreateWithFlags(&ctx->st_exp, cudaStreamNonBlocking));
    for (int i = 0; i < c.n_arenas; i++) {
        CU(cudaMalloc(&ctx->arena[i].dev, ctx->arena_bytes));
        CU(cudaEventCreateWithFlags(&ctx->arena[i].ev_uploaded, cudaEventDisableTiming));
        for (int l = 0; l < ctx->n_lanes; l++) CU(cudaEventCreateWithFlags(&ctx->arena[i].ev_done[l], cudaEventDisableTiming));
    }
    for (int i = 0; i < c.n_slots; i++) {
        CU(cudaEventCreateWithFlags(&ctx->slot[i].done, cudaEventDisableTiming));
        for (int l = 0; l < N_RD; l++) if (l < ctx->n_lanes || l >= MAX_LANES) CU(cudaEventCreateWithFlags(&ctx->slot[i].rd[l], cudaEventDisableTiming));
    }
    for (int i = 0; i <= B200_ST_COUNT; i++) CU(cudaEventCreate(&ctx->prof[i]));
    b200_dbk_layout(c.width, c.height, c.chroma_format_idc, &ctx->dbk);
    ctx->ctb_w = (c.width + (1 << c.log2_ctb_size) - 1) >> c.log2_ctb_size;
    ctx->ctb_h = (c.height + (1 << c.log2_ctb_size) - 1) >> c.log2_ctb_size;
    return 0;
}

extern "C" int b200_ctx_create(const B200Config *cfg, B200Ctx **out)
{
    std::lock_guard<std::mutex> lk(g_mu);
    if (!out) return B200_EINVAL;
    *out = nullptr;
    if (!config_ok(cfg)) return fail(nullptr, B200_EINVAL, "bad B200Config (dims must be multiples of 8, depth 8..12, cfi 1..3)");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
        cudaGetLastError();
        return fail(nullptr, B200_ECUDA, "no CUDA device: libb200hevc has no CPU fallback");
    }
    if (cfg->device < 0 || cfg->device >= ndev) return fail(nullptr, B200_EINVAL, "device %d out of range (0..%d)", cfg->device, ndev - 1);
    B200Ctx *ctx = new B200Ctx();
    memset(ctx->prof, 0, sizeof(ctx->prof));
    ctx->err[0] = 0;
    ctx->cfg = *cfg;
    int rc = ctx_init(ctx);
    if (rc) {
        memcpy(g_create_err, ctx->err, sizeof(g_create_err));
        b200_ctx_destroy(ctx);
        return rc;
    }
    *out = ctx;
    return 0;
}

static int check_blob(B200Ctx *ctx, const B200BlobHeader *h, uint64_t nbytes)
{
    const B200Config &c = ctx->cfg;
    if (nbytes < sizeof(B200BlobHeader) || h->magic != B200_BLOB_MAGIC || h->version != B200_BLOB_VERSION)
        return fail(ctx, B200_EINVAL, "not a B200 work-list blob (magic/version)");
    if (h->total_bytes != nbytes || nbytes > ctx->arena_bytes) return fail(ctx, B200_EINVAL, "blob size %llu (header %u, arena %llu)", (unsigned long long)nbytes, h->total_bytes, (unsigned long long)ctx->arena_bytes);
    if (h->width != c.width || h->height != c.height || h->chroma_format_idc != c.chroma_format_idc || h->bit_depth != c.bit_depth || h->log2_ctb_size != c.log2_ctb_size)
        return fail(ctx, B200_EINVAL, "blob geometry does not match the context");
    if (h->cur_slot >= c.n_slots) return fail(ctx, B200_EINVAL, "cur_slot %d out of range", h->cur_slot);
    static const uint32_t esz[B200_SEC_COUNT] = { 2, 16, 16, 16, 16, 16, 32, 2, 16 };
    for (int s = 0; s < B200_SEC_COUNT; s++) {
        const uint64_t end = (uint64_t)h->sec[s].off + (uint64_t)h->sec[s].count * esz[s];
        if (h->sec[s].count && ((h->sec[s].off & 15) || end > nbytes)) return fail(ctx, B200_EINVAL, "section %d out of bounds", s);
    }
    if (h->cip.count || (h->flags & B200_FRAME_CIP)) {          // constrained_intra_pred: bitmap of the min-PUs
        const uint64_t end = (uint64_t)h->cip.off + 4ull * h->cip.count;
        if (!(h->flags & B200_FRAME_CIP) || h->cip.count < 4 || (h->cip.off & 15) || end > nbytes) return fail(ctx, B200_EINVAL, "CIP section out of bounds");
        const B200CipHeader *ch = (const B200CipHeader *)((const uint8_t *)h + h->cip.off);
        if (ch->log2_min_pu_size < 2 || ch->log2_min_pu_size > 5 || ch->min_pu_width != ((uint32_t)c.width >> ch->log2_min_pu_size) ||
            ch->min_pu_height != ((uint32_t)c.height >> ch->log2_min_pu_size) || h->cip.count < B200_CIP_WORDS(ch->min_pu_width, ch->min_pu_height))
            return fail(ctx, B200_EINVAL, "CIP section does not match the picture geometry");
    }
    if (h->tqb.count || (h->flags & B200_FRAME_TQB)) {          // restore_tqb_pixels: bitmap of the min-PUs
        const uint64_t end = (uint64_t)h->tqb.off + 4ull * h->tqb.count;
        if (!(h->flags & B200_FRAME_TQB) || h->tqb.count < 4 || (h->tqb.off & 15) || end > nbytes) return fail(ctx, B200_EINVAL, "TQB section out of bounds");
        const B200CipHeader *th = (const B200CipHeader *)((const uint8_t *)h + h->tqb.off);
        if (th->log2_min_pu_size < 2 || th->log2_min_pu_size > 5 || th->min_pu_width != ((uint32_t)c.width >> th->log2_min_pu_size) ||
            th->min_pu_height != ((uint32_t)c.height >> th->log2_min_pu_size) || h->tqb.count < B200_CIP_WORDS(th->min_pu_width, th->min_pu_height))
            return fail(ctx, B200_EINVAL, "TQB section does not match the picture geometry");
    }
    if (h->ccp.count || (h->flags & B200_FRAME_CCP)) {          // cross-component prediction records (validated record by record on the device)
        const uint64_t end = (uint64_t)h->ccp.off + (uint64_t)sizeof(B200CcpRec) * h->ccp.count;
        if (!(h->flags & B200_FRAME_CCP) || !h->ccp.count || (h->ccp.off & 15) || end > nbytes || c.chroma_format_idc != 3)
            return fail(ctx, B200_EINVAL, "CCP section out of bounds (or not a 4:4:4 picture)");
    }
    if (h->reserved_section.off || h->reserved_section.count) return fail(ctx, B200_EINVAL, "reserved header section is not zero");
    if (h->dbd.count) {                                          // deblocking parameters derived on the device: header + arrays inside the section
        const uint64_t sec_bytes = 4ull * h->dbd.count, end = (uint64_t)h->dbd.off + sec_bytes;
        if ((h->dbd.off & 15) || end > nbytes || sec_bytes < sizeof(B200DbdHeader)) return fail(ctx, B200_EINVAL, "DBD section out of bounds");
        const B200DbdHeader *dh = (const B200DbdHeader *)((const uint8_t *)h + h->dbd.off);
        const uint64_t nqp = (uint64_t)dh->min_cb_width * dh->min_cb_height, npcm = (dh->flags & B200_DBDF_PCM) ? (uint64_t)dh->min_pu_width * dh->min_pu_height : 0;
        if (dh->log2_min_cb_size < 3 || dh->log2_min_cb_size > 6 || dh->min_cb_width != ((uint32_t)c.width >> dh->log2_min_cb_size) || dh->min_cb_height != ((uint32_t)c.height >> dh->log2_min_cb_size) ||
            (npcm && (dh->log2_min_pu_size < 2 || dh->log2_min_pu_size > 5 || dh->min_pu_width != ((uint32_t)c.width >> dh->log2_min_pu_size) || dh->min_pu_height != ((uint32_t)c.height >> dh->log2_min_pu_size))) ||
            ((dh->off_leaf | dh->off_qp | dh->off_ctb | dh->off_pcm) & 3) || (uint64_t)dh->off_leaf + 4ull * dh->n_leaf > sec_bytes || (uint64_t)dh->off_qp + nqp > sec_bytes ||
            (uint64_t)dh->off_ctb + 2ull * ctx->ctb_w * ctx->ctb_h > sec_bytes || (uint64_t)dh->off_pcm + npcm > sec_bytes ||
            dh->cb_qp_offset < -12 || dh->cb_qp_offset > 12 || dh->cr_qp_offset < -12 || dh->cr_qp_offset > 12)
            return fail(ctx, B200_EINVAL, "DBD section does not match the picture geometry");
    }
    {   // prediction blocks split on the device: the tile list they expand to must fit the lane's buffer
        uint64_t tiles = 0;
        for (int k = 0; k < 5; k++) tiles += h->mc_tile_count[k];
        if (tiles && (tiles > ctx->mc_tile_cap || tiles < h->sec[B200_SEC_MC].count || h->mc_big_count))
            return fail(ctx, B200_EINVAL, "MC tile counts %llu do not fit (blocks %u, capacity %llu)", (unsigned long long)tiles, h->sec[B200_SEC_MC].count, (unsigned long long)ctx->mc_tile_cap);
    }
    if (h->mc_big_count > h->sec[B200_SEC_MC].count) return fail(ctx, B200_EINVAL, "mc_big_count %u > %u MC records", h->mc_big_count, h->sec[B200_SEC_MC].count);
    if (h->sec[B200_SEC_DBK].count && h->sec[B200_SEC_DBK].count != ctx->dbk.total) return fail(ctx, B200_EINVAL, "deblock grid size %u != %u", h->sec[B200_SEC_DBK].count, ctx->dbk.total);
    if (h->sec[B200_SEC_SAO].count && h->sec[B200_SEC_SAO].count != (uint32_t)(3 * ctx->ctb_w * ctx->ctb_h)) return fail(ctx, B200_EINVAL, "SAO grid size mismatch");
    return 0;
}

// ---- slot hazards.  All calls come from the (single) submitting thread, in decode order, so "the event as recorded so
// far" is exactly the set of earlier accesses.  `who`: lane index, RD_DOWN or RD_EXT. ----
static int slot_acquire(B200Ctx *ctx, int slot, cudaStream_t st, int who, bool write)
{
    SlotState &S = ctx->slot[slot];
    if (S.writer != -1 && S.writer != who) CU(cudaStreamWaitEvent(st, S.done, 0));        // RAW / WAW
    if (write)
        for (int l = 0; l < N_RD; l++)
            if ((S.readers & (1u << l)) && l != who) CU(cudaStreamWaitEvent(st, S.rd[l], 0));   // WAR
    return 0;
}
static int slot_release(B200Ctx *ctx, int slot, cudaStream_t st, int who, bool write)
{
    SlotState &S = ctx->slot[slot];
    if (write) { CU(cudaEventRecord(S.done, st)); S.readers = 0; S.writer = who < MAX_LANES ? who : -2; }
    else { CU(cudaEventRecord(S.rd[who], st)); S.readers |= 1u << who; }
    return 0;
}

extern "C" int b200_slot_begin_access(B200Ctx *ctx, int slot, void *stream, int write)
{
    if (!ctx || slot < 0 || slot >= ctx->cfg.n_slots) return B200_EINVAL;
    CU(cudaSetDevice(ctx->cfg.device));
    return slot_acquire(ctx, slot, (cudaStream_t)stream, RD_EXT, write != 0);
}
extern "C" int b200_slot_end_access(B200Ctx *ctx, int slot, void *stream, int write)
{
    if (!ctx || slot < 0 || slot >= ctx->cfg.n_slots) return B200_EINVAL;
    CU(cudaSetDevice(ctx->cfg.device));
    return slot_release(ctx, slot, (cudaStream_t)stream, RD_EXT, write != 0);
}

// b200_stream() (lane 0) waits for everything submitted so far on every lane: an event the caller records on it
// afterwards marks the completion of all pictures (timing, external consumers)
extern "C" int b200_join(B200Ctx *ctx)
{
    if (!ctx) return B200_EINVAL;
    CU(cudaSetDevice(ctx->cfg.device));
    for (int l = 1; l < ctx->n_lanes; l++)
        if (ctx->lane[l].used) CU(cudaStreamWaitEvent(ctx->lane[0].st, ctx->lane[l].tail, 0));
    return 0;
}

extern "C" int b200_frame_upload(B200Ctx *ctx, const void *blob, uint64_t nbytes, int arena)
{
    if (!ctx || !blob || arena < 0 || arena >= ctx->cfg.n_arenas) return B200_EINVAL;
    if (ctx->err_code) return ctx->err_code;
    const B200BlobHeader *h = (const B200BlobHeader *)blob;
    int rc = check_blob(ctx, h, nbytes);
    if (rc) { ctx->err_code = 0; return rc; }
    // every record is validated before it is used: on the device, in front of the picture's kernels (k_validate, a few
    // microseconds; errors surface from b200_sync like the other device-side errors)
    CU(cudaSetDevice(ctx->cfg.device));
    Arena &a = ctx->arena[arena];
    const void *src = blob;
    cudaPointerAttributes at;
    bool pinned = cudaPointerGetAttributes(&at, blob) == cudaSuccess && at.type == cudaMemoryTypeHost;
    cudaGetLastError();
    if (!pinned) {   // stage through pinned memory so the copy stays asynchronous w.r.t. compute
        if (a.resident) CU(cudaEventSynchronize(a.ev_uploaded));
        if (a.stage_bytes < nbytes) {                       // staging grows with the blobs it has seen (a worst-case blob is ~4x a typical one)
            if (a.stage) { cudaFreeHost(a.stage); a.stage = nullptr; a.stage_bytes = 0; }
            uint64_t want = (nbytes + (nbytes >> 2) + ((1u << 22) - 1)) & ~(uint64_t)((1u << 22) - 1);
            if (want > ctx->arena_bytes) want = ctx->arena_bytes;
            CU(host_alloc_near_gpu((void **)&a.stage, want));
            a.stage_bytes = want;
        }
        memcpy(a.stage, blob, nbytes);
        src = a.stage;
    }
    for (int l = 0; l < ctx->n_lanes; l++)          // every execution of the arena's previous blob has finished
        if (a.done_mask & (1u << l)) CU(cudaStreamWaitEvent(ctx->st_copy, a.ev_done[l], 0));
    a.done_mask = 0;
    CU(cudaMemcpyAsync(a.dev, src, nbytes, cudaMemcpyHostToDevice, ctx->st_copy));
    CU(cudaEventRecord(a.ev_uploaded, ctx->st_copy));
    a.hdr = *h;
    if (h->cip.count) a.cip_hdr = *(const B200CipHeader *)((const uint8_t *)blob + h->cip.off);
    if (h->tqb.count) a.tqb_hdr = *(const B200CipHeader *)((const uint8_t *)blob + h->tqb.off);
    if (h->dbd.count) a.dbd_hdr = *(const B200DbdHeader *)((const uint8_t *)blob + h->dbd.off);
    a.resident = true;
    return 0;
}

extern "C" int b200_frame_execute(B200Ctx *ctx, int arena) { return b200_frame_execute_ex(ctx, arena, -1, nullptr, 0); }

extern "C" int b200_frame_execute_ex(B200Ctx *ctx, int arena, int cur_slot, const uint8_t *ref_slots, int n_ref)
{
    if (!ctx || arena < 0 || arena >= ctx->cfg.n_arenas) return B200_EINVAL;
    if (ctx->err_code) return ctx->err_code;
    Arena &a = ctx->arena[arena];
    if (!a.resident) return fail(ctx, B200_ESTATE, "arena %d holds no blob", arena);
    CU(cudaSetDevice(ctx->cfg.device));
    B200BlobHeader h = a.hdr;
    if (cur_slot >= 0) {                       // same work list, different DPB placement (GOP-periodic streams)
        if (cur_slot >= ctx->cfg.n_slots) return fail(ctx, B200_EINVAL, "cur_slot override %d out of range", cur_slot);
        h.cur_slot = (uint8_t)cur_slot;
    }
    if (ref_slots) {
        if (n_ref < 0 || n_ref > 16) return fail(ctx, B200_EINVAL, "n_ref %d", n_ref);
        h.n_ref = (uint8_t)n_ref;
        memcpy(h.ref_slot, ref_slots, (size_t)n_ref);
    }
    RefTable rt;
    memset(&rt, 0, sizeof(rt));
    for (int i = 0; i < h.n_ref && i < 16; i++) {
        if (h.ref_slot[i] >= ctx->cfg.n_slots) return fail(ctx, B200_EINVAL, "reference table entry %d -> slot %d out of range", i, h.ref_slot[i]);
        rt.w[i >> 3] |= (uint64_t)h.ref_slot[i] << (8 * (i & 7));
    }
    if (h.sec[B200_SEC_MC].count && !h.n_ref) return fail(ctx, B200_EINVAL, "inter records without a reference table");
    // profiling runs serially on lane 0 (clean stage times)
    int li = 0;
    if (ctx->profiling) { int rc = b200_join(ctx); if (rc) return rc; }
    else {
        // Lane choice.  What orders pictures on the device is the data (slot events), never the lane, so the only job
        // here is to keep independent pictures out of each other's way: consecutive pictures go to consecutive lanes
        // (round-robin over the general lanes), which lets every picture start the moment its references are written.
        // B200_TRACE showed what a cleverer rule cost: preferring "an idle lane, else the lane of a reference" put runs
        // of 20-30 pictures on ONE lane (1.28 pictures in flight on average): the device is almost never
        // idle-free: with the submitting thread ahead of the device every lane has work queued, so the fall-back rule decided.
        // The last lane is kept for pictures without references: an I picture is one long latency-bound wavefront (K3)
        // that nothing earlier feeds, so it should start the moment it is submitted instead of queueing behind inter pictures.
        const int nl = ctx->n_lanes, n_gen = nl > 1 ? nl - 1 : 1;
        const bool intra_only = h.n_ref == 0;
        if (intra_only && nl > 1) li = nl - 1;
        else { li = ctx->next_lane % n_gen; ctx->next_lane = (li + 1) % n_gen; }
    }
    Lane &L = ctx->lane[li];
    cudaStream_t st = L.st;
    const int bd = ctx->cfg.bit_depth;
    const bool has_sao = h.sec[B200_SEC_SAO].count != 0;
    const FrameDesc &out = ctx->slot_desc[h.cur_slot];
    const FrameDesc &cur = has_sao ? L.work_desc : out;   // reconstruct + deblock here
    const bool pf = ctx->profiling;
    uint32_t ref_seen[(MAX_SLOTS + 31) / 32] = {};
    for (int i = 0; i < h.n_ref; i++) {
        const int r = h.ref_slot[i];
        if (r == h.cur_slot) return fail(ctx, B200_EINVAL, "reference table entry %d is the picture's own slot %d", i, r);
        if (ref_seen[r >> 5] & (1u << (r & 31))) continue;
        ref_seen[r >> 5] |= 1u << (r & 31);
        int rc = slot_acquire(ctx, r, st, li, false); if (rc) return rc;
    }
    { int rc = slot_acquire(ctx, h.cur_slot, st, li, true); if (rc) return rc; }
    CU(cudaStreamWaitEvent(st, a.ev_uploaded, 0));
    CU(cudaMemsetAsync(L.counter, 0, 2 * sizeof(uint32_t), st));          // K3 ticket + this picture's validation gate
    // whole prediction blocks in the list: cut them into tiles first (k_mc_expand); everything behind works on the tile list
    const B200McRec *mc_list = (const B200McRec *)(a.dev + h.sec[B200_SEC_MC].off);
    uint32_t mc_count = h.sec[B200_SEC_MC].count, mc_big = h.mc_big_count;
    {
        uint64_t tiles = 0;
        for (int k = 0; k < 5; k++) tiles += h.mc_tile_count[k];
        if (tiles) {
            const size_t bytes = ctx->mc_tile_cap * sizeof(B200McRec);
            if (!L.mc_tiles) CU(cudaMalloc(&L.mc_tiles, bytes));
            // a new stamp per picture; when the 24 bits run out (or on first use) no tile in the list may carry the next one
            if (!L.mc_tag || L.mc_tag == 0xffffffu) { CU(cudaMemsetAsync(L.mc_tiles, 0, bytes, st)); L.mc_tag = 0; }
            L.mc_tag++;
            ctx->launches += launch_mc_expand(st, mc_list, mc_count, L.mc_tiles, h.mc_tile_count, L.mc_tag, L.counter);
            mc_list = L.mc_tiles; mc_count = (uint32_t)tiles; mc_big = h.mc_tile_count[0];
        }
    }
    ctx->launches += launch_validate(st, a.dev, h, ctx->pw, ctx->ph, ctx->arena_bytes, L.counter, mc_list == L.mc_tiles ? mc_list : nullptr, mc_count, mc_big, L.mc_tag);
    B200Ctx::TraceRec *tr = nullptr;
    if (ctx->trace_path && ctx->trace.size() < 4096) {
        ctx->trace.emplace_back();
        tr = &ctx->trace.back();
        tr->lane = li; tr->arena = arena; tr->poc = h.poc; tr->n_ref = h.n_ref;
        for (int k = 0; k < 7; k++) tr->ev[k] = nullptr;
        for (int k = 0; k < 6; k++) CU(cudaEventCreate(&tr->ev[k]));
        CU(cudaEventRecord(tr->ev[0], st));
    }
    if (pf) CU(cudaEventRecord(ctx->prof[0], st));
    // K1 inter
    ctx->launches += launch_mc(st, mc_list, (int)mc_count, (int)mc_big, cur, ctx->dpb_desc_dev, rt, bd, L.counter);
    if (pf) CU(cudaEventRecord(ctx->prof[1], st));
    if (tr) CU(cudaEventRecord(tr->ev[1], st));
    // K2 residual
    const int16_t *pool = (const int16_t *)(a.dev + h.sec[B200_SEC_COEFF].off);
    const B200TuRec *tu[4]; int ntu[4];
    for (int s = 0; s < 4; s++) { tu[s] = (const B200TuRec *)(a.dev + h.sec[B200_SEC_TU4 + s].off); ntu[s] = (int)h.sec[B200_SEC_TU4 + s].count; }
    ctx->launches += launch_residual(st, tu, ntu, pool, L.parked, cur, bd, L.counter);
    if (h.flags & B200_FRAME_CCP)                       // 4:4:4 cross-component prediction: combine the parked luma / chroma residuals
        ctx->launches += launch_ccp(st, (const B200CcpRec *)(a.dev + h.ccp.off), (int)h.ccp.count, L.parked, cur, bd, L.counter, ctx->arena_bytes);
    if (pf) CU(cudaEventRecord(ctx->prof[2], st));
    if (tr) CU(cudaEventRecord(tr->ev[2], st));
    // K3 intra
    ctx->launches += launch_intra(st, (const B200IntraRec *)(a.dev + h.sec[B200_SEC_INTRA].off), (int)h.sec[B200_SEC_INTRA].count, L.parked, cur, bd,
                                  L.flags, ctx->flag_stride, L.counter,
                                  (h.flags & B200_FRAME_CIP) && h.cip.count ? (const uint32_t *)(a.dev + h.cip.off) : nullptr, &a.cip_hdr, ctx->cfg.chroma_format_idc);
    if (pf) CU(cudaEventRecord(ctx->prof[3], st));
    if (tr) CU(cudaEventRecord(tr->ev[3], st));
    // K4 deblock: the edge parameters come recorded from the reference's own filter calls (DBK grids) or are derived here from
    // the picture's motion, coded-block flags and QP map (DBD section, k_dbd.cuh); with both present the two are compared
    const uint16_t *grid = h.sec[B200_SEC_DBK].count ? (const uint16_t *)(a.dev + h.sec[B200_SEC_DBK].off) : nullptr;
    if (h.dbd.count) {
        if (!L.dbd.mot) {
            const size_t U = (size_t)(ctx->pw[0] / 4) * (ctx->ph[0] / 4);
            const size_t o_cbf = 16 * U, o_bsv = o_cbf + ((U + 15) & ~(size_t)15), o_bsh = o_bsv + ((U + 15) & ~(size_t)15), o_grid = o_bsh + ((U + 15) & ~(size_t)15);
            L.dbd_bytes = o_grid + 2 * (size_t)ctx->dbk.total;
            uint8_t *m = nullptr;
            CU(cudaMalloc(&m, L.dbd_bytes));
            L.dbd.mot = (uint4 *)m; L.dbd.cbf = m + o_cbf; L.dbd.bsv = m + o_bsv; L.dbd.bsh = m + o_bsh; L.dbd.grid = (uint16_t *)(m + o_grid);
            L.dbd.uw = ctx->pw[0] / 4; L.dbd.uh = ctx->ph[0] / 4;
        }
        ctx->launches += launch_dbd(st, a.dev, h, a.dbd_hdr, a.dev + h.dbd.off, L.dbd, L.dbd_bytes, ctx->dbk, rt, ctx->ctb_w, L.counter, grid);
        grid = L.dbd.grid;
    }
    if (grid)
        ctx->launches += launch_deblock(st, grid, ctx->dbk, cur, bd);
    if (pf) CU(cudaEventRecord(ctx->prof[4], st));
    if (tr) CU(cudaEventRecord(tr->ev[4], st));
    // K5 SAO
    if (has_sao)
        ctx->launches += launch_sao(st, (const B200SaoRec *)(a.dev + h.sec[B200_SEC_SAO].off), cur, out, bd, ctx->cfg.log2_ctb_size, ctx->ctb_w, ctx->ctb_h, ctx->cfg.chroma_format_idc,
                                    (h.flags & B200_FRAME_TQB) && h.tqb.count ? (const uint32_t *)(a.dev + h.tqb.off) : nullptr, &a.tqb_hdr);
    if (pf) { CU(cudaEventRecord(ctx->prof[5], st)); ctx->prof_valid = true; }
    if (tr) CU(cudaEventRecord(tr->ev[5], st));
    CU(cudaEventRecord(a.ev_done[li], st));
    a.done_mask |= 1u << li;
    { int rc = slot_release(ctx, h.cur_slot, st, li, true); if (rc) return rc; }
    memset(ref_seen, 0, sizeof(ref_seen));
    for (int i = 0; i < h.n_ref; i++) {
        const int r = h.ref_slot[i];
        if (ref_seen[r >> 5] & (1u << (r & 31))) continue;
        ref_seen[r >> 5] |= 1u << (r & 31);
        int rc = slot_release(ctx, r, st, li, false); if (rc) return rc;
    }
    CU(cudaEventRecord(L.tail, st));
    L.used = true;
    CU(cudaGetLastError());
    return 0;
}

extern "C" int b200_frame_submit_ex(B200Ctx *ctx, const void *blob, uint64_t nbytes, uint32_t *upload_token)
{
    if (!ctx) return B200_EINVAL;
    const int a = ctx->next_arena;
    int rc = b200_frame_upload(ctx, blob, nbytes, a);
    if (rc) return rc;
    ctx->next_arena = (a + 1) % ctx->cfg.n_arenas;
    if (upload_token) *upload_token = (uint32_t)a;
    return b200_frame_execute(ctx, a);
}
extern "C" int b200_frame_submit(B200Ctx *ctx, const void *blob, uint64_t nbytes) { return b200_frame_submit_ex(ctx, blob, nbytes, nullptr); }

// Safe from any thread: touches the arena's event handle only.  The copy stream is FIFO, so if the arena has been re-used
// since, the wait is for a later upload -- which implies this one.
extern "C" int b200_upload_wait(B200Ctx *ctx, uint32_t upload_token)
{
    if (!ctx || upload_token >= (uint32_t)ctx->cfg.n_arenas) return B200_EINVAL;
    cudaSetDevice(ctx->cfg.device);
    const cudaError_t e = cudaEventSynchronize(ctx->arena[upload_token].ev_uploaded);
    return e == cudaSuccess ? 0 : B200_ECUDA;
}

extern "C" int b200_slot_upload(B200Ctx *ctx, int slot, const void *const planes[3], const int64_t strides[3])
{
    if (!ctx || slot < 0 || slot >= ctx->cfg.n_slots || !planes || !strides) return B200_EINVAL;
    if (ctx->err_code) return ctx->err_code;
    CU(cudaSetDevice(ctx->cfg.device));
    const int B = ctx->cfg.bit_depth > 8 ? 2 : 1;
    { int rc = slot_acquire(ctx, slot, ctx->st_compute, 0, true); if (rc) return rc; }
    for (int p = 0; p < 3; p++)
        CU(cudaMemcpy2DAsync(ctx->slot_desc[slot].p[p].base, ctx->pitch[p], planes[p], (size_t)strides[p], (size_t)ctx->pw[p] * B, ctx->ph[p], cudaMemcpyHostToDevice, ctx->st_compute));
    return slot_release(ctx, slot, ctx->st_compute, 0, true);
}

extern "C" int b200_slot_readback(B200Ctx *ctx, int slot, void *const planes[3], const int64_t strides[3])
{
    if (!ctx || slot < 0 || slot >= ctx->cfg.n_slots || !planes || !strides) return B200_EINVAL;
    if (ctx->err_code) return ctx->err_code;
    CU(cudaSetDevice(ctx->cfg.device));
    const int B = ctx->cfg.bit_depth > 8 ? 2 : 1;
    { int rc = slot_acquire(ctx, slot, ctx->st_down, RD_DOWN, false); if (rc) return rc; }
    for (int p = 0; p < 3; p++) {
        if (strides[p] == ctx->pitch[p])     // contiguous on both sides: one linear copy
            CU(cudaMemcpyAsync(planes[p], ctx->slot_desc[slot].p[p].base, (size_t)ctx->pitch[p] * ctx->ph[p], cudaMemcpyDeviceToHost, ctx->st_down));
        else
            CU(cudaMemcpy2DAsync(planes[p], (size_t)strides[p], ctx->slot_desc[slot].p[p].base, ctx->pitch[p], (size_t)ctx->pw[p] * B, ctx->ph[p], cudaMemcpyDeviceToHost, ctx->st_down));
    }
    return slot_release(ctx, slot, ctx->st_down, RD_DOWN, false);
}

// read-back whose completion ANOTHER thread waits for (the decoder's output path): the token names an event of a ring on the
// read-back stream; b200_readback_wait may be called from any thread (it touches that event handle only; the stream is
// FIFO, so a recycled ring entry stands for a later read-back, which implies this one)
extern "C" int b200_slot_readback_async(B200Ctx *ctx, int slot, void *const planes[3], const int64_t strides[3], uint32_t *token)
{
    int rc = b200_slot_readback(ctx, slot, planes, strides);
    if (rc) return rc;
    const uint32_t i = ctx->rb_next;
    ctx->rb_next = (i + 1) % RB_RING;
    CU(cudaEventRecord(ctx->rb_ev[i], ctx->st_down));
    if (token) *token = i;
    return 0;
}
extern "C" int b200_readback_wait(B200Ctx *ctx, uint32_t token)
{
    if (!ctx || token >= RB_RING) return B200_EINVAL;
    cudaSetDevice(ctx->cfg.device);
    const cudaError_t e = cudaEventSynchronize(ctx->rb_ev[token]);
    return e == cudaSuccess ? 0 : B200_ECUDA;
}

// device-to-device copy of one slot (cropped) into caller memory: a reader of the slot on the export stream, completion named
// by a ring of events like the read-backs
extern "C" int b200_slot_export_async(B200Ctx *ctx, int slot, const B200Export *e, uint32_t *token)
{
    if (!ctx || slot < 0 || slot >= ctx->cfg.n_slots || !e) return B200_EINVAL;
    if (ctx->err_code) return ctx->err_code;
    const int sx = ctx->cfg.chroma_format_idc != 3, sy = ctx->cfg.chroma_format_idc == 1;
    int x = e->crop_x, y = e->crop_y, w = e->crop_w, h = e->crop_h;
    if (!w && !h) { x = 0; y = 0; w = ctx->cfg.width; h = ctx->cfg.height; }
    const int B = ctx->cfg.bit_depth > 8 ? 2 : 1;
    // argument errors are reported, not latched: the context stays usable
    int rc = 0;
    if (x < 0 || y < 0 || w <= 0 || h <= 0 || (int64_t)x + w > ctx->cfg.width || (int64_t)y + h > ctx->cfg.height || ((x | w) & sx) || ((y | h) & sy))
        rc = fail(ctx, B200_EINVAL, "export crop window %d,%d %dx%d does not fit the %dx%d picture / its chroma grid", x, y, w, h, ctx->cfg.width, ctx->cfg.height);
    for (int p = 0; p < 3 && !rc; p++) {
        const int64_t row = (int64_t)(w >> (p ? sx : 0)) * B;
        if (!e->planes[p]) rc = fail(ctx, B200_EINVAL, "export plane %d is NULL", p);
        else if (e->pitches[p] < row) rc = fail(ctx, B200_EINVAL, "export plane %d: pitch %lld < %lld bytes per row", p, (long long)e->pitches[p], (long long)row);
    }
    if (rc) { ctx->err_code = 0; return rc; }
    CU(cudaSetDevice(ctx->cfg.device));
    if (e->after_event && cudaStreamWaitEvent(ctx->st_exp, (cudaEvent_t)e->after_event, 0) != cudaSuccess) {
        cudaGetLastError();
        rc = fail(ctx, B200_EINVAL, "export: after_event is not a valid CUDA event of this device");
        ctx->err_code = 0;
        return rc;
    }
    if ((rc = slot_acquire(ctx, slot, ctx->st_exp, RD_EXP, false))) return rc;
    cudaError_t ce = cudaSuccess;
    for (int p = 0; p < 3 && ce == cudaSuccess; p++) {
        const int hs = p ? sx : 0, vs = p ? sy : 0;
        const PlaneDesc &d = ctx->slot_desc[slot].p[p];
        ce = cudaMemcpy2DAsync(e->planes[p], (size_t)e->pitches[p], d.base + (size_t)(y >> vs) * d.pitch + (size_t)(x >> hs) * B, d.pitch,
                               (size_t)(w >> hs) * B, (size_t)(h >> vs), cudaMemcpyDeviceToDevice, ctx->st_exp);
    }
    // the reader is published even when a copy failed to enqueue: a later writer of the slot must not skip what was queued
    if ((rc = slot_release(ctx, slot, ctx->st_exp, RD_EXP, false))) return rc;
    if (ce != cudaSuccess) return fail(ctx, B200_ECUDA, "export copy: %s", cudaGetErrorString(ce));
    const uint32_t i = ctx->ex_next;
    ctx->ex_next = (i + 1) % RB_RING;
    CU(cudaEventRecord(ctx->ex_ev[i], ctx->st_exp));
    if (token) *token = i;
    return 0;
}
extern "C" int b200_export_wait(B200Ctx *ctx, uint32_t token)
{
    if (!ctx || token >= RB_RING) return B200_EINVAL;
    cudaSetDevice(ctx->cfg.device);
    const cudaError_t e = cudaEventSynchronize(ctx->ex_ev[token]);
    return e == cudaSuccess ? 0 : B200_ECUDA;
}
extern "C" void *b200_export_event(B200Ctx *ctx, uint32_t token)
{
    return ctx && token < RB_RING ? (void *)ctx->ex_ev[token] : nullptr;
}

extern "C" int b200_yuv_to_rgb(const B200RgbArgs *a, void *stream)
{
    if (!a) return B200_EINVAL;
    YuvRgbJob j;
    if (a->chroma_format_idc < 1 || a->chroma_format_idc > 3 || a->bit_depth < 8 || a->bit_depth > 12 || (a->out_float != 0 && a->out_float != 1) ||
        !yuv_rgb_coef(a->matrix, a->full_range != 0, a->bit_depth, a->out_float, &j.k))
        return B200_ENOTSUP;
    j.sx = a->chroma_format_idc != 3; j.sy = a->chroma_format_idc == 1;
    j.x0 = a->crop_x; j.y0 = a->crop_y; j.w = a->crop_w; j.h = a->crop_h;
    if (!j.w && !j.h) { j.x0 = 0; j.y0 = 0; j.w = a->width; j.h = a->height; }
    if (a->width <= 0 || a->height <= 0 || j.x0 < 0 || j.y0 < 0 || j.w <= 0 || j.h <= 0 || (int64_t)j.x0 + j.w > a->width || (int64_t)j.y0 + j.h > a->height || !a->out)
        return B200_EINVAL;
    const int B = a->bit_depth > 8 ? 2 : 1;
    for (int p = 0; p < 3; p++) {
        const int pw = p ? (a->width + j.sx) >> j.sx : a->width;
        if (!a->planes[p] || a->pitches[p] < (int64_t)pw * B) return B200_EINVAL;
        j.src[p] = (const uint8_t *)a->planes[p];
        j.pitch[p] = a->pitches[p];
    }
    j.tx0 = j.x0 >> 1; j.ty0 = j.y0 >> 1;
    j.dst = a->out;
    // The library links its own (static) CUDA runtime, so this thread's last-error state holds errors of this library only,
    // never those of the caller's runtime (torch ...).  Every other b200_* call checks its CUDA calls as it makes them and
    // returns what failed, so an error still pending here was reported already.  Clear it, so that the check after the launch
    // reports the launch alone.
    cudaGetLastError();
    launch_yuv_rgb((cudaStream_t)stream, j, a->bit_depth, a->out_float);
    return cudaGetLastError() == cudaSuccess ? 0 : B200_ECUDA;
}

// Device-side error latches without a synchronisation: the kernels mirror them into mapped host memory (one word per lane)
extern "C" int b200_poll_errors(B200Ctx *ctx)
{
    if (!ctx) return B200_EINVAL;
    if (ctx->err_code) return ctx->err_code;
    for (int l = 0; l < ctx->n_lanes; l++) {
        const uint32_t v = ctx->err_host[l];
        if (!v) continue;
        ctx->err_host[l] = 0;
        if (v & 0x80000000u) return fail(ctx, B200_EINVAL, "intra work list is not in decode order (dependency wait timed out)");
        int rc = fail(ctx, B200_EINVAL, "work list rejected on the device: invalid record in section mask 0x%x (picture not executed)", v);
        ctx->err_code = 0;
        return rc;
    }
    return 0;
}

extern "C" int b200_host_register(void *p, uint64_t bytes)
{
    if (!p || !bytes) return B200_EINVAL;
    if (cudaHostRegister(p, bytes, cudaHostRegisterDefault) != cudaSuccess) { cudaGetLastError(); return B200_ECUDA; }
    return 0;
}
extern "C" int b200_host_unregister(void *p)
{
    if (!p) return B200_EINVAL;
    if (cudaHostUnregister(p) != cudaSuccess) { cudaGetLastError(); return B200_ECUDA; }
    return 0;
}

extern "C" int b200_slot_wait_readback(B200Ctx *ctx, int slot)
{
    if (!ctx || slot < 0 || slot >= ctx->cfg.n_slots) return B200_EINVAL;
    CU(cudaSetDevice(ctx->cfg.device));
    if (ctx->slot[slot].readers & (1u << RD_DOWN)) CU(cudaEventSynchronize(ctx->slot[slot].rd[RD_DOWN]));
    return ctx->err_code;
}

extern "C" int b200_slot_fill(B200Ctx *ctx, int slot, int value)
{
    if (!ctx || slot < 0 || slot >= ctx->cfg.n_slots) return B200_EINVAL;
    if (ctx->err_code) return ctx->err_code;
    CU(cudaSetDevice(ctx->cfg.device));
    { int rc = slot_acquire(ctx, slot, ctx->st_compute, 0, true); if (rc) return rc; }
    ctx->launches += launch_fill(ctx->st_compute, ctx->slot_desc[slot], ctx->cfg.bit_depth, value);
    CU(cudaGetLastError());
    return slot_release(ctx, slot, ctx->st_compute, 0, true);
}

extern "C" int b200_wait_uploads(B200Ctx *ctx)
{
    if (!ctx) return B200_EINVAL;
    CU(cudaSetDevice(ctx->cfg.device));
    CU(cudaStreamSynchronize(ctx->st_copy));
    return ctx->err_code;
}

extern "C" int b200_sync(B200Ctx *ctx)
{
    if (!ctx) return B200_EINVAL;
    CU(cudaSetDevice(ctx->cfg.device));
    CU(cudaStreamSynchronize(ctx->st_copy));
    for (int l = 0; l < ctx->n_lanes; l++) CU(cudaStreamSynchronize(ctx->lane[l].st));
    CU(cudaStreamSynchronize(ctx->st_down));
    CU(cudaStreamSynchronize(ctx->st_exp));
    for (int l = 0; l < ctx->n_lanes; l++) {
        if (!ctx->lane[l].used) continue;
        uint32_t st[4] = { 0, 0, 0, 0 };
        CU(cudaMemcpy(st, ctx->lane[l].counter, sizeof(st), cudaMemcpyDeviceToHost));
        if (st[2]) return fail(ctx, B200_EINVAL, "intra work list is not in decode order (dependency wait timed out)");
        if (st[3]) {                                     // k_validate closed the gate of a picture on this lane: it was not executed
            CU(cudaMemset(ctx->lane[l].counter + 3, 0, sizeof(uint32_t)));
            ctx->err_host[l] = 0;
            int rc = fail(ctx, B200_EINVAL, "work list rejected on the device: invalid record in section mask 0x%x (picture not executed)", st[3]);
            ctx->err_code = 0;                           // the context stays usable, like after a rejected upload
            return rc;
        }
    }
    return ctx->err_code;
}

// debug only (not part of include/b200hevc.h): device buffer of 8 x uint64 per intra record for in-kernel timestamps
extern "C" int b200_debug_set_intra_trace(void *dev_ptr) { return set_intra_trace((unsigned long long *)dev_ptr); }

extern "C" int b200_set_profiling(B200Ctx *ctx, int on)
{
    if (!ctx) return B200_EINVAL;
    ctx->profiling = on != 0;
    ctx->prof_valid = false;
    return 0;
}

extern "C" int b200_get_stage_ms(B200Ctx *ctx, float ms[B200_ST_COUNT])
{
    if (!ctx || !ms) return B200_EINVAL;
    if (!ctx->prof_valid) return fail(ctx, B200_ESTATE, "no profiled frame");
    CU(cudaSetDevice(ctx->cfg.device));
    CU(cudaEventSynchronize(ctx->prof[5]));
    for (int s = 0; s < 5; s++) CU(cudaEventElapsedTime(&ms[s], ctx->prof[s], ctx->prof[s + 1]));
    CU(cudaEventElapsedTime(&ms[B200_ST_TOTAL], ctx->prof[0], ctx->prof[5]));
    return 0;
}
