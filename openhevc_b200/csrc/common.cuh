// common.cuh — shared device-side declarations for the B200 HEVC reconstruction kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/b200hevc_worklist.h"

struct PlaneDesc {
    uint8_t *base;   // device pointer to sample (0,0)
    int      pitch;  // bytes per row
    int      w, h;   // samples
};
struct FrameDesc {
    PlaneDesc p[3];
};
struct RefTable {
    uint64_t w[2];      // B200BlobHeader.ref_slot[16] packed little-endian (possibly overridden at execute time)
};

// HD: code that is also compiled for the host (with plain-C versions of the 16x2 instructions below) so that the CPU suite's
// warp emulator (tests/emul/warp/, test infrastructure) runs the very same source; the product never executes it on the host
#define HD __host__ __device__ __forceinline__
HD int clip3i(int v, int lo, int hi) { return v < lo ? lo : v > hi ? hi : v; }
HD int clip16i(int v) { return v < -32768 ? -32768 : v > 32767 ? 32767 : v; }
HD int imin(int a, int b) { return a < b ? a : b; }
HD int imax(int a, int b) { return a > b ? a : b; }

// ---- 16x2 SIMD integer helpers: the sm_90a (DPX) instructions (VIADD.16x2, VIADDMNMX.S16x2.RELU, VIMNMX.U16x2, PRMT, SHF)
// on the device, their definition in plain C on the host ----
HD uint32_t prmt32(uint32_t a, uint32_t b, uint32_t sel)          // prmt.b32, generic mode, selectors 0..7 only
{
#ifdef __CUDA_ARCH__
    uint32_t r;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(sel));
    return r;
#else
    const uint64_t src = ((uint64_t)b << 32) | a;
    uint32_t r = 0;
    for (int i = 0; i < 4; i++) r |= (uint32_t)((src >> (8 * ((sel >> (4 * i)) & 7))) & 0xff) << (8 * i);
    return r;
#endif
}
HD uint32_t vadd2(uint32_t a, uint32_t b)                         // per-half wrapping add
{
#ifdef __CUDA_ARCH__
    return __vadd2(a, b);
#else
    return ((a + b) & 0xffffu) | ((((a >> 16) + (b >> 16)) & 0xffffu) << 16);
#endif
}
HD uint32_t viaddmin_s16x2_relu(uint32_t a, uint32_t b, uint32_t c)   // per half: max(min(s16(a + b), s16(c)), 0)
{
#ifdef __CUDA_ARCH__
    return __viaddmin_s16x2_relu(a, b, c);
#else
    uint32_t r = 0;
    for (int h = 0; h < 2; h++) {
        const int s = (int16_t)(uint16_t)(((a >> (16 * h)) + (b >> (16 * h))) & 0xffff), m = (int16_t)(uint16_t)((c >> (16 * h)) & 0xffff);
        int v = s < m ? s : m;
        if (v < 0) v = 0;
        r |= (uint32_t)(v & 0xffff) << (16 * h);
    }
    return r;
#endif
}
HD uint32_t vminu2(uint32_t a, uint32_t b)                        // per-half unsigned minimum
{
#ifdef __CUDA_ARCH__
    return __vminu2(a, b);
#else
    const uint32_t lo = (a & 0xffff) < (b & 0xffff) ? (a & 0xffff) : (b & 0xffff), hi = (a >> 16) < (b >> 16) ? (a >> 16) : (b >> 16);
    return lo | (hi << 16);
#endif
}
HD uint4 LDG128(const void *p)                                     // read-only 16-byte load
{
#ifdef __CUDA_ARCH__
    return __ldg(reinterpret_cast<const uint4 *>(p));
#else
    return *reinterpret_cast<const uint4 *>(p);
#endif
}
HD uint32_t fsl16(uint32_t lo, uint32_t hi) { return (hi << 16) | (lo >> 16); }   // funnel shift left by 16 of hi:lo, upper word
HD uint32_t fsr16(uint32_t lo, uint32_t hi) { return (lo >> 16) | (hi << 16); }   // funnel shift right by 16 of hi:lo, lower word

// plane descriptor of a kernel-parameter FrameDesc by register selects: indexing the parameter struct with a runtime
// plane number would make the compiler copy it to local memory (an L2 round trip per access for a cold warp)
HD PlaneDesc plane_of(const FrameDesc &f, int plane)
{
    PlaneDesc d;
    d.base = plane == 0 ? f.p[0].base : plane == 1 ? f.p[1].base : f.p[2].base;
    d.pitch = plane == 0 ? f.p[0].pitch : plane == 1 ? f.p[1].pitch : f.p[2].pitch;
    d.w = plane == 0 ? f.p[0].w : plane == 1 ? f.p[1].w : f.p[2].w;
    d.h = plane == 0 ? f.p[0].h : plane == 1 ? f.p[1].h : f.p[2].h;
    return d;
}

template <typename PIX>
HD PIX *px_ptr(const PlaneDesc &p, int x, int y)
{
    return reinterpret_cast<PIX *>(p.base + (size_t)y * p.pitch) + x;
}

// launchers (kernels.cu) -- all asynchronous on `st`; return number of kernels launched
int launch_validate(cudaStream_t st, const uint8_t *blob_dev, const B200BlobHeader &h, const int pw[3], const int ph[3], unsigned long long arena_bytes, uint32_t *gate,
                    const B200McRec *mc_tiles = nullptr, uint32_t mc_count = 0, uint32_t mc_big = 0, uint32_t mc_tag = 0);
int launch_mc_expand(cudaStream_t st, const B200McRec *blocks, uint32_t n_blocks, B200McRec *tiles, const uint32_t count[5], uint32_t tag, uint32_t *gate);
int launch_mc(cudaStream_t st, const B200McRec *recs, int count, int n_big, const FrameDesc &cur, const FrameDesc *dpb_dev, const RefTable &rt, int bd, const uint32_t *gate);
int launch_residual(cudaStream_t st, const B200TuRec *const recs[4], const int counts[4], const int16_t *pool, int16_t *parked, const FrameDesc &cur, int bd, const uint32_t *gate);
int launch_ccp(cudaStream_t st, const B200CcpRec *recs, int count, int16_t *parked, const FrameDesc &cur, int bd, uint32_t *gate, unsigned long long arena_bytes);
int launch_intra(cudaStream_t st, const B200IntraRec *recs, int count, const int16_t *pool, const FrameDesc &cur, int bd,
                 uint2 *edges[3], const int edge_stride[3], uint32_t *counter, const uint32_t *cip_words, const B200CipHeader *cip_hdr, int cfi);
int launch_deblock(cudaStream_t st, const uint16_t *grid, const B200DbkLayout &L, const FrameDesc &cur, int bd);
// on-device derivation of the deblocking parameters (k_dbd.cuh): per-lane scratch, one allocation starting at `mot`
struct DbdMaps {
    uint4 *mot;             // per 4x4 luma unit: x = mv0 (x | y << 16), y = mv1, z = ref0 | ref1 << 8 | pred << 16 (0 intra, 1 one mv (in mv0), 3 two)
    uint8_t *cbf;           // per unit: a luma transform block with coefficients covers it
    uint8_t *bsv, *bsh;     // per unit: bs of its left / top edge
    uint16_t *grid;         // B200_SEC_DBK layout
    int uw, uh;             // units per row / rows
};

int launch_dbd(cudaStream_t st, const uint8_t *blob_dev, const B200BlobHeader &h, const B200DbdHeader &hd, const uint8_t *dbd, const DbdMaps &maps, size_t maps_bytes,
               const B200DbkLayout &L, const RefTable &rt, int ctb_w, uint32_t *gate, const uint16_t *check);
int launch_sao(cudaStream_t st, const B200SaoRec *grid, const FrameDesc &src, const FrameDesc &dst, int bd,
               int log2_ctb, int ctb_w, int ctb_h, int chroma_format_idc, const uint32_t *tqb_words, const B200CipHeader *tqb_hdr);
int set_intra_trace(unsigned long long *p);
int launch_fill(cudaStream_t st, const FrameDesc &f, int bd, int value);
