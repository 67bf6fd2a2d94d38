// k_yuv_rgb.cuh — the YUV -> planar RGB conversion of b200_yuv_to_rgb (k_yuv_rgb in kernels.cu).  Host + device: the
// coefficient derivation runs on the host, the per-sample arithmetic on the device, and tests/emul/ compiles the same code
// for the CPU.  tests/test_device_output_cpu.py restates both in numpy; the outputs are defined bit for bit:
//
//   coefficients (Q13), from Kr / Kb of the matrix, the range and W = the white level of the output
//   (255 for uint8, (1 << bit_depth) - 1 for float32):
//     limited range: sy = W / (219 << (bd - 8)),  sc = W / (224 << (bd - 8)),  yoff = 16 << (bd - 8)
//     full range:    sy = sc = W / ((1 << bd) - 1),                           yoff = 0
//     coff = 1 << (bd - 1),  Kg = 1 - Kr - Kb,  q(x) = floor(x * 8192 + 0.5)   (double precision)
//     cy = q(sy),  crv = q(2 (1 - Kr) sc),  cbu = q(2 (1 - Kb) sc),  cgu = q(2 Kb (1 - Kb) / Kg sc),  cgv = q(2 Kr (1 - Kr) / Kg sc)
//   per luma sample (nearest chroma: the chroma sample that covers it), int32:
//     l = cy (Y - yoff),  u = Cb - coff,  v = Cr - coff
//     R = clip((l + crv v + 4096) >> 13, 0, W),  G = clip((l - cgu u - cgv v + 4096) >> 13, 0, W),  B = clip((l + cbu u + 4096) >> 13, 0, W)
//   uint8 output: the clipped integer; float32 output: (float)integer * (float)(1.0 / W), one IEEE multiply.
#pragma once
#include <math.h>
#include "common.cuh"

struct YuvRgbCoef {
    int cy, crv, cgu, cgv, cbu;     // Q13
    int yoff, coff, maxv;           // maxv = W
    float scale;                    // float32 output: 1 / W (1 for uint8)
};

// matrix_coefficients of H.265 Table E.5: 1 (BT.709), 5 / 6 (BT.601), 9 (BT.2020 non-constant luminance); 0 = unsupported
static inline int yuv_rgb_coef(int matrix, int full_range, int bd, int out_float, YuvRgbCoef *k)
{
    double kr, kb;
    if (matrix == 1) { kr = 0.2126; kb = 0.0722; }
    else if (matrix == 5 || matrix == 6) { kr = 0.299; kb = 0.114; }
    else if (matrix == 9) { kr = 0.2627; kb = 0.0593; }
    else return 0;
    const double kg = 1.0 - kr - kb;
    const int W = out_float ? (1 << bd) - 1 : 255;
    const double sy = full_range ? (double)W / (double)((1 << bd) - 1) : (double)W / (double)(219 << (bd - 8));
    const double sc = full_range ? (double)W / (double)((1 << bd) - 1) : (double)W / (double)(224 << (bd - 8));
    auto q = [](double x) { return (int)floor(x * 8192.0 + 0.5); };
    k->cy = q(sy);
    k->crv = q(2.0 * (1.0 - kr) * sc);
    k->cbu = q(2.0 * (1.0 - kb) * sc);
    k->cgu = q(2.0 * kb * (1.0 - kb) / kg * sc);
    k->cgv = q(2.0 * kr * (1.0 - kr) / kg * sc);
    k->yoff = full_range ? 0 : 16 << (bd - 8);
    k->coff = 1 << (bd - 1);
    k->maxv = W;
    k->scale = out_float ? (float)(1.0 / (double)W) : 1.0f;
    return 1;
}

HD void yuv_rgb_px(const YuvRgbCoef &k, int Y, int Cb, int Cr, int (&o)[3])
{
    const int l = k.cy * (Y - k.yoff) + 4096, u = Cb - k.coff, v = Cr - k.coff;
    o[0] = clip3i((l + k.crv * v) >> 13, 0, k.maxv);
    o[1] = clip3i((l - k.cgu * u - k.cgv * v) >> 13, 0, k.maxv);
    o[2] = clip3i((l + k.cbu * u) >> 13, 0, k.maxv);
}

HD void yuv_rgb_store(uint8_t *d, int v, float) { *d = (uint8_t)v; }
HD void yuv_rgb_store(float *d, int v, float scale) { *d = (float)v * scale; }

struct YuvRgbJob {
    const uint8_t *src[3];          // Y, Cb, Cr in AVFrame layout
    long long pitch[3];             // bytes
    int x0, y0, w, h;               // crop window, luma samples
    int sx, sy;                     // chroma subsampling shifts
    int tx0, ty0;                   // first 2x2 tile (absolute luma coordinates / 2)
    void *dst;                      // R, G, B planes of h rows of w samples, contiguous
    YuvRgbCoef k;
};

// One thread: the 2x2 tile of luma samples at absolute (2 tx, 2 ty), those of them inside the crop window.  Tiles are aligned
// in picture coordinates, so a 4:2:0 tile has exactly one chroma sample whatever the crop offsets.
template <typename PIX, typename OUT>
HD void yuv_rgb_tile(const YuvRgbJob &j, int tx, int ty)
{
    OUT *dst = reinterpret_cast<OUT *>(j.dst);
    const size_t plane = (size_t)j.w * j.h;
    for (int dy = 0; dy < 2; dy++) {
        const int y = 2 * ty + dy;
        if (y < j.y0 || y >= j.y0 + j.h) continue;
        const PIX *ly = reinterpret_cast<const PIX *>(j.src[0] + (size_t)y * j.pitch[0]);
        const PIX *cb = reinterpret_cast<const PIX *>(j.src[1] + (size_t)(y >> j.sy) * j.pitch[1]);
        const PIX *cr = reinterpret_cast<const PIX *>(j.src[2] + (size_t)(y >> j.sy) * j.pitch[2]);
        for (int dx = 0; dx < 2; dx++) {
            const int x = 2 * tx + dx;
            if (x < j.x0 || x >= j.x0 + j.w) continue;
            int o[3];
            yuv_rgb_px(j.k, ly[x], cb[x >> j.sx], cr[x >> j.sx], o);
            const size_t at = (size_t)(y - j.y0) * j.w + (x - j.x0);
            yuv_rgb_store(dst + at, o[0], j.k.scale);
            yuv_rgb_store(dst + plane + at, o[1], j.k.scale);
            yuv_rgb_store(dst + 2 * plane + at, o[2], j.k.scale);
        }
    }
}
