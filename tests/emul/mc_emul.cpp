// mc_emul.cpp — TEST INFRASTRUCTURE, part of libkernel_emul.so.  K1 on the CPU: emul_mc() hands host planes to the product's
// inter-prediction launcher (kernels.cu launch_mc) as compiled into libb200hevc_emul.so, where the kernel runs as
// warp-lockstep fibers with its own group-local barriers.  tests/test_kernel_emul_cpu.py compares the result with the oracle.
#include "common.cuh"
#include <vector>

// dpb_planes[slot * 3 + plane]: host planes of the reference pictures (same pitches as the current picture);
// ref_slot[i] = DPB slot of entry i of the picture's reference table (16 entries)
extern "C" int emul_mc(const B200McRec *recs, int count, int n_big, uint8_t *const cur_planes[3], uint8_t *const *dpb_planes, int n_slots, const int pitch[3],
                       int width, int height, int cfi, int bd, const uint8_t *ref_slot)
{
    auto describe = [&](FrameDesc &f, uint8_t *const planes[3]) {
        for (int p = 0; p < 3; p++) {
            const int hs = p && cfi != 3, vs = p && cfi == 1;
            f.p[p].base = planes[p]; f.p[p].pitch = pitch[p]; f.p[p].w = width >> hs; f.p[p].h = height >> vs;
        }
    };
    FrameDesc cur;
    describe(cur, cur_planes);
    std::vector<FrameDesc> dpb(n_slots);
    for (int s = 0; s < n_slots; s++) describe(dpb[s], dpb_planes + 3 * s);
    RefTable rt = { { 0, 0 } };
    for (int i = 0; i < 16; i++) rt.w[i >> 3] |= (uint64_t)ref_slot[i] << (8 * (i & 7));
    uint32_t gate[4] = { 0, 0, 0, 0 };                   // [1] != 0 would mean "work list rejected": the kernel then does nothing
    launch_mc(nullptr, recs, count, n_big, cur, dpb.data(), rt, bd, gate);
    return 0;
}
