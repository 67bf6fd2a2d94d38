#!/bin/bash
# TEST INFRASTRUCTURE — builds the reference decoder WITH the B200 hooks of INTEGRATION.md into
# oracle/_ref/libohevc_b200.so: the six files that receive a hook are copied to oracle/_ref/patched/ (git-ignored),
# the hook lines are inserted with sed, every other object is reused from the plain reference build.
# Needs /root/reference; on the GPU box the prebuilt library is used.
set -euo pipefail
REF=${REF:-/root/reference}
HERE=$(cd "$(dirname "$0")" && pwd)
OUT=$HERE/_ref
ROOT=$(dirname "$HERE")
if [ ! -d "$REF/libavcodec" ]; then echo "build_patched: $REF not present - keeping prebuilt"; exit 0; fi
[ -f "$OUT/libohevc_ref.so" ] || "$HERE/build_ref.sh"
P=$OUT/patched/libavcodec
mkdir -p "$P" "$OUT/obj_b200"
for f in hevc.c hevcdsp.c hevcpred.c videodsp.c hevc_refs.c hevc_filter.c utils.c; do cp "$REF/libavcodec/$f" "$P/$f"; done
inc='#include "b200hevc_tables.h"'
# table hooks: one more arch-init call, exactly where the x86 / arm ones are (hevcdsp.c:1326-1327, hevcpred.c:84, videodsp.c:57-58)
sed -i -e "0,/^#include/s//$inc\n#include/" \
       -e 's/^\(\s*\)if (ARCH_ARM) ff_hevcdsp_init_arm(hevcdsp, bit_depth);/&\n\1ff_hevcdsp_init_b200(hevcdsp, bit_depth);/' "$P/hevcdsp.c"
sed -i -e "0,/^#include/s//$inc\n#include/" \
       -e 's/^\(\s*\)if (ARCH_X86) ff_hevcpred_init_x86(hpc, bit_depth);/&\n\1ff_hevcpred_init_b200(hpc, bit_depth);/' "$P/hevcpred.c"
sed -i -e "0,/^#include/s//$inc\n#include/" \
       -e '/ff_videodsp_init_x86(ctx, bpc);/a\    ff_videodsp_init_b200(ctx, bpc);' "$P/videodsp.c"
# frame life cycle, worker jobs, decoder close (hevc.c:3271 / 3446 / 4141; 2764 / 2847 / 2931; 4193: the read-back hook sits right behind decode_nal_units, before its result is looked at)
sed -i -e "0,/^#include/s//$inc\n#include/" \
       -e 's/^\(\s*\)ff_thread_finish_setup(s->avctx);/\1if ((ret = b200_frame_begin(s)) < 0) goto fail;\n&/' \
       -e '/^\s*s->is_decoded = 1;/,/tiles_filters(s);/ s/^\(\s*\)tiles_filters(s);/&\n\1if ((ret = b200_frame_end(s)) < 0) goto fail;   \/* after the filters of tile threads *\//' \
       -e 's|^\(\s*\)ret    = decode_nal_units(s, avpkt->data, avpkt->size);|&\n\1b200_frame_readback(s, s->is_decoded \&\& s->ref ? s->ref->frame : NULL);   /* NULL: no complete picture came out of the packet */|' \
       -e 's|^\(\s*\)av_frame_move_ref(data, s->output_frame);|\1b200_output_wait(s, s->output_frame);   /* the picture leaves the decoder: its read-back has landed */\n&|' \
       -e 's/^\(\s*\)s = s1->sList\[self_id\];/\1b200_worker_begin(s1);   \/* execute2 job: this worker records for s1'"'"'s picture *\/\n&/' \
       -e 's/^\(\s*\)s = s->sList\[self_id\];/\1b200_worker_begin(s);\n&/' \
       -e '/^static int hls_decode_entry(AVCodecContext \*avctxt, void \*isFilterThread)/,/^}/ s/^\(\s*\)int ctb_addr_ts = .*;$/&\n\1b200_worker_begin(s);   \/* execute(): with slice threads this runs on a worker thread too *\//' \
       -e '/^static av_cold int hevc_decode_free/,/^}/ s/^\(\s*\)pic_arrays_free(s);/\1b200_decoder_close(s);   \/* the device side of this decoder goes away with it *\/\n&/' \
       -e '/^\s*ret = ff_hevc_output_frame(s, data, 1);/,/^\s*return ret;/ s|^\(\s*\)return ret;|&\n        if (ret > 0) b200_output_wait(s, data);|' "$P/hevc.c"
# the decoder's frame pool in pinned memory (utils.c:558-561 passes av_buffer_allocz)
sed -i -e "0,/^#include/s//$inc\n#include/" \
       -e '/^static int update_frame_pool/,/^}/ s/^\(\s*\)av_buffer_allocz);/\1b200_frame_buffer_alloc);/' "$P/utils.c"
# a reference picture the stream does not contain (hevc_refs.c:538-606 fills a grey frame on the host): the device slot gets the same fill
sed -i -e "0,/^#include/s//$inc\n#include/" \
       -e '/^static HEVCFrame \*generate_missing_ref/,/^}/ s/^    return frame;/    b200_frame_fill(s, frame);\n&/' "$P/hevc_refs.c"
# optional, performance only (B200_NO_COPY_GUARD=1 builds without it): sao_filter_CTB's CTB copies between the host frame and
# sao_frame feed nothing once the SAO tables record (hevc_filter.c:151-161)
# deblocking control on the device (SURVEY.md 8f N2): the two host functions that derive boundary strengths / tc / beta hand over
sed -i -e '/^void ff_hevc_deblocking_boundary_strengths(HEVCContext \*s, int x0, int y0,/,/^}/ s/^    int i, j, bs;/&\n    if (b200_bs_on_device(s, x0, y0, log2_trafo_size)) return;/' \
       -e '/^static void deblocking_filter_CTB/,/^}/ s/^    uint8_t \*src;/    uint8_t *src = NULL;\n    if (b200_deblock_on_device()) return;/' "$P/hevc_filter.c"
# experiment, NOT applied by default (B200_AWAIT_GUARD=1 builds with it): hevc_await_progress (hevc.c:1951-1958) makes a frame thread wait
# until the rows of a reference picture its motion vector reaches have been reconstructed by another thread -- for pixels nobody reads on
# the host once the MC tables record (the device runs the pictures in decode order; the TMVP wait, hevc_mvs.c:260, would stay).  Bit-exact
# (CPU suite, emulated device with 4 / 8 frame threads, MD5 on the GPU at 32 threads); host-only (record and drop, 8 cores) +5 % at 8 and
# +12 % at 16 threads, but with the device no gain was measured, so the decoder keeps its own synchronisation.
if [ -n "${B200_AWAIT_GUARD:-}" ]; then
  sed -i -e '/^static void hevc_await_progress(HEVCContext \*s, HEVCFrame \*ref,/,/^}/ s/^    int y = (mv->y >> 2) + y0 + height + 9;/&\n    if (b200_host_pixels_unused()) return;   \/* reference PIXELS are not read on the host *\//' "$P/hevc.c"
  grep -q "b200_host_pixels_unused()) return;   /\* reference PIXELS" "$P/hevc.c" || { echo "await guard was not inserted" >&2; exit 1; }
fi
if [ -z "${B200_NO_COPY_GUARD:-}" ]; then
  sed -i -e "0,/^#include/s//$inc\n#include/" \
         -e '/^static void copy_CTB/,/^}/ s/^    int i;/&\n    if (b200_host_pixels_unused()) return;/' "$P/hevc_filter.c"
  grep -q "b200_host_pixels_unused" "$P/hevc_filter.c" || { echo "hook b200_host_pixels_unused was not inserted" >&2; exit 1; }
fi
for pat in ff_hevcdsp_init_b200 ff_hevcpred_init_b200 ff_videodsp_init_b200 b200_frame_begin b200_frame_end b200_frame_readback b200_frame_fill b200_frame_buffer_alloc b200_bs_on_device b200_deblock_on_device b200_worker_begin b200_decoder_close; do
  grep -q "$pat" "$P"/*.c || { echo "hook $pat was not inserted" >&2; exit 1; }
done
CFLAGS=$(cat "$OUT/cflags.txt")
for f in hevc hevcdsp hevcpred videodsp hevc_refs hevc_filter utils; do
  gcc $CFLAGS -fPIC -std=gnu99 -w -DPIC -I"$OUT/gen" -I"$REF/libavcodec" -I"$REF" -I"$REF/gpac/modules/openhevc_dec" -I"$ROOT/include" \
      -c "$P/$f.c" -o "$OUT/obj_b200/libavcodec_$f.o"
done
objs=$(ls "$OUT"/obj/*.o | grep -v -e 'libavcodec_hevc\.o' -e 'libavcodec_hevcdsp\.o' -e 'libavcodec_hevcpred\.o' -e 'libavcodec_videodsp\.o' -e 'libavcodec_hevc_refs\.o' -e 'libavcodec_hevc_filter\.o' -e 'libavcodec_utils\.o')
gcc -shared -o "$OUT/libohevc_b200.so" $objs "$OUT"/obj_b200/*.o -L"$OUT" -lb200hevc_shim -L"$ROOT/openhevc_b200" -lb200hevc \
    -Wl,-rpath,'$ORIGIN:$ORIGIN/../../openhevc_b200' -lm -lpthread
echo "built $OUT/libohevc_b200.so"
