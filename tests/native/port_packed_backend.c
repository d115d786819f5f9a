/* port_packed_backend.c — TEST INFRASTRUCTURE ONLY.  The CPU backend of port_motion_backend.c (reconstruction, error maps
 * and motion export restated in plain C) with the packed output on top: port_pack_picture restates the definition in
 * include/edge264_packed.h sample by sample, from the picture the restatement reconstructed.  tests/test_packed_output.py
 * links both files with the product's host sources (decoder.c, slice_dec.c) into a library of the whole edge264 API on
 * the CPU, both exports included, and compares the device with it.  The link uses -Wl,--wrap=e264_default_backend: the
 * decoder binds the table below, which is port_motion_backend.c's table (__real_) plus submit_outputs. */
#include <string.h>
#include "../../edge264_b200/csrc/dec.h"

/* one plane: src the first cropped sample, w x h its cropped size; dst_step 1, or 2 for a component of NV12's CbCr rows */
static void pack_plane(uint8_t *dst, int dst_stride, int dst_step, const uint8_t *src, int src_stride, int w, int h, int k) {
	const int n = 1 << k;
	for (int y = 0; y * n < h; y++) for (int x = 0; x * n < w; x++) {
		int sum = 0;
		for (int dy = 0; dy < n; dy++) for (int dx = 0; dx < n; dx++) {
			const int sy = y * n + dy < h ? y * n + dy : h - 1, sx = x * n + dx < w ? x * n + dx : w - 1;
			sum += src[(size_t)sy * src_stride + sx];
		}
		dst[(size_t)y * dst_stride + x * dst_step] = (uint8_t)((sum + (n * n >> 1)) >> (2 * k));
	}
}

/* frame: a picture in the layout of E264PicDesc (Y plane, then chroma rows alternating Cb, Cr) */
void port_pack_picture(uint8_t *out, const E264PicDesc *pd, const uint8_t *frame, const E264PackedDesc *pk) {
	const E264PackedLayout l = e264_packed_layout(pk);
	const uint8_t *cb = frame + pd->plane_y + (size_t)(pk->top >> 1) * pd->stride_c + (pk->left >> 1), *cr = cb + (pd->stride_c >> 1);
	const int nv12 = pk->format == E264_PACKED_NV12, k = pk->log2_scale, wc = pk->width >> 1, hc = pk->height >> 1;
	pack_plane(out + l.offset[0], l.stride[0], 1, frame + (size_t)pk->top * pd->stride_y + pk->left, pd->stride_y, pk->width, pk->height, k);
	pack_plane(out + l.offset[1], l.stride[1], nv12 ? 2 : 1, cb, pd->stride_c, wc, hc, k);
	if (nv12) pack_plane(out + l.offset[1] + 1, l.stride[1], 2, cr, pd->stride_c, wc, hc, k);
	else pack_plane(out + l.offset[2], l.stride[2], 1, cr, pd->stride_c, wc, hc, k);
}

const E264Backend *__real_e264_default_backend(void);
static E264Backend packed_backend;

/* host_out receives the whole frame slot, so the picture is packed from it */
static int be_submit_outputs(void *ctx, const E264PicDesc *pd, uint8_t *host_out, const E264Outputs *o, uint64_t *ticket) {
	int r = o->motion ? packed_backend.submit_motion(ctx, pd, host_out, o->map, o->motion, o->slot_ids, o->motion_on_device, ticket)
	                  : packed_backend.submit_maps(ctx, pd, host_out, o->map, ticket);
	if (r || !o->packed) return r;
	port_pack_picture(o->packed, pd, host_out, &o->pk);
	if (o->packed_on_device) *o->packed_on_device = 0;
	return 0;
}
const E264Backend *__wrap_e264_default_backend(void) {
	packed_backend = *__real_e264_default_backend();
	packed_backend.name = "port-packed";
	packed_backend.submit_outputs = be_submit_outputs;
	return &packed_backend;
}
