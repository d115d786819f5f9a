/* port_resized_backend.c — TEST INFRASTRUCTURE ONLY.  port_packed_backend.c (the CPU backend of port_motion_backend.c
 * with the power-of-two packed output) with the resized output on top: port_resize_picture restates the definition in
 * include/edge264_packed.h sample by sample, from the picture the restatement reconstructed, with the span and rounding
 * helpers of the kernel's resize_math.cuh (tests/test_resized_output.py checks those against Python integers and this
 * file against numpy).  The test links it with port_motion_backend.c and the product's host sources (decoder.c,
 * slice_dec.c) into a library of the whole edge264 API on the CPU, using -Wl,--wrap=e264_default_backend: the decoder
 * binds the table below, which is port_packed_backend.c's table with its submit_outputs extended to the resized mode. */
#define __wrap_e264_default_backend port_packed_default_backend
#include "port_packed_backend.c"
#undef __wrap_e264_default_backend
#include "../../edge264_b200/csrc/resize_math.cuh"

/* one plane: src the first cropped sample, s_w x s_h its cropped size, t_w x t_h the output's; dst_step 1, or 2 for a
 * component of NV12's CbCr rows */
static void resize_plane(uint8_t *dst, int dst_stride, int dst_step, const uint8_t *src, int src_stride, int s_w, int s_h, int t_w, int t_h) {
	const int64_t d = (int64_t)s_w * s_h;
	const double inv = e264_rs_inv(d);
	for (int y = 0; y < t_h; y++) {
		const RsSpan sy = e264_rs_span(y, s_h, t_h);
		for (int x = 0; x < t_w; x++) {
			const RsSpan sx = e264_rs_span(x, s_w, t_w);
			int64_t n = 0;
			for (int j = sy.first; j <= sy.last; j++) {
				const int64_t b = t_h - (j == sy.first ? sy.cut_first : 0) - (j == sy.last ? sy.cut_last : 0);
				for (int i = sx.first; i <= sx.last; i++)
					n += b * (t_w - (i == sx.first ? sx.cut_first : 0) - (i == sx.last ? sx.cut_last : 0)) * src[(size_t)j * src_stride + i];
			}
			dst[(size_t)y * dst_stride + x * dst_step] = (uint8_t)e264_rs_round(n, d, inv);
		}
	}
}

/* frame: a picture in the layout of E264PicDesc (Y plane, then chroma rows alternating Cb, Cr) */
void port_resize_picture(uint8_t *out, const E264PicDesc *pd, const uint8_t *frame, const E264PackedDesc *pk) {
	const E264PackedLayout l = e264_packed_layout(pk);
	const uint8_t *cb = frame + pd->plane_y + (size_t)(pk->top >> 1) * pd->stride_c + (pk->left >> 1), *cr = cb + (pd->stride_c >> 1);
	const int nv12 = pk->format == E264_PACKED_NV12, wc = pk->width >> 1, hc = pk->height >> 1;
	resize_plane(out + l.offset[0], l.stride[0], 1, frame + (size_t)pk->top * pd->stride_y + pk->left, pd->stride_y, pk->width, pk->height, l.width, l.height);
	resize_plane(out + l.offset[1], l.stride[1], nv12 ? 2 : 1, cb, pd->stride_c, wc, hc, l.width_C, l.height_C);
	if (nv12) resize_plane(out + l.offset[1] + 1, l.stride[1], 2, cr, pd->stride_c, wc, hc, l.width_C, l.height_C);
	else resize_plane(out + l.offset[2], l.stride[2], 1, cr, pd->stride_c, wc, hc, l.width_C, l.height_C);
}

static E264Backend resized_backend;

static int be_submit_resized(void *ctx, const E264PicDesc *pd, uint8_t *host_out, const E264Outputs *o, uint64_t *ticket) {
	if (!o->packed || !o->pk.target_width) return packed_backend.submit_outputs(ctx, pd, host_out, o, ticket);
	E264Outputs rest = *o;
	rest.packed = NULL;
	const int r = packed_backend.submit_outputs(ctx, pd, host_out, &rest, ticket);
	if (r) return r;
	port_resize_picture(o->packed, pd, host_out, &o->pk);
	if (o->packed_on_device) *o->packed_on_device = 0;
	return 0;
}
const E264Backend *__wrap_e264_default_backend(void) {
	resized_backend = *port_packed_default_backend();
	resized_backend.name = "port-resized";
	resized_backend.submit_outputs = be_submit_resized;
	return &resized_backend;
}
