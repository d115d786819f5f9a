/* port_picstats_backend.c — TEST INFRASTRUCTURE ONLY.  port_resized_backend.c (the CPU backend with error maps, the motion
 * export, the packed and the resized output) with the picture statistics on top: port_picstats_picture restates the
 * definition in include/edge264_picstats.h sample by sample, from the picture the restatement reconstructed and the
 * cropping rectangle of the submit (tests/test_picstats.py checks it against numpy and compares the device with it).  The
 * test links it with port_resized_backend.c, port_motion_backend.c and the product's host sources (decoder.c,
 * slice_dec.c) into a library of the whole edge264 API on the CPU, using -Wl,--wrap=e264_default_backend: the decoder
 * binds the table below, which is port_resized_backend.c's table with its submit_outputs extended to the statistics.
 * port_resized_backend.c names its table __wrap_e264_default_backend too, so the test renames that symbol in its object
 * file to port_resized_default_backend (objcopy --redefine-sym) before the link. */
#include <string.h>
#include "../../edge264_b200/csrc/dec.h"

/* frame: a picture in the layout of E264PicDesc (Y plane, then chroma rows alternating Cb, Cr) */
void port_picstats_picture(uint8_t *out, const E264PicDesc *pd, const uint8_t *frame, int left, int top, int width, int height) {
	const size_t nmb = (size_t)pd->width_mbs * pd->height_mbs;
	uint32_t *hist = (uint32_t *)(out + E264_PICSTATS_HIST), *sum = (uint32_t *)(out + E264_PICSTATS_SUM), *sum_sq = (uint32_t *)(out + E264_PICSTATS_SUM_SQ(nmb));
	memset(hist, 0, 3 * 256 * sizeof(uint32_t));
	for (int p = 0; p < 3; p++) {
		const int n = p ? 8 : 16, sh = p ? 1 : 0, stride = p ? pd->stride_c : pd->stride_y;
		const uint8_t *plane = p == 0 ? frame : frame + pd->plane_y + (p == 2 ? pd->stride_c >> 1 : 0);
		for (int y = 0; y < pd->height_mbs * n; y++) for (int x = 0; x < pd->width_mbs * n; x++) {
			const uint32_t v = plane[(size_t)y * stride + x];
			if (x >= left >> sh && x < (left + width) >> sh && y >= top >> sh && y < (top + height) >> sh) hist[p * 256 + v]++;
		}
		for (int mby = 0; mby < pd->height_mbs; mby++) for (int mbx = 0; mbx < pd->width_mbs; mbx++) {
			uint32_t s = 0, q = 0;
			for (int y = 0; y < n; y++) for (int x = 0; x < n; x++) {
				const uint32_t v = plane[(size_t)(mby * n + y) * stride + mbx * n + x];
				s += v; q += v * v;
			}
			sum[p * nmb + (size_t)mby * pd->width_mbs + mbx] = s;
			sum_sq[p * nmb + (size_t)mby * pd->width_mbs + mbx] = q;
		}
	}
}

const E264Backend *port_resized_default_backend(void);
static E264Backend picstats_backend;
static int (*resized_submit_outputs)(void *ctx, const E264PicDesc *pd, uint8_t *host_out, const E264Outputs *o, uint64_t *ticket);

static int be_submit_picstats(void *ctx, const E264PicDesc *pd, uint8_t *host_out, const E264Outputs *o, uint64_t *ticket) {
	if (!o->picstats) return resized_submit_outputs(ctx, pd, host_out, o, ticket);
	E264Outputs rest = *o;
	rest.picstats = NULL;
	const int r = resized_submit_outputs(ctx, pd, host_out, &rest, ticket);
	if (r) return r;
	port_picstats_picture(o->picstats, pd, host_out, o->ps_left, o->ps_top, o->ps_width, o->ps_height);
	if (o->picstats_on_device) *o->picstats_on_device = 0;
	return 0;
}
const E264Backend *__wrap_e264_default_backend(void) {
	picstats_backend = *port_resized_default_backend();
	resized_submit_outputs = picstats_backend.submit_outputs;
	picstats_backend.name = "port-picstats";
	picstats_backend.submit_outputs = be_submit_picstats;
	return &picstats_backend;
}
