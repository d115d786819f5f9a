/* port_outputs_backend.c — TEST INFRASTRUCTURE ONLY.  The CPU restatement (oracle/port_recon.c) behind the decoder's
 * backend interface with every optional output of E264Outputs, each restated in plain C from its definition (not from
 * the kernels): the error maps (port_error_map.c; every frame slot has one, fill_slot makes a slot's map all 100), the
 * motion export (include/edge264_motion.h), the packed and the resized output (include/edge264_packed.h, the resized one
 * with the span and rounding helpers of the kernel's resize_math.cuh) and the picture statistics
 * (include/edge264_picstats.h), all from the picture the restatement reconstructed.  tests/checkers.py links it with the
 * product's host sources (decoder.c, slice_dec.c) into a library of the whole edge264 API on the CPU, and the tests
 * compare the device with it.  With E264_CHECK_RECORDS=1 every submitted picture is checked against the record contract
 * (oracle/record_check.c, and err <= 100); violations are counted (e264_test_record_violations). */
#include <errno.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../../edge264_b200/csrc/dec.h"
#include "../../edge264_b200/csrc/resize_math.cuh"
#include "../../oracle/record_check.h"

void port_recon_picture(uint8_t *frames, const E264PicDesc *pd, const E264MbRec *recs, const int16_t *coefs, const E264SliceRec *slices);
void port_error_map(uint8_t *maps, const E264PicDesc *pd, const E264MbRec *recs);

/* out: E264_MOTION_BYTES per macroblock, the four arrays of records.h; slot_ids: E264_MAX_SLOTS FrameIds */
void port_motion_export(uint8_t *out, const E264PicDesc *pd, const E264MbRec *recs, const int32_t *slot_ids) {
	const int W = pd->width_mbs, H = pd->height_mbs;
	const size_t nmb = (size_t)W * H;
	int16_t *mv = (int16_t *)(out + E264_MOTION_MV * nmb);
	int32_t *ref = (int32_t *)(out + E264_MOTION_REF * nmb);
	for (int l = 0; l < 2; l++) {
		for (int y = 0; y < 4 * H; y++) for (int x = 0; x < 4 * W; x++) {   /* 4x4 blocks in raster order */
			const E264MbRec *r = recs + (size_t)(y / 4) * W + x / 4;
			const int b = e264_blk_z(x % 4, y % 4);
			const int used = r->kind == MBK_INTER && r->ref_idx[l][b / 4] >= 0;
			int16_t *o = mv + (((size_t)l * 4 * H + y) * 4 * W + x) * 2;
			o[0] = used ? r->mv[l][b][0] : 0;
			o[1] = used ? r->mv[l][b][1] : 0;
		}
		for (int y = 0; y < 2 * H; y++) for (int x = 0; x < 2 * W; x++) {   /* 8x8 blocks in raster order */
			const E264MbRec *r = recs + (size_t)(y / 2) * W + x / 2;
			const int i8 = (y % 2) * 2 + x % 2, slot = r->ref_pic[l][i8];
			const int used = r->kind == MBK_INTER && r->ref_idx[l][i8] >= 0 && slot >= 0 && slot < E264_MAX_SLOTS;
			ref[((size_t)l * 2 * H + y) * 2 * W + x] = used ? slot_ids[slot] : -1;
		}
	}
	for (size_t a = 0; a < nmb; a++) {
		out[E264_MOTION_TYPE * nmb + a] = recs[a].kind == MBK_INTER && (recs[a].flags & MBF_SKIP) ? 5 : recs[a].kind;
		out[E264_MOTION_QP * nmb + a] = recs[a].qp[0];
	}
}

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

#define NSTAGE 8
typedef struct {
	E264PicDesc g; int n_slots, n_stage, stage; size_t nmb;
	uint8_t *frames_alloc, *frames, *maps;
	E264MbRec *recs[E264_MAX_SLOTS];
	int16_t *coefs[NSTAGE]; uint32_t coef_cap;
	E264SliceRec *slices[NSTAGE];
	uint32_t *intra_list[NSTAGE];
} Ctx;

static int violations;
static char last_violation[256];
int e264_test_record_violations(void) { return __atomic_load_n(&violations, __ATOMIC_RELAXED); }
const char *e264_test_last_violation(void) { return last_violation; }

static void free_all(Ctx *c) {
	free(c->frames_alloc); free(c->maps); c->frames_alloc = c->maps = NULL;
	for (int i = 0; i < E264_MAX_SLOTS; i++) { free(c->recs[i]); c->recs[i] = NULL; }
	for (int i = 0; i < NSTAGE; i++) { free(c->coefs[i]); free(c->slices[i]); free(c->intra_list[i]); c->coefs[i] = NULL; c->slices[i] = NULL; c->intra_list[i] = NULL; }
}
static int be_create(void **ctx) { *ctx = calloc(1, sizeof(Ctx)); return *ctx ? 0 : -1; }
static void be_destroy(void *ctx) { free_all((Ctx *)ctx); free(ctx); }
static int be_configure(void *ctx, const E264PicDesc *g, int n_slots) {
	Ctx *c = (Ctx *)ctx;
	free_all(c);
	c->g = *g; c->n_slots = n_slots; c->nmb = (size_t)g->width_mbs * g->height_mbs;
	size_t margin = (size_t)g->stride_y * 2 + 64;
	if (!(c->frames_alloc = calloc((size_t)g->frame_bytes * n_slots + 2 * margin, 1)) || !(c->maps = calloc(c->nmb * n_slots, 1))) return -1;
	c->frames = c->frames_alloc + margin;
	for (int i = 0; i < n_slots; i++) if (!(c->recs[i] = calloc(c->nmb, sizeof(E264MbRec)))) return -1;
	c->coef_cap = (uint32_t)(c->nmb * 408);
	c->n_stage = g->staging > 0 ? (g->staging < NSTAGE ? g->staging : NSTAGE) : 2;
	c->stage = 0;
	for (int i = 0; i < c->n_stage; i++)
		if (!(c->coefs[i] = calloc(c->coef_cap, 2)) || !(c->slices[i] = calloc(E264_MAX_SLICES, sizeof(E264SliceRec))) || !(c->intra_list[i] = calloc(c->nmb, 4))) return -1;
	return 0;
}
static void *be_alloc(void *ctx, size_t bytes) { (void)ctx; return calloc(bytes, 1); }
static void be_free(void *ctx, void *p) { (void)ctx; free(p); }
static int be_acquire(void *ctx, int slot, E264Staging *out) {
	Ctx *c = (Ctx *)ctx;
	c->stage = (c->stage + 1) % c->n_stage;
	out->handle = c->stage; out->recs = c->recs[slot]; out->coefs = c->coefs[c->stage]; out->coef_capacity = c->coef_cap;
	out->slices = c->slices[c->stage]; out->intra_list = c->intra_list[c->stage];
	return 0;
}
/* one picture and whatever o asks for besides its samples; host_out receives the whole frame slot, so the packed output
 * and the statistics are computed from it */
static int be_submit_outputs(void *ctx, const E264PicDesc *pd, uint8_t *host_out, const E264Outputs *o, uint64_t *ticket) {
	Ctx *c = (Ctx *)ctx;
	*ticket = 0;
	if (pd->staging < 0 || pd->staging >= c->n_stage) return -1;
	const E264MbRec *recs = c->recs[pd->dst_slot];
	const char *chk = getenv("E264_CHECK_RECORDS");
	if (chk && atoi(chk)) {
		char why[256]; why[0] = 0;
		int bad = e264_check_records(pd, recs, c->coefs[pd->staging], c->slices[pd->staging], c->intra_list[pd->staging], c->n_slots, why, sizeof(why));
		for (size_t a = 0; a < c->nmb && !bad; a++) if (recs[a].err > 100) { bad = 1; snprintf(why, sizeof(why), "mb %zu: err %d", a, recs[a].err); }
		if (bad) { __atomic_add_fetch(&violations, 1, __ATOMIC_RELAXED); memcpy(last_violation, why, sizeof(why)); }
	}
	port_recon_picture(c->frames, pd, recs, c->coefs[pd->staging], c->slices[pd->staging]);
	memcpy(host_out, c->frames + (size_t)pd->dst_slot * pd->frame_bytes, (size_t)pd->frame_bytes);
	port_error_map(c->maps, pd, recs);
	if (pd->err_pic && o->map) memcpy(o->map, c->maps + (size_t)pd->dst_slot * c->nmb, c->nmb);
	if (o->motion) {
		int32_t ids[E264_MAX_SLOTS];   /* FrameIds past n_ids are -1, as in the device's table */
		for (int k = 0; k < E264_MAX_SLOTS; k++) ids[k] = k < o->n_ids ? o->slot_ids[k] : -1;
		port_motion_export(o->motion, pd, recs, ids);
	}
	if (o->packed) (o->pk.target_width ? port_resize_picture : port_pack_picture)(o->packed, pd, host_out, &o->pk);
	if (o->picstats) port_picstats_picture(o->picstats, pd, host_out, o->ps_left, o->ps_top, o->ps_width, o->ps_height);
	if (o->motion_on_device) *o->motion_on_device = 0;
	if (o->packed_on_device) *o->packed_on_device = 0;
	if (o->picstats_on_device) *o->picstats_on_device = 0;
	return 0;
}
static int be_submit(void *ctx, const E264PicDesc *pd, uint8_t *host_out, uint64_t *ticket) { return be_submit_outputs(ctx, pd, host_out, &(E264Outputs){0}, ticket); }
static int be_submit_maps(void *ctx, const E264PicDesc *pd, uint8_t *host_out, uint8_t *host_map, uint64_t *ticket) {
	return be_submit_outputs(ctx, pd, host_out, &(E264Outputs){.map = host_map}, ticket);
}
static int be_submit_motion(void *ctx, const E264PicDesc *pd, uint8_t *host_out, uint8_t *host_map, uint8_t *motion, const int32_t *slot_ids, int *on_device, uint64_t *ticket) {
	return be_submit_outputs(ctx, pd, host_out, &(E264Outputs){.map = host_map, .motion = motion, .slot_ids = slot_ids, .n_ids = E264_MAX_SLOTS, .motion_on_device = on_device}, ticket);
}
static int be_wait(void *ctx, uint64_t ticket) { (void)ctx; (void)ticket; return 0; }
static int be_poll(void *ctx, uint64_t ticket) { (void)ctx; (void)ticket; return 0; }
static int be_fill(void *ctx, int slot, int y, int cc) {
	Ctx *c = (Ctx *)ctx;
	uint8_t *f = c->frames + (size_t)slot * c->g.frame_bytes;
	memset(f, y, (size_t)c->g.plane_y); memset(f + c->g.plane_y, cc, (size_t)c->g.frame_bytes - c->g.plane_y);
	memset(c->maps + (size_t)slot * c->nmb, 100, c->nmb);   /* a made-up picture: every macroblock wrong */
	return 0;
}
static const E264Backend outputs_backend = {"port-outputs", be_create, be_destroy, be_configure, be_alloc, be_free, be_acquire, be_submit, be_wait, be_fill, be_poll,
                                            be_submit_maps, be_alloc, be_free, be_submit_motion, be_submit_outputs};
const E264Backend *e264_default_backend(void) { return &outputs_backend; }
