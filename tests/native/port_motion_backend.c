/* port_motion_backend.c — TEST INFRASTRUCTURE ONLY.  The CPU backend of port_maps_backend.c (the plain-C restatement of
 * the reconstruction and of the error maps) with the motion export on top: port_motion_export restates, from the layout
 * of include/edge264_motion.h, what e264_motion_kernel derives from a picture's records.  tests/test_motion_export.py links
 * it with the product's host sources (decoder.c, slice_dec.c) into a library of the whole edge264 API on the CPU, motion
 * export included, and compares the device with it. */
#define e264_default_backend e264_maps_default_backend
#include "port_maps_backend.c"
#undef e264_default_backend

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

static int be_submit_motion(void *ctx, const E264PicDesc *pd, uint8_t *host_out, uint8_t *host_map, uint8_t *motion, const int32_t *slot_ids, int *on_device, uint64_t *ticket) {
	Ctx *c = (Ctx *)ctx;
	int r = be_submit_maps(ctx, pd, host_out, host_map, ticket);
	if (r) return r;
	port_motion_export(motion, pd, c->recs[pd->dst_slot], slot_ids);
	*on_device = 0;
	return 0;
}
static const E264Backend motion_backend = {"port-motion", be_create, be_destroy, be_configure, be_alloc, be_free, be_acquire, be_submit, be_wait, be_fill, be_poll,
                                           be_submit_maps, be_alloc, be_free, be_submit_motion};
const E264Backend *e264_default_backend(void) { return &motion_backend; }
