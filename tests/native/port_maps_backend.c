/* port_maps_backend.c — TEST INFRASTRUCTURE ONLY.  The CPU restatement (oracle/port_recon.c) behind the decoder's backend
 * interface like oracle/port_backend.c, and in addition the error maps: every frame slot has one, pictures with err_pic
 * get theirs from port_error_map.c, fill_slot makes a slot's map all 100.  tests/test_mb_errors.py links it with the
 * product's host sources (decoder.c, slice_dec.c) into a library of the whole edge264 API on the CPU, error maps
 * included, and compares the device with it.  With E264_CHECK_RECORDS=1 every submitted picture is checked against the
 * record contract (oracle/record_check.c, and err <= 100); violations are counted (e264_test_record_violations). */
#include <errno.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../../edge264_b200/csrc/dec.h"
#include "../../oracle/record_check.h"

void port_recon_picture(uint8_t *frames, const E264PicDesc *pd, const E264MbRec *recs, const int16_t *coefs, const E264SliceRec *slices);
void port_error_map(uint8_t *maps, const E264PicDesc *pd, const E264MbRec *recs);

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
static int be_submit_maps(void *ctx, const E264PicDesc *pd, uint8_t *host_out, uint8_t *host_map, uint64_t *ticket) {
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
	if (pd->err_pic && host_map) memcpy(host_map, c->maps + (size_t)pd->dst_slot * c->nmb, c->nmb);
	return 0;
}
static int be_submit(void *ctx, const E264PicDesc *pd, uint8_t *host_out, uint64_t *ticket) { return be_submit_maps(ctx, pd, host_out, NULL, ticket); }
static int be_wait(void *ctx, uint64_t ticket) { (void)ctx; (void)ticket; return 0; }
static int be_poll(void *ctx, uint64_t ticket) { (void)ctx; (void)ticket; return 0; }
static int be_fill(void *ctx, int slot, int y, int cc) {
	Ctx *c = (Ctx *)ctx;
	uint8_t *f = c->frames + (size_t)slot * c->g.frame_bytes;
	memset(f, y, (size_t)c->g.plane_y); memset(f + c->g.plane_y, cc, (size_t)c->g.frame_bytes - c->g.plane_y);
	memset(c->maps + (size_t)slot * c->nmb, 100, c->nmb);   /* a made-up picture: every macroblock wrong */
	return 0;
}
static const E264Backend maps_backend = {"port-maps", be_create, be_destroy, be_configure, be_alloc, be_free, be_acquire, be_submit, be_wait, be_fill, be_poll,
                                         be_submit_maps, be_alloc, be_free};
const E264Backend *e264_default_backend(void) { return &maps_backend; }
