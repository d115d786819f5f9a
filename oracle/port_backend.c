/* oracle/port_backend.c — TEST INFRASTRUCTURE ONLY.  Binds the CPU restatement (port_recon.c) behind
 * the decoder's backend interface so that the host parser + record ABI can be validated against the
 * compiled reference decoder without a GPU (tests/test_oracle_vs_ref.py), and so that GPU output can
 * be compared with it picture by picture.  Linked only into oracle/liboracle_dec.so. */
#include <errno.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../edge264_b200/csrc/dec.h"
#include "record_check.h"

void port_recon_picture(uint8_t *frames, const E264PicDesc *pd, const E264MbRec *recs, const int16_t *coefs, const E264SliceRec *slices);

#define PORT_NSTAGE 8
typedef struct PortCtx {
	E264PicDesc g; int n_slots;
	uint8_t *frames_alloc, *frames;
	E264MbRec *recs[E264_MAX_SLOTS];
	/* staging areas, handed out round robin like the CUDA runtime's (a threaded decoder fills several pictures at once) */
	int16_t *coefs[PORT_NSTAGE]; uint32_t coef_cap;
	E264SliceRec *slices[PORT_NSTAGE];
	uint32_t *intra_list[PORT_NSTAGE];
	int stage, n_stage;
	int cur_slot;
	uint64_t tick_seq; int polls[64]; int n_waits;      /* E264_PORT_LATE: see port_submit */
} PortCtx;
static int port_late(void) { static int v = -1; if (v < 0) { const char *e = getenv("E264_PORT_LATE"); v = e ? atoi(e) : 0; } return v; }

static int port_create(void **ctx) { *ctx = calloc(1, sizeof(PortCtx)); return *ctx ? 0 : -1; }
static void port_free_all(PortCtx *c) {
	free(c->frames_alloc); for (int i = 0; i < E264_MAX_SLOTS; i++) { free(c->recs[i]); c->recs[i] = NULL; }
	for (int i = 0; i < PORT_NSTAGE; i++) { free(c->coefs[i]); free(c->slices[i]); free(c->intra_list[i]); c->coefs[i] = NULL; c->slices[i] = NULL; c->intra_list[i] = NULL; }
	c->frames_alloc = NULL;
}
static void port_destroy(void *ctx) { port_free_all((PortCtx *)ctx); free(ctx); }
static int port_configure(void *ctx, const E264PicDesc *g, int n_slots) {
	PortCtx *c = (PortCtx *)ctx;
	port_free_all(c);
	c->g = *g; c->n_slots = n_slots;
	size_t margin = (size_t)g->stride_y * 2 + 64;
	c->frames_alloc = (uint8_t *)calloc((size_t)g->frame_bytes * n_slots + 2 * margin, 1);
	if (!c->frames_alloc) return -1;
	c->frames = c->frames_alloc + margin;
	size_t nmb = (size_t)g->width_mbs * g->height_mbs;
	for (int i = 0; i < n_slots; i++) if (!(c->recs[i] = (E264MbRec *)calloc(nmb, sizeof(E264MbRec)))) return -1;
	c->coef_cap = (uint32_t)(nmb * 408);
	c->n_stage = g->staging > 0 ? (g->staging < PORT_NSTAGE ? g->staging : PORT_NSTAGE) : 2;
	c->stage = 0;
	for (int i = 0; i < c->n_stage; i++) {
		c->coefs[i] = (int16_t *)calloc(c->coef_cap, sizeof(int16_t));
		c->slices[i] = (E264SliceRec *)calloc(E264_MAX_SLICES, sizeof(E264SliceRec));
		c->intra_list[i] = (uint32_t *)calloc(nmb, sizeof(uint32_t));
		if (!c->coefs[i] || !c->slices[i] || !c->intra_list[i]) return -1;
	}
	return 0;
}
static void *port_host_alloc(void *ctx, size_t bytes) { (void)ctx; return calloc(bytes, 1); }
static void port_host_free(void *ctx, void *p) { (void)ctx; free(p); }
static int port_acquire(void *ctx, int slot, E264Staging *out) {
	PortCtx *c = (PortCtx *)ctx;
	c->stage = (c->stage + 1) % c->n_stage;
	out->handle = c->stage; out->recs = c->recs[slot]; out->coefs = c->coefs[c->stage]; out->coef_capacity = c->coef_cap; out->slices = c->slices[c->stage]; out->intra_list = c->intra_list[c->stage];
	c->cur_slot = slot;
	return 0;
}
static int port_submit(void *ctx, const E264PicDesc *pd, uint8_t *host_out, uint64_t *ticket) {
	PortCtx *c = (PortCtx *)ctx;
	static int pic_no;
	const char *dump = getenv("E264_DUMP");   /* "pic,mbx,mby": print that macroblock's record (debugging aid) */
	if (dump) {
		int pn, mx, my;
		if (sscanf(dump, "%d,%d,%d", &pn, &mx, &my) == 3 && pn == pic_no) {
			const E264MbRec *r = c->recs[pd->dst_slot] + my * pd->width_mbs + mx;
			fprintf(stderr, "pic %d mb(%d,%d) kind %d flags %02x qp %d %d %d chroma_mode %02x i16 %02x coded %08x\n modes", pn, mx, my, r->kind, r->flags, r->qp[0], r->qp[1], r->qp[2], r->chroma_mode, r->i16_mode, r->coded);
			for (int i = 0; i < 16; i++) fprintf(stderr, " %02x", r->modes[i]);
			fprintf(stderr, "\n ref_idx"); for (int i = 0; i < 8; i++) fprintf(stderr, " %d", ((int8_t *)r->ref_idx)[i]);
			fprintf(stderr, " ref_pic"); for (int i = 0; i < 8; i++) fprintf(stderr, " %d", ((int8_t *)r->ref_pic)[i]);
			for (int l = 0; l < 2; l++) { fprintf(stderr, "\n mv%d", l); for (int i = 0; i < 16; i++) fprintf(stderr, " (%d,%d)", r->mv[l][i][0], r->mv[l][i][1]); }
			fprintf(stderr, "\n");
		}
	}
	pic_no++;
	if (pd->staging < 0 || pd->staging >= c->n_stage) return -1;
	/* E264_CHECK_RECORDS=1: every submitted picture must keep the record contract (records.h); stop at the first violation */
	const char *chk = getenv("E264_CHECK_RECORDS");
	if (chk && atoi(chk)) {
		char why[256];
		if (e264_check_records(pd, c->recs[pd->dst_slot], c->coefs[pd->staging], c->slices[pd->staging], c->intra_list[pd->staging], c->n_slots, why, sizeof(why))) {
			fprintf(stderr, "E264_CHECK_RECORDS: picture %d (slot %d): %s\n", pic_no - 1, pd->dst_slot, why);
			abort();
		}
	}
	if (!getenv("E264_NULL_RECON")) port_recon_picture(c->frames, pd, c->recs[pd->dst_slot], c->coefs[pd->staging], c->slices[pd->staging]);
	if (!getenv("E264_NULL_RECON")) memcpy(host_out, c->frames + (size_t)pd->dst_slot * pd->frame_bytes, (size_t)pd->frame_bytes);
	/* E264_PORT_LATE=n (tests of the decoder's output logic): pictures get tickets and count as "still on the device" until
	 * they have been polled n times or waited for, like a GPU that has not finished yet */
	*ticket = port_late() ? ++c->tick_seq : 0;
	if (*ticket) c->polls[*ticket % 64] = 0;
	return 0;
}
static int g_port_waits;
static int port_wait(void *ctx, uint64_t ticket) { PortCtx *c = (PortCtx *)ctx; if (ticket && c->polls[ticket % 64] < port_late()) { c->polls[ticket % 64] = 1 << 30; c->n_waits++; __atomic_add_fetch(&g_port_waits, 1, __ATOMIC_RELAXED); } return 0; }
static int port_fill(void *ctx, int slot, int y, int cc) {
	PortCtx *c = (PortCtx *)ctx;
	uint8_t *f = c->frames + (size_t)slot * c->g.frame_bytes;
	memset(f, y, (size_t)c->g.plane_y); memset(f + c->g.plane_y, cc, (size_t)c->g.frame_bytes - c->g.plane_y);
	return 0;
}
static int port_poll(void *ctx, uint64_t ticket) {
	PortCtx *c = (PortCtx *)ctx;
	if (!ticket) return 0;
	if (c->polls[ticket % 64] >= port_late()) return 0;
	c->polls[ticket % 64]++;
	return EAGAIN;
}
/* test hook: how often a decoder had to WAIT for a picture that was not finished (it may only do so after ENOBUFS / at the
 * end of the stream) */
int e264_port_waits(void) { return __atomic_load_n(&g_port_waits, __ATOMIC_RELAXED); }
static const E264Backend port_backend = {"oracle-port", port_create, port_destroy, port_configure, port_host_alloc, port_host_free, port_acquire, port_submit, port_wait, port_fill, port_poll};
const E264Backend *e264_default_backend(void) { return &port_backend; }
