/* record_fuzz — random pictures of records, drawn at the edges where the reconstruction arithmetic branches, through the
 * device (libedge264_b200.so's e264b_* entry points) and through the CPU restatement (oracle/port_recon.c); every frame
 * must come out byte for byte the same.  Every picture keeps the record contract (oracle/record_check.c) before either
 * side sees it.  tests/test_record_fuzz.py builds and runs it.
 *   record_fuzz [--cpu-only] [--lib libedge264_b200.so] [--seeds A-B] [--pictures N] [--geom WxH] [--contexts M] [--inflight K]
 * --cpu-only generates, checks and reconstructs on the CPU restatement only.  At the end it prints one line per coverage
 * counter ("cov NAME VALUE"), counted from the generated inputs and, for saturation and wrap-around, in the port.
 * --contexts M --inflight K (default 1 and 1: one picture at a time, compared before the next is drawn) runs M device
 * contexts on M host threads, each taking every M-th seed with its own geometry, slot count and number of staging areas
 * (often fewer than K).  A context draws K pictures, reconstructing each on the port at once and keeping the port's
 * frame, then submits the K back to back, each with its own output buffer, and only then waits for them and compares
 * them in order.  References stay random among the other slots, biased towards the slot of the picture drawn just
 * before, so that pictures read slots that pictures in flight still write and overwrite slots they still read.  Extra
 * counters: inflight_max, contexts, ref_slot_in_flight, dst_slot_read_in_flight, and staging_wrapped (pictures submitted
 * while every staging area of the context was in use, so that e264b_acquire_staging had to wait), after one line of
 * pictures per context.
 * --dump DIR (one picture in flight) writes seed k to DIR/seed_k.bin (the format of tests/picture_dumps.py): the geometry,
 * the initial fill of every frame slot, then for every picture its E264PicDesc, records, slice records, levels, the
 * picture before deblocking and the picture after it (tests/test_deblock_spec.py, tests/test_picture_spec.py).  The picture
 * before deblocking is reconstructed first, from a copy of the records with MBF_DEBLOCK / MBF_EDGE_* cleared and
 * any_deblock 0, by the port (--cpu-only) or by the device; then the picture is reconstructed as drawn, so the frame
 * slots hold what they hold without --dump.  The draws are the same with and without it. */
#define _GNU_SOURCE
#include <dlfcn.h>
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../../oracle/record_check.h"
#include "../../edge264_b200/csrc/h264_tables.h"

#define MAX_SLOTS 20
#define MAX_SLICES 64

void port_recon_picture(uint8_t *frames, const E264PicDesc *pd, const E264MbRec *recs, const int16_t *coefs, const E264SliceRec *slices);
int port_boundary_strength(const E264MbRec *p, int bp, const E264MbRec *q, int bq, int mb_edge);
extern long port_cov_residual[6], port_cov_wp_bi_sat16;
/* the port counts its saturation and wrap-around events (and its E264_COVERAGE limits) in process-wide counters: the
 * contexts' host threads reconstruct on it one at a time */
static pthread_mutex_t port_mu = PTHREAD_MUTEX_INITIALIZER;

/* ---- the device, through the product library's C ABI (include/e264b_recon.h) ---- */
static struct {
	int (*create)(void **);
	void (*destroy)(void *);
	int (*configure)(void *, const E264PicDesc *, int);
	void *(*host_alloc)(void *, size_t);
	void (*host_free)(void *, void *);
	int (*acquire)(void *, int, E264Staging *);
	int (*submit)(void *, const E264PicDesc *, uint8_t *, uint64_t *);
	int (*wait)(void *, uint64_t);
	int (*fill)(void *, int, int, int);
	int (*error_flag)(void *);
} D;

static void load_device(const char *lib) {
	void *h = dlopen(lib, RTLD_NOW);
	if (!h) { fprintf(stderr, "dlopen %s: %s\n", lib, dlerror()); exit(3); }
#define SYM(f, name) if (!(*(void **)&D.f = dlsym(h, name))) { fprintf(stderr, "missing %s\n", name); exit(3); }
	SYM(create, "e264b_create") SYM(destroy, "e264b_destroy") SYM(configure, "e264b_configure") SYM(host_alloc, "e264b_host_alloc")
	SYM(host_free, "e264b_host_free") SYM(acquire, "e264b_acquire_staging") SYM(submit, "e264b_submit") SYM(wait, "e264b_wait")
	SYM(fill, "e264b_fill_slot") SYM(error_flag, "e264b_error_flag")
#undef SYM
}

/* ---- random numbers (the generator's state is per host thread: each context draws its own pictures; the coverage
 * counters below too, summed when the thread ends) ---- */
static _Thread_local uint64_t rng;
static uint32_t r32(void) { rng ^= rng >> 12; rng ^= rng << 25; rng ^= rng >> 27; return (uint32_t)((rng * 0x2545F4914F6CDD1Dull) >> 32); }
static int rnd(int n) { return n > 0 ? (int)(r32() % (unsigned)n) : 0; }
static int pct(int p) { return rnd(100) < p; }
static int pick(const int *v, int n) { return v[rnd(n)]; }

/* ---- coverage counters ---- */
enum {
	C_QPY, C_QPCB, C_QPCR, C_LEVEL_MAX, C_LEVEL_MIN, C_SCL_FLAT, C_SCL_255, C_SCL_1, C_SCL_RANDOM,
	C_W_M128, C_W_127, C_W128_UNI_LWD7, C_O_M128, C_O_127, C_LWD0, C_LWD7, C_IW_M64, C_IW_128, C_IW_OTHER, C_SAMEPIC_TWO_IDX,
	C_MV_INT16, C_MV_BORDER, C_DMV3X, C_DMV4X, C_DMV3Y, C_DMV4Y, C_SAME_BOTH_LISTS, C_SWAPPED, C_ONE_VS_TWO,
	C_BS,   /* 30 entries: [left, top, internal][t4x4, t8x8][bS 0..4] */
	C_FOFF_M12 = C_BS + 30, C_FOFF_P12, C_IDC0, C_IDC1, C_IDC2, C_SLICES64,
	C_INTRA_COMBOS, C_IPCM, C_CONCEAL_INTER, C_CONCEAL_INTRA,
	C_FRAC_0, C_FRAC_1, C_FRAC_BELOW, C_FRAC_AT, C_FRAC_ABOVE, C_FRAC_ALL, C_WP_LWD7_BRIGHT, C_PICTURES,
	C_INFLIGHT_MAX, C_REF_IN_FLIGHT, C_DST_READ_IN_FLIGHT, C_STAGING_WRAPPED, C_CONTEXTS, C_N   /* counted with pictures in flight */
};
static _Thread_local long cov[C_N];
static _Thread_local uint64_t qp_seen[3];
static _Thread_local uint8_t intra_seen[3 + 1][9][16];   /* kind (I4x4, I8x8, I16x16, chroma) x mode x unavailability */
static const char *bs_name(int i) {
	static char b[40]; snprintf(b, sizeof(b), "bs_%s_%s_%d", (i / 10) == 0 ? "left" : (i / 10) == 1 ? "top" : "internal", (i / 5) & 1 ? "t8x8" : "t4x4", i % 5); return b;
}

/* ---- geometry and frames ---- */
#define FUZZ_NSTAGE 8   /* staging areas e264b_configure allocates at most (NSTAGE of recon.cu) */
typedef struct {        /* a picture drawn and reconstructed on the port, not yet compared with the device */
	int pic, dst; uint32_t reads;               /* reads: bit s = some block predicts from slot s */
	E264PicDesc pd; uint64_t ticket;
	uint8_t *host_out, *port;                   /* the device's frame (e264b_host_alloc) and the port's frame of the same slot */
	E264MbRec *recs; int16_t *coefs; E264SliceRec *slices; uint32_t *intra_list;   /* its records */
} Pending;
typedef struct {
	E264PicDesc g; int n_slots, nmb;
	uint8_t *port_frames, *port_alloc;     /* the port's frame slots */
	E264MbRec *recs; int16_t *coefs; uint32_t coef_cap; E264SliceRec *slices; uint32_t *intra_list;   /* one picture being built */
	void *dev;
	int inflight, n_stage;                 /* pictures submitted ahead at most; staging areas of the device context */
	Pending *q; int q_head, n_out;         /* the pictures drawn and not yet compared, oldest first */
	int prev_dst;                          /* slot of the picture drawn last (with pictures in flight) */
	FILE *dump; E264MbRec *dump_recs; uint8_t *dump_pre, *dump_dev;   /* --dump: the file, flags-cleared records, picture before deblocking */
} Ctx;
static const char *dump_dir;

static void geometry(Ctx *c, int W, int H, int n_slots) {
	memset(&c->g, 0, sizeof(c->g));
	c->g.width_mbs = W; c->g.height_mbs = H;
	c->g.stride_y = W * 16; if (!(c->g.stride_y & 2047)) c->g.stride_y += 16;     /* the decoder's layout (decoder.c) */
	c->g.stride_c = W * 16; if (!(c->g.stride_c & 4095)) c->g.stride_c += 16;
	c->g.plane_y = c->g.stride_y * H * 16;
	c->g.frame_bytes = c->g.plane_y + c->g.stride_c * H * 8 + 16;
	c->n_slots = n_slots; c->nmb = W * H;
	size_t margin = (size_t)c->g.stride_y * 2 + 64;
	c->port_alloc = calloc((size_t)c->g.frame_bytes * n_slots + 2 * margin, 1);
	c->port_frames = c->port_alloc + margin;
	c->recs = calloc(c->nmb, sizeof(E264MbRec));
	c->coef_cap = c->nmb * 408u;
	c->coefs = calloc(c->coef_cap, 2);
	c->slices = calloc(MAX_SLICES, sizeof(E264SliceRec));
	c->intra_list = calloc(c->nmb, 4);
}

/* ---- drawing one picture ---- */
static int16_t draw_level(int hard) {
	if (!hard || pct(50)) { int v = pct(80) ? rnd(4) : rnd(64); return (int16_t)(pct(50) ? -v : v); }
	if (pct(25)) { int v = pick((const int[]){32767, -32768, -32767, 32766}, 4); cov[v == 32767 ? C_LEVEL_MAX : C_LEVEL_MIN] += v == 32767 || v == -32768; return (int16_t)v; }
	int v = (1 << rnd(15)) + rnd(5) - 2;     /* every power of two, just below and just past it: crosses each overflow threshold */
	return (int16_t)(pct(50) ? -v : v);
}

static void draw_slice(E264SliceRec *s, int n_slots) {
	memset(s, 0, sizeof(*s));
	static const int offs[] = {-12, 12, 0, -6, 6};
	s->filter_offset_a = (int8_t)(pct(50) ? pick(offs, 5) : 2 * (rnd(13) - 6));
	s->filter_offset_b = (int8_t)(pct(50) ? pick(offs, 5) : 2 * (rnd(13) - 6));
	s->deblock_idc = (uint8_t)rnd(3);
	s->slice_type = (uint8_t)rnd(3);
	s->wp_mode = (uint8_t)rnd(3);
	s->luma_log2_wd = (uint8_t)(pct(60) ? pick((const int[]){0, 7}, 2) : rnd(8));
	s->chroma_log2_wd = (uint8_t)(pct(60) ? pick((const int[]){0, 7}, 2) : rnd(8));
	for (int l = 0; l < 2; l++) for (int i = 0; i < 16; i++) for (int k = 0; k < 3; k++) {
		int lwd = k ? s->chroma_log2_wd : s->luma_log2_wd;
		int w = pct(30) ? pick((const int[]){-128, 127, 128, 0, 1}, 5) : pct(50) ? (1 << lwd) : rnd(256) - 128;
		if (lwd == 7 && pct(30)) w = 128;      /* the inferred default at logWD 7 */
		s->wp_w[l][i][k] = (int16_t)w;
		s->wp_o[l][i][k] = (int16_t)(pct(30) ? pick((const int[]){-128, 127, 0}, 3) : rnd(256) - 128);
	}
	if (pct(15)) {   /* conforming explicit bi-prediction at logWD 7 (w0 + w1 = 127, positive offsets): on bright sources the
	                  * weighted sum plus the offset term leaves int16, which the reference saturates (port_recon.c wp_bi) */
		int a = 64 + rnd(64);
		s->wp_mode = WP_EXPLICIT; s->luma_log2_wd = s->chroma_log2_wd = 7;
		for (int l = 0; l < 2; l++) for (int i = 0; i < 16; i++) for (int k = 0; k < 3; k++) {
			s->wp_w[l][i][k] = (int16_t)(l ? 127 - a : a);
			s->wp_o[l][i][k] = (int16_t)(1 + rnd(127));
		}
		cov[C_WP_LWD7_BRIGHT]++;
	}
	for (int i = 0; i < 16; i++) for (int j = 0; j < 16; j++) s->implicit_w1[i][j] = (int16_t)(pct(40) ? pick((const int[]){-64, 128, 32}, 3) : rnd(193) - 64);
	int kind = rnd(4);
	cov[C_SCL_FLAT + kind]++;
	for (int i = 0; i < 96; i++) s->scaling4x4[i >> 4][i & 15] = (uint8_t)(kind == 0 ? 16 : kind == 1 ? 255 : kind == 2 ? 1 : 1 + rnd(255));
	for (int i = 0; i < 128; i++) s->scaling8x8[i >> 6][i & 63] = (uint8_t)(kind == 0 ? 16 : kind == 1 ? 255 : kind == 2 ? 1 : 1 + rnd(255));
	(void)n_slots;
}

/* unavailability bits of 6.4.11.4 for one block (the parser's sx_unavail*), from the neighbours present (A=1 B=2 C=4 D=8) */
static int un4x4(int z, int have) {
	int x = e264_blk_x(z), y = e264_blk_y(z), u = 0;
	if (x == 0 && !(have & 1)) u |= 1;
	if (y == 0 && !(have & 2)) u |= 2;
	if (y == 0) { if (x < 3 ? !(have & 2) : !(have & 4)) u |= 4; }
	else if (x == 3 || e264_blk_z(x + 1, y - 1) > z) u |= 4;
	if (x == 0 && y == 0) { if (!(have & 8)) u |= 8; }
	else if (x == 0) { if (!(have & 1)) u |= 8; }
	else if (y == 0) { if (!(have & 2)) u |= 8; }
	return u;
}
static int un8x8(int i, int have) {
	int u = 0;
	if (!(i & 1) && !(have & 1)) u |= 1;
	if (!(i & 2) && !(have & 2)) u |= 2;
	if (i == 0 ? !(have & 2) : i == 1 ? !(have & 4) : i == 3) u |= 4;
	if (i == 0 ? !(have & 8) : i == 1 ? !(have & 2) : i == 2 ? !(have & 1) : 0) u |= 8;
	return u;
}
static int legal_mode(int kind, int un) {
	int n = (kind == MBK_I4x4 || kind == MBK_I8x8) ? 9 : 4, m;
	do m = rnd(n); while (!e264_intra_mode_legal(kind, m, un));
	intra_seen[kind == -1 ? 3 : kind][m][un]++;
	return IMODE(m, un);
}

static int16_t clamp16(long v) { return (int16_t)(v < -32768 ? -32768 : v > 32767 ? 32767 : v); }

/* a motion vector for 4x4 block b of the macroblock at (mbx, mby) */
static void draw_mv(Ctx *c, int mbx, int mby, int b, int16_t mv[2], const int16_t base[2]) {
	int r = rnd(10);
	if (r == 0) {
		static const int ext[] = {-32768, 32767, -32767, 32764, 0};
		mv[0] = (int16_t)pick(ext, 5); mv[1] = (int16_t)pick(ext, 5); cov[C_MV_INT16]++;
	} else if (r <= 2) {   /* the block lands within 3 samples of a picture border, any fraction */
		int W = c->g.width_mbs * 16, H = c->g.height_mbs * 16;
		int X = mbx * 16 + e264_blk_x(b) * 4, Y = mby * 16 + e264_blk_y(b) * 4;
		int tx = pick((const int[]){-4, 0, W - 4, W}, 4) + rnd(7) - 3, ty = pick((const int[]){-4, 0, H - 4, H}, 4) + rnd(7) - 3;
		if (pct(30)) tx = X; else if (pct(30)) ty = Y;
		mv[0] = clamp16((long)(tx - X) * 4 + rnd(4)); mv[1] = clamp16((long)(ty - Y) * 4 + rnd(4)); cov[C_MV_BORDER]++;
	} else {
		mv[0] = clamp16(base[0] + rnd(17) - 8); mv[1] = clamp16(base[1] + rnd(17) - 8);
	}
}

/* a reference slot other than dst; with pictures in flight, often the slot of the picture submitted just before it */
static int draw_ref(Ctx *c, int dst) {
	if (c->inflight > 1 && c->prev_dst != dst && pct(25)) return c->prev_dst;
	int ref = rnd(c->n_slots - 1);
	return ref >= dst ? ref + 1 : ref;
}

/* the slot of the next picture; with pictures in flight, often one that a picture in flight predicts from */
static int draw_dst(Ctx *c) {
	if (c->inflight > 1 && c->n_out && pct(30)) {
		uint32_t m = 0;
		for (int k = 0; k < c->n_out; k++) m |= c->q[(c->q_head + k) % c->inflight].reads;
		if (m) { int n = rnd(__builtin_popcount(m)); while (n--) m &= m - 1; return __builtin_ctz(m); }
	}
	return rnd(c->n_slots);
}

/* draw the records of one picture into c->recs / coefs / slices; returns n_coefs */
static void draw_picture(Ctx *c, E264PicDesc *pd, int dst, int pcm_content) {
	const int W = c->g.width_mbs, nmb = c->nmb;
	*pd = c->g; pd->dst_slot = dst;
	/* slices: contiguous runs in raster order */
	int n_slices = pcm_content >= 0 ? 1 : pct(10) && nmb >= MAX_SLICES ? MAX_SLICES : 1 + rnd(nmb < 8 ? nmb : 8);
	static _Thread_local int start[MAX_SLICES + 1];
	start[0] = 0;
	for (int i = 1; i < n_slices; i++) start[i] = i;                 /* distinct cut points */
	for (int i = 1; i < n_slices; i++) { int lo = start[i - 1] + 1, hi = nmb - (n_slices - i); start[i] = lo + rnd(hi - lo + 1); }
	start[n_slices] = nmb;
	for (int i = 0; i < n_slices; i++) draw_slice(c->slices + i, c->n_slots);
	if (n_slices == MAX_SLICES) cov[C_SLICES64]++;
	/* which macroblocks are intra: the fraction decides between the intra kernels (recon.cu: rows when n_intra > nmb/2) */
	int fr = rnd(7), n_want;
	n_want = fr == 0 ? 0 : fr == 1 ? 1 : fr == 2 ? nmb / 2 - 1 : fr == 3 ? nmb / 2 : fr == 4 ? nmb / 2 + 1 : fr == 5 ? nmb : rnd(nmb + 1);
	if (pcm_content >= 0) n_want = nmb;
	if (n_want < 0) n_want = 0;
	if (n_want > nmb) n_want = nmb;
	static _Thread_local uint8_t is_intra[1 << 16];
	memset(is_intra, 0, (size_t)nmb);
	for (int k = 0, left = n_want; k < nmb; k++) { if (rnd(nmb - k) < left) { is_intra[k] = 1; left--; } }
	cov[C_FRAC_0] += n_want == 0; cov[C_FRAC_1] += n_want == 1; cov[C_FRAC_ALL] += n_want == nmb && nmb > 2;
	cov[C_FRAC_BELOW] += nmb > 2 && n_want == nmb / 2 - 1; cov[C_FRAC_AT] += nmb > 2 && n_want == nmb / 2; cov[C_FRAC_ABOVE] += nmb > 2 && n_want == nmb / 2 + 1;

	uint32_t n_coefs = 0; int n_intra = 0, any_dbk = 0;
	for (int s = 0, a = 0; s < n_slices; s++) for (; a < start[s + 1]; a++) {
		E264MbRec *r = c->recs + a; const E264SliceRec *sr = c->slices + s;
		const int mbx = a % W, mby = a / W;
		memset(r, 0, sizeof(*r));
		memset(r->ref_idx, -1, sizeof(r->ref_idx)); memset(r->ref_pic, -1, sizeof(r->ref_pic));
		r->slice_idx = (uint8_t)s;
		int have = 0;
		if (mbx > 0 && a - 1 >= start[s]) have |= 1;
		if (mby > 0 && a - W >= start[s]) have |= 2;
		if (mby > 0 && mbx < W - 1 && a - W + 1 >= start[s]) have |= 4;
		if (mby > 0 && mbx > 0 && a - W - 1 >= start[s]) have |= 8;
		int conceal = pcm_content < 0 && pct(4);
		r->qp[0] = (uint8_t)rnd(52); r->qp[1] = h264_qpc[rnd(52)]; r->qp[2] = h264_qpc[rnd(52)];
		if (pct(20)) r->qp[1] = r->qp[2] = 39;
		if (conceal) {   /* the records decoder.c conceal_missing writes: no deblocking, no levels, QP 26 */
			r->qp[0] = r->qp[1] = r->qp[2] = 26; r->coef_off = 0;
			if (is_intra[a]) { r->kind = MBK_I16x16; r->i16_mode = IMODE(2, 11); r->chroma_mode = IMODE(0, 11); cov[C_CONCEAL_INTRA]++; }
			else {
				r->kind = MBK_INTER; r->flags = MBF_SKIP;
				int ref = draw_ref(c, dst);
				for (int i8 = 0; i8 < 4; i8++) { r->ref_idx[0][i8] = 0; r->ref_pic[0][i8] = (int8_t)ref; }
				cov[C_CONCEAL_INTER]++;
			}
		} else {
			if (is_intra[a]) {
				int k = pcm_content >= 0 ? MBK_IPCM : pick((const int[]){MBK_I4x4, MBK_I8x8, MBK_I16x16, MBK_IPCM, MBK_I4x4, MBK_I16x16}, 6);
				r->kind = (uint8_t)k;
				if (k == MBK_I4x4) for (int b = 0; b < 16; b++) r->modes[b] = (uint8_t)legal_mode(k, un4x4(b, have));
				if (k == MBK_I8x8) { r->flags |= MBF_T8x8; for (int i = 0; i < 4; i++) r->modes[i] = (uint8_t)legal_mode(k, un8x8(i, have)); }
				if (k == MBK_I16x16) r->i16_mode = (uint8_t)legal_mode(k, (have & 1 ? 0 : 1) | (have & 2 ? 0 : 2) | (have & 8 ? 0 : 8));
				if (k != MBK_IPCM) r->chroma_mode = (uint8_t)legal_mode(-1, (have & 1 ? 0 : 1) | (have & 2 ? 0 : 2) | (have & 8 ? 0 : 8));
				if (k == MBK_IPCM) { r->qp[0] = 0; cov[C_IPCM]++; }
			} else {
				r->kind = MBK_INTER;
				if (pct(10)) r->flags |= MBF_SKIP;
				if (pct(40)) r->flags |= MBF_T8x8;
				/* a neighbour to copy the motion from (boundary strengths 0/1 and |delta mv| 3 vs 4 need near-equal motion) */
				const E264MbRec *nb = NULL;
				if (pct(50) && mbx > 0 && c->recs[a - 1].kind == MBK_INTER) nb = c->recs + a - 1;
				else if (pct(50) && mby > 0 && c->recs[a - W].kind == MBK_INTER) nb = c->recs + a - W;
				int16_t base[2][2] = {{(int16_t)(rnd(65) - 32), (int16_t)(rnd(65) - 32)}, {(int16_t)(rnd(65) - 32), (int16_t)(rnd(65) - 32)}};
				for (int i8 = 0; i8 < 4; i8++) {
					if (nb && pct(80)) {
						int sw = pct(20);   /* same pictures with the lists swapped */
						for (int l = 0; l < 2; l++) { r->ref_idx[l][i8] = nb->ref_idx[l ^ sw][i8]; r->ref_pic[l][i8] = nb->ref_pic[l ^ sw][i8]; }
						for (int l = 0; l < 2; l++) for (int j = 0; j < 4; j++) memcpy(r->mv[l][i8 * 4 + j], nb->mv[l ^ sw][i8 * 4 + j], 4);
						if (pct(15) && r->ref_idx[0][i8] >= 0 && r->ref_idx[1][i8] >= 0) { int l = rnd(2); r->ref_idx[l][i8] = r->ref_pic[l][i8] = -1; }   /* one list against two */
					} else {
						int use = 1 + rnd(3);
						for (int l = 0; l < 2; l++) if (use >> l & 1) {
							r->ref_idx[l][i8] = (int8_t)rnd(16);
							int ref = draw_ref(c, dst);
							if (l == 1 && use == 3 && pct(30)) ref = r->ref_pic[0][i8];   /* one picture in both lists */
							r->ref_pic[l][i8] = (int8_t)ref;
						}
						for (int l = 0; l < 2; l++) for (int j = 0; j < 4; j++) draw_mv(c, mbx, mby, i8 * 4 + j, r->mv[l][i8 * 4 + j], base[l]);
					}
					for (int l = 0; l < 2; l++) for (int j = 0; j < 4; j++) if (pct(20)) {   /* exactly 3 or 4 apart from the motion it copies */
						int z = i8 * 4 + j, comp = rnd(2), d = pick((const int[]){3, 4, -3, -4}, 4);
						r->mv[l][z][comp] = clamp16(r->mv[l][z][comp] + d);
					}
					for (int l = 0; l < 2; l++) if (r->ref_idx[l][i8] < 0) memset(r->mv[l][i8 * 4], 0, 16);
				}
			}
		}
		/* residual */
		if (!conceal && r->kind != MBK_IPCM) {
			int dens = pct(30) ? 90 : 30, hard = pct(40);
			uint32_t coded = 0;
			if (r->flags & MBF_T8x8) { for (int i8 = 0; i8 < 4; i8++) if (pct(dens)) coded |= 15u << (4 * i8); }
			else for (int b = 0; b < 16; b++) if (pct(dens)) coded |= 1u << b;
			if (r->kind == MBK_I16x16 && pct(70)) coded |= CODED_Y_DC;
			if (pct(dens)) coded |= pct(50) ? CODED_CB_DC : pct(50) ? CODED_CR_DC : CODED_CB_DC | CODED_CR_DC;
			for (int i = 0; i < 8; i++) if (pct(dens / 2)) coded |= CODED_CB_AC(i & 3) << (i & 4);
			r->coded = coded;
			if (coded & 0xffff) qp_seen[0] |= 1ull << r->qp[0];
			if (coded & (CODED_CB_DC | (0xfu << 16))) qp_seen[1] |= 1ull << r->qp[1];
			if (coded & (CODED_CR_DC | (0xfu << 20))) qp_seen[2] |= 1ull << r->qp[2];
			r->coef_off = n_coefs;
			int n = e264_rec_coef_count(r);
			for (int i = 0; i < n; i++) c->coefs[n_coefs + i] = draw_level(hard);
			/* slot 0 of a chroma AC block is unused and zero (records.h) */
			int ac = n - 16 * __builtin_popcount((coded >> 16) & 0xff);
			for (int i = ac; i < n; i += 16) c->coefs[n_coefs + i] = 0;
			n_coefs += n;
		} else if (r->kind == MBK_IPCM) {
			r->coef_off = n_coefs;
			uint8_t *p = (uint8_t *)(c->coefs + n_coefs);
			int kind = pcm_content >= 0 ? pcm_content : rnd(3), v = rnd(256), ph = rnd(3);
			for (int i = 0; i < 384; i++) {
				int x = i < 256 ? i & 15 : i & 7, y = i < 256 ? i >> 4 : (i >> 3) & 7;
				p[i] = (uint8_t)(kind == 0 ? rnd(256) : kind == 1 ? v : ((x + ph) % 3 == 1) == ((y + ph) % 3 == 1) ? 255 : 0);
			}
			n_coefs += 192;
		}
		/* deblocking flags of the slice */
		if (!conceal && sr->deblock_idc != 1) {
			r->flags |= MBF_DEBLOCK; any_dbk = 1;
			if (mbx > 0 && (sr->deblock_idc == 0 || (have & 1))) r->flags |= MBF_EDGE_L;
			if (mby > 0 && (sr->deblock_idc == 0 || (have & 2))) r->flags |= MBF_EDGE_T;
			cov[C_FOFF_M12] += sr->filter_offset_a == -12 || sr->filter_offset_b == -12;
			cov[C_FOFF_P12] += sr->filter_offset_a == 12 || sr->filter_offset_b == 12;
		}
		cov[C_IDC0 + sr->deblock_idc]++;
		if (r->kind != MBK_INTER) c->intra_list[n_intra++] = (uint32_t)a;
	}
	pd->n_slices = n_slices; pd->n_coefs = (int32_t)n_coefs; pd->any_deblock = any_dbk; pd->n_intra = n_intra;
}

/* coverage of the inputs that only the finished picture shows: weights in use, boundary strengths, motion differences */
static void count_picture(Ctx *c) {
	const int W = c->g.width_mbs;
	for (int a = 0; a < c->nmb; a++) {
		const E264MbRec *q = c->recs + a; const E264SliceRec *sr = c->slices + q->slice_idx;
		if (q->kind == MBK_INTER) for (int i8 = 0; i8 < 4; i8++) {
			int u0 = q->ref_idx[0][i8] >= 0, u1 = q->ref_idx[1][i8] >= 0, r0 = q->ref_idx[0][i8] & 15, r1 = q->ref_idx[1][i8] & 15;
			if (sr->wp_mode == WP_EXPLICIT) {
				for (int l = 0; l < 2; l++) if (l ? u1 : u0) {
					int w = sr->wp_w[l][l ? r1 : r0][0], o = sr->wp_o[l][l ? r1 : r0][0];
					cov[C_W_M128] += w == -128; cov[C_W_127] += w == 127; cov[C_O_M128] += o == -128; cov[C_O_127] += o == 127;
					cov[C_W128_UNI_LWD7] += w == 128 && !(u0 && u1) && sr->luma_log2_wd == 7;
				}
				cov[C_LWD0] += sr->luma_log2_wd == 0; cov[C_LWD7] += sr->luma_log2_wd == 7;
			}
			if (sr->wp_mode == WP_IMPLICIT && u0 && u1) { int w1 = sr->implicit_w1[r0][r1]; cov[w1 == -64 ? C_IW_M64 : w1 == 128 ? C_IW_128 : C_IW_OTHER]++; }
			if (u0 && u1 && q->ref_pic[0][i8] == q->ref_pic[1][i8]) cov[C_SAME_BOTH_LISTS]++;
		}
		if (!(q->flags & MBF_DEBLOCK)) continue;
		int t8 = !!(q->flags & MBF_T8x8);
		for (int dir = 0; dir < 2; dir++) for (int e = 0; e < 4; e++) {
			const E264MbRec *p = q;
			if (e == 0) { if (!(q->flags & (dir ? MBF_EDGE_T : MBF_EDGE_L))) continue; p = dir ? q - W : q - 1; }
			if (t8 && (e & 1)) continue;
			for (int k = 0; k < 4; k++) {
				int bq = e264_blk_z(dir ? k : e, dir ? e : k), bp = e264_blk_z(dir ? k : (e ? e - 1 : 3), dir ? (e ? e - 1 : 3) : k);
				int bs = port_boundary_strength(p, bp, q, bq, e == 0);
				cov[C_BS + (e == 0 ? dir : 2) * 10 + t8 * 5 + bs]++;
				if (p->kind != MBK_INTER || q->kind != MBK_INTER) continue;
				int pr[2] = {p->ref_pic[0][bp >> 2], p->ref_pic[1][bp >> 2]}, qr[2] = {q->ref_pic[0][bq >> 2], q->ref_pic[1][bq >> 2]};
				if (pr[0] >= 0 && pr[1] >= 0 && pr[0] != pr[1] && pr[0] == qr[1] && pr[1] == qr[0]) cov[C_SWAPPED]++;
				if ((pr[0] >= 0) + (pr[1] >= 0) != (qr[0] >= 0) + (qr[1] >= 0)) cov[C_ONE_VS_TWO]++;
				for (int l = 0; l < 2; l++) if (pr[l] >= 0 && pr[l] == qr[l]) for (int comp = 0; comp < 2; comp++) {
					int d = abs(p->mv[l][bp][comp] - q->mv[l][bq][comp]);
					if (d == 3) cov[comp ? C_DMV3Y : C_DMV3X]++;
					if (d == 4) cov[comp ? C_DMV4Y : C_DMV4X]++;
				}
			}
		}
	}
	for (int s = 0; s < MAX_SLICES; s++) {   /* one picture at two reference indices with different weights */
		const E264SliceRec *sr = c->slices + s;
		if (sr->wp_mode == WP_EXPLICIT && sr->wp_w[0][0][0] != sr->wp_w[0][1][0]) { cov[C_SAMEPIC_TWO_IDX]++; break; }
	}
}

static void dump_mb(const E264MbRec *recs, const E264SliceRec *slices, int W, int a) {
	const E264MbRec *r = recs + a;
	fprintf(stderr, "  mb %d (%d,%d) kind %d flags %02x qp %d %d %d chroma %02x i16 %02x slice %d coded %08x coef_off %u\n  modes", a, a % W, a / W,
	        r->kind, r->flags, r->qp[0], r->qp[1], r->qp[2], r->chroma_mode, r->i16_mode, r->slice_idx, r->coded, r->coef_off);
	for (int i = 0; i < 16; i++) fprintf(stderr, " %02x", r->modes[i]);
	fprintf(stderr, "\n  ref_idx"); for (int i = 0; i < 8; i++) fprintf(stderr, " %d", ((const int8_t *)r->ref_idx)[i]);
	fprintf(stderr, " ref_pic"); for (int i = 0; i < 8; i++) fprintf(stderr, " %d", ((const int8_t *)r->ref_pic)[i]);
	for (int l = 0; l < 2; l++) { fprintf(stderr, "\n  mv%d", l); for (int i = 0; i < 16; i++) fprintf(stderr, " (%d,%d)", r->mv[l][i][0], r->mv[l][i][1]); }
	const E264SliceRec *s = slices + r->slice_idx;
	fprintf(stderr, "\n  slice: offsets %d %d idc %d wp %d log2_wd %d %d scaling4x4[0][0] %d scaling8x8[0][0] %d\n", s->filter_offset_a, s->filter_offset_b, s->deblock_idc,
	        s->wp_mode, s->luma_log2_wd, s->chroma_log2_wd, s->scaling4x4[0][0], s->scaling8x8[0][0]);
}

/* --dump entries (tests/picture_dumps.py): a tag, then the entry */
enum { DUMP_PICTURE = 1, DUMP_FILL = 2, DUMP_CONFIGURE = 3 };
static void dump_tag(Ctx *c, uint32_t tag) { fwrite(&tag, 4, 1, c->dump); }
/* the geometry and the number of frame slots, at the start of each seed's file */
static void dump_configure(Ctx *c) { int32_t n = c->n_slots; dump_tag(c, DUMP_CONFIGURE); fwrite(&c->g, sizeof(c->g), 1, c->dump); fwrite(&n, 4, 1, c->dump); }
/* a slot set to y on its luma plane and cc after it */
static void dump_fill(Ctx *c, int slot, int y, int cc) { int32_t v[3] = {slot, y, cc}; dump_tag(c, DUMP_FILL); fwrite(v, 4, 3, c->dump); }
/* one picture's description, records, slices, levels, the picture before deblocking and after it */
static void dump_picture(Ctx *c, const E264PicDesc *pd, const E264MbRec *recs, const E264SliceRec *slices, const int16_t *coefs, const uint8_t *post) {
	dump_tag(c, DUMP_PICTURE);
	fwrite(pd, sizeof(*pd), 1, c->dump); fwrite(recs, sizeof(E264MbRec), (size_t)c->nmb, c->dump);
	fwrite(slices, sizeof(E264SliceRec), (size_t)pd->n_slices, c->dump); fwrite(coefs, 2, (size_t)pd->n_coefs, c->dump);
	fwrite(c->dump_pre, 1, (size_t)pd->frame_bytes, c->dump); fwrite(post, 1, (size_t)pd->frame_bytes, c->dump);
}

/* --dump: the picture before deblocking, reconstructed from the records with the deblocking flags cleared (a picture the
 * record contract allows), by the port or the device, into c->dump_pre */
static void reconstruct_pre(Ctx *c, const E264PicDesc *pd, int cpu_only) {
	E264PicDesc p0 = *pd; p0.any_deblock = 0;
	memcpy(c->dump_recs, c->recs, (size_t)c->nmb * sizeof(E264MbRec));
	for (int a = 0; a < c->nmb; a++) c->dump_recs[a].flags &= (uint8_t)~(MBF_DEBLOCK | MBF_EDGE_L | MBF_EDGE_T);
	if (cpu_only) {
		pthread_mutex_lock(&port_mu);
		long res[6], sat = port_cov_wp_bi_sat16;     /* the port's counters count the picture once */
		memcpy(res, port_cov_residual, sizeof(res));
		port_recon_picture(c->port_frames, &p0, c->dump_recs, c->coefs, c->slices);
		memcpy(port_cov_residual, res, sizeof(res)); port_cov_wp_bi_sat16 = sat;
		pthread_mutex_unlock(&port_mu);
		memcpy(c->dump_pre, c->port_frames + (size_t)pd->dst_slot * c->g.frame_bytes, (size_t)c->g.frame_bytes);
		return;
	}
	E264Staging st; uint64_t t;
	if (D.acquire(c->dev, p0.dst_slot, &st)) { fprintf(stderr, "acquire_staging failed\n"); exit(3); }
	memcpy(st.recs, c->dump_recs, (size_t)c->nmb * sizeof(E264MbRec));
	memcpy(st.coefs, c->coefs, (size_t)p0.n_coefs * 2);
	memcpy(st.slices, c->slices, (size_t)p0.n_slices * sizeof(E264SliceRec));
	memcpy(st.intra_list, c->intra_list, (size_t)p0.n_intra * 4);
	p0.staging = st.handle;
	if (D.submit(c->dev, &p0, c->dump_dev, &t) || D.wait(c->dev, t)) { fprintf(stderr, "submit of the picture before deblocking failed\n"); exit(3); }
	memcpy(c->dump_pre, c->dump_dev, (size_t)c->g.frame_bytes);
}

/* wait for the oldest picture in flight and compare it with the port's frame of the same picture; returns 0 when they agree */
static int retire(Ctx *c, int cpu_only) {
	Pending *p = c->q + c->q_head;
	c->q_head = (c->q_head + 1) % c->inflight; c->n_out--;
	if (cpu_only) return 0;
	if (D.wait(c->dev, p->ticket)) { fprintf(stderr, "picture %d: wait failed\n", p->pic); return 1; }
	if (c->dump) dump_picture(c, &p->pd, p->recs, p->slices, p->coefs, p->host_out);   /* before the comparison: a picture that fails it is judged too */
	const int W = c->g.width_mbs, H = c->g.height_mbs;
	for (int pl = 0; pl < 3; pl++) {
		int w = pl ? W * 8 : W * 16, h = pl ? H * 8 : H * 16, stride = pl ? c->g.stride_c : c->g.stride_y;
		size_t base = pl == 0 ? 0 : (size_t)c->g.plane_y + (pl == 2 ? c->g.stride_c / 2 : 0);
		for (int y = 0; y < h; y++) for (int x = 0; x < w; x++) {
			size_t o = base + (size_t)y * stride + x;
			if (p->host_out[o] == p->port[o]) continue;
			int a = (y / (pl ? 8 : 16)) * W + x / (pl ? 8 : 16);
			fprintf(stderr, "MISMATCH picture %d (slot %d, %dx%d macroblocks, %d intra) plane %d x %d y %d: device %d port %d\n", p->pic, p->dst, W, H, p->pd.n_intra, pl, x, y, p->host_out[o], p->port[o]);
			dump_mb(p->recs, p->slices, W, a);
			return 1;
		}
	}
	return 0;
}

/* submit every picture drawn since the last comparison, back to back so that the device is still working on the earlier
 * ones (the port is far slower than the device: a picture submitted on its own is finished before the next is drawn),
 * then compare them in order; returns 0 while the device agrees with the port */
static int flush(Ctx *c, int cpu_only) {
	for (int k = 0; k < c->n_out && !cpu_only; k++) {
		Pending *p = c->q + (c->q_head + k) % c->inflight;
		E264Staging st;
		if (D.acquire(c->dev, p->dst, &st)) { fprintf(stderr, "acquire_staging failed\n"); exit(3); }
		memcpy(st.recs, p->recs, (size_t)c->nmb * sizeof(E264MbRec));
		memcpy(st.coefs, p->coefs, (size_t)p->pd.n_coefs * 2);
		memcpy(st.slices, p->slices, (size_t)p->pd.n_slices * sizeof(E264SliceRec));
		memcpy(st.intra_list, p->intra_list, (size_t)p->pd.n_intra * 4);
		p->pd.staging = st.handle;
		if (D.submit(c->dev, &p->pd, p->host_out, &p->ticket)) { fprintf(stderr, "picture %d: submit failed\n", p->pic); exit(3); }
	}
	int bad = 0;
	while (c->n_out && !bad) bad = retire(c, cpu_only);
	return bad;
}

/* one picture: drawn and reconstructed on the port at once, in draw order; it goes to the device with the pictures drawn
 * before it once c->inflight pictures are waiting.  Returns 0 while the device agrees with the port */
static int run_picture(Ctx *c, int pic, int dst, int pcm_content, int cpu_only) {
	E264PicDesc pd;
	draw_picture(c, &pd, dst, pcm_content);
	char why[256];
	if (e264_check_records(&pd, c->recs, c->coefs, c->slices, c->intra_list, c->n_slots, why, sizeof(why))) {
		fprintf(stderr, "generator broke the record contract, picture %d: %s\n", pic, why);
		exit(2);
	}
	count_picture(c);
	cov[C_PICTURES]++;
	uint32_t reads = 0;
	for (int a = 0; a < c->nmb; a++) if (c->recs[a].kind == MBK_INTER)
		for (int l = 0; l < 2; l++) for (int i8 = 0; i8 < 4; i8++) if (c->recs[a].ref_idx[l][i8] >= 0) reads |= 1u << c->recs[a].ref_pic[l][i8];
	if (c->inflight > 1) {   /* what this picture shares with the pictures in flight when it is submitted, and whether the staging ring is full */
		int ref_in = 0, dst_in = 0;
		for (int k = 0; k < c->n_out; k++) { const Pending *o = c->q + (c->q_head + k) % c->inflight; ref_in |= reads >> o->dst & 1; dst_in |= o->reads >> dst & 1; }
		cov[C_REF_IN_FLIGHT] += ref_in; cov[C_DST_READ_IN_FLIGHT] += dst_in; cov[C_STAGING_WRAPPED] += c->n_out >= c->n_stage;
	}
	if (c->dump) reconstruct_pre(c, &pd, cpu_only);
	pthread_mutex_lock(&port_mu);
	port_recon_picture(c->port_frames, &pd, c->recs, c->coefs, c->slices);
	pthread_mutex_unlock(&port_mu);
	if (c->dump && cpu_only) dump_picture(c, &pd, c->recs, c->slices, c->coefs, c->port_frames + (size_t)dst * c->g.frame_bytes);
	Pending *p = c->q + (c->q_head + c->n_out) % c->inflight;
	p->pic = pic; p->dst = dst; p->reads = reads; p->pd = pd;
	if (++c->n_out > cov[C_INFLIGHT_MAX]) cov[C_INFLIGHT_MAX] = c->n_out;
	if (c->inflight > 1) c->prev_dst = dst;
	if (!cpu_only) {
		memcpy(p->port, c->port_frames + (size_t)dst * c->g.frame_bytes, (size_t)c->g.frame_bytes);
		memcpy(p->recs, c->recs, (size_t)c->nmb * sizeof(E264MbRec));
		memcpy(p->coefs, c->coefs, (size_t)pd.n_coefs * 2);
		memcpy(p->slices, c->slices, (size_t)pd.n_slices * sizeof(E264SliceRec));
		memcpy(p->intra_list, c->intra_list, (size_t)pd.n_intra * 4);
	}
	return c->n_out == c->inflight ? flush(c, cpu_only) : 0;
}

/* ---- one host thread per context: seeds first + k * step, one after the other, each on a context from e264b_create ---- */
static const int geoms[][2] = {{1, 1}, {1, 9}, {9, 1}, {63, 2}, {64, 3}, {65, 2}, {129, 2}, {3, 7}, {4, 8}, {2, 9},
                               {3, 15}, {2, 16}, {3, 17}, {2, 33}, {120, 68}, {256, 2}, {5, 4}, {7, 6}};
typedef struct {
	int first, last, step, cpu_only, pictures, gw, gh, inflight;   /* in */
	int total, fails;                                             /* out */
} Job;
static struct {   /* every context's counters, summed as its thread ends */
	pthread_mutex_t mu; long cov[C_N]; uint64_t qp_seen[3]; uint8_t intra_seen[4][9][16];
} all = {PTHREAD_MUTEX_INITIALIZER};

static void *run_context(void *arg) {
	Job *j = (Job *)arg;
	const int n_geoms = sizeof(geoms) / sizeof(geoms[0]), K = j->inflight, cpu_only = j->cpu_only;
	for (int seed = j->first; seed <= j->last; seed += j->step) {
		rng = 0x9E3779B97F4A7C15ull * (uint64_t)(seed + 1) ^ 0xD1B54A32D192ED03ull;
		int W = j->gw ? j->gw : geoms[seed % n_geoms][0], H = j->gh ? j->gh : geoms[seed % n_geoms][1];
		Ctx c; memset(&c, 0, sizeof(c));
		geometry(&c, W, H, 2 + rnd(MAX_SLOTS - 1));
		c.inflight = K;
		if (K > 1) {   /* often fewer staging areas than pictures in flight: e264b_acquire_staging then waits for the oldest */
			c.g.staging = pct(50) ? K : 2 + rnd(K - 1);
			c.n_stage = c.g.staging < FUZZ_NSTAGE ? c.g.staging : FUZZ_NSTAGE;
		}
		int n_pics = j->pictures ? j->pictures : W * H >= 4096 ? 3 : W * H >= 100 ? 12 : 24;
		if (K > 1 && !j->pictures) n_pics += 2 * K;
		c.q = calloc(K, sizeof(Pending));
		if (dump_dir) {
			char path[4096]; snprintf(path, sizeof(path), "%s/seed_%d.bin", dump_dir, seed);
			if (!(c.dump = fopen(path, "wb"))) { fprintf(stderr, "cannot write %s\n", path); exit(3); }
			c.dump_recs = malloc((size_t)c.nmb * sizeof(E264MbRec)); c.dump_pre = malloc(c.g.frame_bytes);
		}
		if (!cpu_only) {
			if (D.create(&c.dev)) { fprintf(stderr, "e264b_create failed\n"); exit(3); }
			if (D.configure(c.dev, &c.g, c.n_slots)) { fprintf(stderr, "e264b_configure failed\n"); exit(3); }
			for (int k = 0; k < K; k++) {
				Pending *p = c.q + k;
				p->host_out = D.host_alloc(c.dev, c.g.frame_bytes); p->port = malloc(c.g.frame_bytes);
				p->recs = malloc((size_t)c.nmb * sizeof(E264MbRec)); p->coefs = malloc((size_t)c.coef_cap * 2);
				p->slices = malloc(MAX_SLICES * sizeof(E264SliceRec)); p->intra_list = malloc((size_t)c.nmb * 4);
				if (!p->host_out || !p->port || !p->recs || !p->coefs || !p->slices || !p->intra_list) { fprintf(stderr, "out of memory\n"); exit(3); }
			}
			if (c.dump) c.dump_dev = D.host_alloc(c.dev, c.g.frame_bytes);
		}
		if (c.dump) dump_configure(&c);
		for (int s = 0; s < c.n_slots; s++) {   /* every slot starts identical on both sides */
			int y = rnd(256), cc = rnd(256);
			uint8_t *f = c.port_frames + (size_t)s * c.g.frame_bytes;
			memset(f, y, c.g.plane_y); memset(f + c.g.plane_y, cc, c.g.frame_bytes - c.g.plane_y);
			if (!cpu_only) D.fill(c.dev, s, y, cc);
			if (c.dump) dump_fill(&c, s, y, cc);
		}
		int bad = 0, first_pic = j->total;
		for (int s = 0; s < c.n_slots && !bad; s++) bad = run_picture(&c, j->total++, s, s % 3, cpu_only);   /* textured references */
		for (int p = 0; p < n_pics && !bad; p++) bad = run_picture(&c, j->total++, draw_dst(&c), -1, cpu_only);
		if (c.n_out && !bad) bad = flush(&c, cpu_only);
		if (!cpu_only && c.n_out) D.wait(c.dev, c.q[(c.q_head + c.n_out - 1) % K].ticket);   /* after a mismatch: nothing left writing into host_out */
		if (!cpu_only && !bad && D.error_flag(c.dev)) { fprintf(stderr, "device error word %d\n", D.error_flag(c.dev)); bad = 1; }
		if (bad) { fprintf(stderr, "seed %d (%dx%d, %d slots, pictures %d-%d, %d in flight, %d staging) failed\n", seed, W, H, c.n_slots, first_pic, j->total - 1, K, c.n_stage); j->fails++; }
		if (!cpu_only) {
			for (int k = 0; k < K; k++) { Pending *p = c.q + k; D.host_free(c.dev, p->host_out); free(p->port); free(p->recs); free(p->coefs); free(p->slices); free(p->intra_list); }
			if (c.dump) D.host_free(c.dev, c.dump_dev);
			D.destroy(c.dev);
		}
		if (c.dump) { fclose(c.dump); free(c.dump_recs); free(c.dump_pre); }
		free(c.q); free(c.port_alloc); free(c.recs); free(c.coefs); free(c.slices); free(c.intra_list);
	}
	pthread_mutex_lock(&all.mu);
	for (int i = 0; i < C_N; i++) all.cov[i] = i == C_INFLIGHT_MAX ? (cov[i] > all.cov[i] ? cov[i] : all.cov[i]) : all.cov[i] + cov[i];
	for (int i = 0; i < 3; i++) all.qp_seen[i] |= qp_seen[i];
	for (int k = 0; k < 4; k++) for (int m = 0; m < 9; m++) for (int u = 0; u < 16; u++) all.intra_seen[k][m][u] |= intra_seen[k][m][u];
	pthread_mutex_unlock(&all.mu);
	return NULL;
}

int main(int argc, char **argv) {
	int cpu_only = 0, s0 = 1, s1 = 1, pictures = 0, gw = 0, gh = 0, M = 1, K = 1;
	const char *lib = NULL;
	for (int i = 1; i < argc; i++) {
		if (!strcmp(argv[i], "--cpu-only")) cpu_only = 1;
		else if (!strcmp(argv[i], "--lib") && i + 1 < argc) lib = argv[++i];
		else if (!strcmp(argv[i], "--seeds") && i + 1 < argc) { if (sscanf(argv[++i], "%d-%d", &s0, &s1) == 1) s1 = s0; }
		else if (!strcmp(argv[i], "--pictures") && i + 1 < argc) pictures = atoi(argv[++i]);
		else if (!strcmp(argv[i], "--geom") && i + 1 < argc) sscanf(argv[++i], "%dx%d", &gw, &gh);
		else if (!strcmp(argv[i], "--contexts") && i + 1 < argc) M = atoi(argv[++i]);
		else if (!strcmp(argv[i], "--inflight") && i + 1 < argc) K = atoi(argv[++i]);
		else if (!strcmp(argv[i], "--dump") && i + 1 < argc) dump_dir = argv[++i];
		else { fprintf(stderr, "usage: %s [--cpu-only] [--lib path] [--seeds A-B] [--pictures N] [--geom WxH] [--contexts M] [--inflight K] [--dump DIR]\n", argv[0]); return 2; }
	}
	if (dump_dir && K != 1) { fprintf(stderr, "--dump takes one picture in flight\n"); return 2; }
	if (M < 1 || K < 1 || s1 < s0) { fprintf(stderr, "--contexts and --inflight take at least 1, --seeds A-B needs A <= B\n"); return 2; }
	if (M > s1 - s0 + 1) M = s1 - s0 + 1;
	if (!cpu_only) { if (!lib) { fprintf(stderr, "--lib is needed without --cpu-only\n"); return 2; } load_device(lib); }
	/* widths around INTER_CHUNK (64) and the row-above staging, heights around IR_ROWS / DBK_PAIRS bands, 1-wide pictures,
	 * 4096-sample strides, 1080p: the list geoms above, seed k takes geometry k % 18 */
	Job *jobs = calloc(M, sizeof(Job));
	pthread_t *th = calloc(M, sizeof(pthread_t));
	for (int t = 0; t < M; t++) {
		jobs[t] = (Job){s0 + t, s1, M, cpu_only, pictures, gw, gh, K, 0, 0};
		if (pthread_create(th + t, NULL, run_context, jobs + t)) { fprintf(stderr, "pthread_create failed\n"); return 3; }
	}
	int fails = 0, total = 0;
	for (int t = 0; t < M; t++) { pthread_join(th[t], NULL); fails += jobs[t].fails; total += jobs[t].total; }
	const int concurrent = M > 1 || K > 1;
	if (concurrent) for (int t = 0; t < M; t++) printf("context %d: %d pictures, %d failing seeds\n", t, jobs[t].total, jobs[t].fails);
	all.cov[C_CONTEXTS] = M;
	int combos = 0;
	for (int k = 0; k < 4; k++) for (int m = 0; m < 9; m++) for (int u = 0; u < 16; u++) combos += all.intra_seen[k][m][u] != 0;
	all.cov[C_INTRA_COMBOS] = combos;
	all.cov[C_QPY] = __builtin_popcountll(all.qp_seen[0]); all.cov[C_QPCB] = __builtin_popcountll(all.qp_seen[1]); all.cov[C_QPCR] = __builtin_popcountll(all.qp_seen[2]);
	static const char *names[C_N] = {"qp_y_values", "qp_cb_values", "qp_cr_values", "level_32767", "level_-32768", "scaling_flat16", "scaling_all255",
		"scaling_all1", "scaling_random", "weight_-128", "weight_127", "weight_128_uni_logwd7", "offset_-128", "offset_127", "explicit_logwd0",
		"explicit_logwd7", "implicit_w1_-64", "implicit_w1_128", "implicit_w1_other", "one_picture_two_weights", "mv_int16_extreme", "mv_near_border",
		"dmv_x_3", "dmv_x_4", "dmv_y_3", "dmv_y_4", "same_picture_both_lists", "swapped_lists", "one_list_vs_two"};
	for (int i = 0; i <= C_PICTURES; i++) {
		if (i >= C_BS && i < C_BS + 30) {
			int e = (i - C_BS) / 10, bs = (i - C_BS) % 5;
			if ((e < 2 && bs == 3) || (e == 2 && bs == 4)) continue;   /* macroblock edges take 4 where internal edges take 3 */
			printf("cov %s %ld\n", bs_name(i - C_BS), all.cov[i]);
			continue;
		}
		if (i >= C_BS + 30 && i < C_FOFF_M12) continue;
		static const char *tail[] = {"filter_offset_-12", "filter_offset_12", "deblock_idc_0", "deblock_idc_1", "deblock_idc_2", "slices_64",
			"intra_mode_availability_pairs", "ipcm", "conceal_inter", "conceal_intra", "intra_fraction_0", "intra_fraction_1",
			"intra_fraction_below_half", "intra_fraction_half", "intra_fraction_above_half", "intra_fraction_all", "explicit_bi_logwd7_bright", "pictures"};
		printf("cov %s %ld\n", i < C_BS ? names[i] : tail[i - C_FOFF_M12], all.cov[i]);
	}
	static const char *res[6] = {"sat16_4x4", "wrap_8x8_div_lt6", "wrap_8x8_div_ge6", "wrap_luma_dc32", "chroma_dc_qpc39", "wrap16_dc_only"};
	for (int i = 0; i < 6; i++) printf("cov %s %ld\n", res[i], port_cov_residual[i]);
	printf("cov wp_bi_sat16 %ld\n", port_cov_wp_bi_sat16);
	if (concurrent) {
		static const char *inflight_names[] = {"inflight_max", "ref_slot_in_flight", "dst_slot_read_in_flight", "staging_wrapped", "contexts"};
		for (int i = C_INFLIGHT_MAX; i < C_N; i++) printf("cov %s %ld\n", inflight_names[i - C_INFLIGHT_MAX], all.cov[i]);
	}
	printf("%d pictures, %d failing seeds\n", total, fails);
	return fails ? 1 : 0;
}
