/* gen264 — synthetic H.264 Annex-B stream generator (TEST / BENCH INFRASTRUCTURE, not product).
 *
 * Plays the role tests/gen_avc.py plays for the reference (YAML -> .264, CAVLC only), but is
 * self-contained and fast enough for 1080p..8K CABAC IPB streams: it draws random syntax
 * (macroblock types, prediction modes, motion vectors, coefficients) from a seeded PRNG and writes
 * it through the WRITER direction of the shared slice-data code (edge264_b200/csrc/syntax_impl.h,
 * mb_impl.h compiled with -DE264_ENCODER).  Every stream it produces is first checked against the
 * compiled reference decoder (tests/, oracle/_ref) — that decoder, not this tool, is the judge of
 * what the bitstream means.
 *
 *   gen264 -o out.264 [-W mbs] [-H mbs] [-n frames] [-s seed] [--cavlc] [--gop I|IP|IPB] [--idr N]
 *          [--refs N] [--t8x8 pct] [--scaling 0|1|2] [--wp 0|1|2] [--slices N] [--deblock 0|1|2]
 *          [--deblock-off nonref|all]       (disable_deblocking_filter_idc = 1 in the slices of the non-reference / all
 *                                           pictures; every other bit of the stream, slice data included, is the one
 *                                           written without the option: the twin of a decode that skips the loop filter,
 *                                           include/edge264_loopfilter.h)
 *          [--density pct] [--qp Q] [--temporal] [--pcm permille] [--crop-bottom px] [--level idc]
 *          [--mvrange qpel] [--intra-pct P] [--skip-pct P]
 *          [--no-vui]                       (no VUI in the SPS: the decoder infers max_num_reorder_frames and
 *                                           max_dec_frame_buffering from the level, the case of many cameras)
 *          [--reorder N]                    (max_num_reorder_frames N in the VUI bitstream_restriction, every other value
 *                                           as without the option; with --no-vui, a VUI holding only bitstream_restriction
 *                                           that states the values inferred from the level, with reorder N.  Every other
 *                                           bit of the stream is the one written without the option: the twin of a decode
 *                                           with edge264_set_output_latency(N), include/edge264_latency.h)
 *          [--crop-left px] [--crop-right px] [--crop-top px]   (even numbers; with --crop-bottom: frame cropping rectangle)
 *          [--direct4x4]                    (direct_8x8_inference_flag = 0: direct prediction per 4x4 block)
 *          [--nonref-p]                     (with --gop IP: some P pictures are not used for reference)
 *          [--extra-nals]                   (access unit delimiters, SEI and filler data NAL units between pictures)
 *          [--bref]                         (with --gop IPB: the first B picture of each pair is a reference picture)
 *          [--i-period N]                   (with --gop IP / IPB: a non-IDR I picture in place of the next P anchor once
 *                                           N pictures have been coded since the last I or IDR picture; the pictures
 *                                           after it may still predict from pictures before it: open GOP)
 *          [--mixed-slices]                 (slices of one picture take different slice types)
 *          [--ps-update]                    (picture parameter sets re-sent with new chroma QP offsets, and the unchanged
 *                                            sequence parameter set repeated, between pictures)
 *          [--dpb] [--mmco5] [--poc-type 0|1|2]  (with --gop IP / IPB: reference-list modification to short- and long-term
 *                                           pictures, memory-management operations 1,2,3,4,6, long-term IDR,
 *                                           4-bit frame_num wrap-around; picture order count types 1 and 2)
 *   the standard's limits (tests/test_limits.py; none of these changes a stream written without them):
 *          [--wp-range full]                (explicit weights over -128..127 with both ends forced now and then, offsets over
 *                                            -128..127, logWD 0..7; B pairs at -128 <= w0 + w1 <= (logWD 7 ? 127 : 128))
 *          [--qp-walk]                      (mb_qp_delta over -26..25, QP_Y wrapping modulo 52 both ways, slice QPs 0 and 51)
 *          [--cqp-offset A,B]               (chroma_qp_index_offset A and second_chroma_qp_index_offset B in every PPS)
 *          [--levels big]                   (levels up to the 8-bit bound -32768..32767: CAVLC escapes, long CABAC suffixes)
 *          [--pcm-extreme]                  (PCM macroblocks with 0/255 steps, full-range ramps, checkers and random bits)
 *   stereo (include/edge264_mvc.h):
 *          [--mvc [seed]]                   (a second view: a subset SPS (Stereo High) after every SPS, a prefix NAL unit before
 *                                            every base view slice and the second view's slices (NAL unit 20) after the base
 *                                            view's.  Anchor access units (I or IDR base view) code a P second view predicted
 *                                            from the base view only; the others a P or B second view whose random reference
 *                                            choices draw the inter-view reference too.  With --dpb the second view takes list
 *                                            modifications, idc 4 and 5 included, and memory-management operations.  Base views
 *                                            with nal_ref_idc 0 carry inter_view_flag 1 or 0, and in the latter case their second
 *                                            view does not predict from them.  The second view draws from its own generator
 *                                            seeded by `seed`, so the base view's NAL units are those written without --mvc.)
 */
#define E264_ENCODER
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../edge264_b200/csrc/mb_impl.h"

typedef struct GenPic {
	int used, frame_num, poc; int32_t uid;
	int is_long, long_idx;   /* --dpb: long-term reference and its LongTermFrameIdx */
	E264MbRec *recs; int32_t slot_uid[E264_MAX_SLOTS];
} GenPic;

typedef struct GenState {
	uint64_t rng;
	int W, H, frames, cabac, gop, idr_period, refs, t8x8_pct, scaling, wp, slices, deblock, density, qp0, temporal, pcm_pm, crop_bottom, level, mvrange, intra_pct, skip_pct;
	GenPic *dpb;            /* the pictures of the view being coded: views[0] or, with --mvc, views[1] */
	GenPic views[2][E264_MAX_SLOTS];
	int mvc, view;          /* --mvc: a second view is written; the view being coded */
	uint64_t rng_view;      /* --mvc: the generator of the view not being coded */
	int max_long_view;      /* --mvc: max_long_idx_plus1 of the view not being coded */
	const GenPic *base;     /* --mvc: the base view picture of the access unit, the second view's inter-view reference */
	int base_inter_view;    /* --mvc: inter_view_flag of that base view picture */
	int au_anchor;          /* the access unit is an anchor (its base view is an I or IDR picture) */
	GenPic *last_pic;       /* the picture encode_picture coded last */
	int32_t next_uid;
	MbInfo *mbi; int16_t *pool;
	int t8x8_mode;          /* PPS transform_8x8_mode_flag */
	int pcm_checker;
	int wp_p, wp_b;         /* weighted_pred_flag, weighted_bipred_idc */
	int log2_max_frame_num, log2_max_poc_lsb;
	int drift[2];           /* per-picture global motion */
	int cur_is_b;
	int i_period;
	int deblock_off;        /* --deblock-off: 0 none, 1 non-reference pictures, 2 all pictures */
	int no_vui, reorder;    /* --no-vui; --reorder N (-1 without it) */
	int direct4x4, nonref_p, extra_nals, bref, crop_left, crop_right, crop_top, mixed, ps_update, dpb_mode, mmco5, poc_type, max_long_idx_plus1, stat_rplm, stat_mmco[7], stat_idr_long;   /* --dpb: list modification + memory-management stress on I P P P streams; --poc-type 0|1|2 */
	int wp_full, qp_walk, cqp_fixed, cqp[2], levels_big, pcm_extreme;   /* the standard's limits (file header) */
} GenState;

static inline uint64_t rnd64(GenState *g) { uint64_t x = g->rng; x ^= x >> 12; x ^= x << 25; x ^= x >> 27; g->rng = x; return x * 0x2545F4914F6CDD1Dull; }
static inline int rnd(GenState *g, int n) { return (int)((rnd64(g) >> 33) % (uint64_t)n); }
static inline int pct(GenState *g, int p) { return rnd(g, 100) < p; }
/* two-sided geometric ("Laplacian") with mean magnitude ~ scale */
static int laplace(GenState *g, int scale) {
	int m = 0;
	while (m < 16 * scale && rnd(g, scale + 1) != 0) m++;
	return rnd(g, 2) ? -m : m;
}

/* ------------------------------------------------------------------------------------------ */
/* headers                                                                                      */
/* ------------------------------------------------------------------------------------------ */
static void put_scaling_list(GenState *g, BitWriter *w, int n, int kind) {
	/* kind 0: random explicit list, 1: useDefaultScalingMatrixFlag (first delta -> 0), 2: short list ending with nextScale == 0 */
	int last = 8;
	if (kind == 1) { bw_se(w, -8); return; }
	for (int j = 0; j < n; j++) {
		int next;
		if (kind == 2 && j == n / 2) { bw_se(w, -last); return; }   /* nextScale = 0: rest repeats lastScale */
		next = 1 + rnd(g, j == 0 ? 40 : 80);
		if (j > 0) { next = last + rnd(g, 13) - 6; if (next < 1) next = 1; if (next > 255) next = 255; }
		int delta = next - last; if (delta > 127) delta -= 256; if (delta < -128) delta += 256;
		bw_se(w, delta); last = next;
	}
}
static void put_scaling_matrix(GenState *g, BitWriter *w, int n_lists) {
	for (int i = 0; i < n_lists; i++) {
		int r = rnd(g, 10);
		if (r < 3) { bw_u(w, 1, 0); continue; }             /* not present: fall-back rule */
		bw_u(w, 1, 1);
		put_scaling_list(g, w, i < 6 ? 16 : 64, r == 3 ? 1 : r == 4 ? 2 : 0);
	}
}

/* MaxDpbFrames (A.3.1 h, Table A-1): what a decoder infers without bitstream_restriction */
static int max_dpb_frames(int level, int mbs) {
	const int max_dpb_mbs = level <= 10 || level == 9 ? 396 : level == 11 ? 900 : level <= 20 ? 2376 : level == 21 ? 4752 : level <= 30 ? 8100 :
	                        level == 31 ? 18000 : level == 32 ? 20480 : level <= 41 ? 32768 : level == 42 ? 34816 : level == 50 ? 110400 :
	                        level <= 52 ? 184320 : 696320;
	return max_dpb_mbs / mbs < 16 ? max_dpb_mbs / mbs : 16;
}

/* subset: the subset SPS of --mvc (NAL unit 15, Stereo High, two views whose second predicts from the first) */
static void write_sps(GenState *g, ByteBuf *out, int subset) {
	BitWriter w; bw_init(&w, 4096);
	bw_u(&w, 8, subset ? 128 : 100); bw_u(&w, 8, 0); bw_u(&w, 8, g->level);
	bw_ue(&w, 0);
	bw_ue(&w, 1); bw_ue(&w, 0); bw_ue(&w, 0); bw_u(&w, 1, 0);
	bw_u(&w, 1, g->scaling == 1 || g->scaling == 3);
	if (g->scaling == 1 || g->scaling == 3) put_scaling_matrix(g, &w, 8);
	bw_ue(&w, g->log2_max_frame_num - 4);
	bw_ue(&w, g->poc_type);
	if (g->poc_type == 0) bw_ue(&w, g->log2_max_poc_lsb - 4);
	else if (g->poc_type == 1) { bw_u(&w, 1, 1); bw_se(&w, 0); bw_se(&w, 0); bw_ue(&w, 1); bw_se(&w, 2); }   /* delta_pic_order_always_zero, offsets 0, one ref frame per cycle, +2 per frame */
	bw_ue(&w, g->refs);
	bw_u(&w, 1, 0);
	bw_ue(&w, g->W - 1); bw_ue(&w, g->H - 1);
	bw_u(&w, 1, 1);                      /* frame_mbs_only_flag */
	bw_u(&w, 1, !g->direct4x4);          /* direct_8x8_inference_flag */
	const int any_crop = g->crop_bottom > 0 || g->crop_left > 0 || g->crop_right > 0 || g->crop_top > 0;
	bw_u(&w, 1, any_crop);
	if (any_crop) { bw_ue(&w, g->crop_left / 2); bw_ue(&w, g->crop_right / 2); bw_ue(&w, g->crop_top / 2); bw_ue(&w, g->crop_bottom / 2); }
	const int vui = !g->no_vui || g->reorder >= 0;
	bw_u(&w, 1, vui);                    /* vui_parameters_present_flag: only bitstream_restriction */
	if (vui) {
		bw_u(&w, 1, 0); bw_u(&w, 1, 0); bw_u(&w, 1, 0); bw_u(&w, 1, 0); bw_u(&w, 1, 0); bw_u(&w, 1, 0); bw_u(&w, 1, 0); bw_u(&w, 1, 0);
		bw_u(&w, 1, 1);
		bw_u(&w, 1, 1); bw_ue(&w, 0); bw_ue(&w, 0); bw_ue(&w, 16); bw_ue(&w, 16);
		bw_ue(&w, g->reorder >= 0 ? g->reorder : g->gop == 2 ? 1 : 0);                      /* max_num_reorder_frames */
		bw_ue(&w, g->no_vui ? max_dpb_frames(g->level, g->W * g->H) : g->refs + (g->gop == 2));   /* max_dec_frame_buffering */
	}
	if (subset) {
		bw_u(&w, 1, 1);                      /* bit_equal_to_one */
		bw_ue(&w, 1); bw_ue(&w, 0); bw_ue(&w, 1);   /* num_views_minus1, view_id 0 and 1 */
		bw_ue(&w, 1); bw_ue(&w, 0); bw_ue(&w, 0);   /* anchor: l0 holds view 0, l1 nothing */
		bw_ue(&w, 1); bw_ue(&w, 0); bw_ue(&w, 1); bw_ue(&w, 0);   /* non-anchor: view 0 in l0 and l1 */
		bw_ue(&w, 0); bw_u(&w, 8, g->level); bw_ue(&w, 0); bw_u(&w, 3, 0); bw_ue(&w, 1); bw_ue(&w, 0); bw_ue(&w, 1); bw_ue(&w, 1);   /* one level, one operation point: both views */
		bw_u(&w, 1, 0);                      /* mvc_vui_parameters_present_flag */
		bw_u(&w, 1, 0);                      /* additional_extension2_flag */
	}
	bw_trailing(&w);
	e264_emit_nal(out, 3, subset ? 15 : 7, w.buf, w.pos / 8); free(w.buf);
	if (g->mvc && !subset) {   /* its scaling lists are drawn from the second view's generator, which the base view never reads */
		uint64_t r = g->rng; g->rng = g->rng_view; g->rng_view = r;
		write_sps(g, out, 1);
		r = g->rng; g->rng = g->rng_view; g->rng_view = r;
	}
}
static void write_pps(GenState *g, ByteBuf *out, int id, int init_qp) {
	BitWriter w; bw_init(&w, 4096);
	bw_ue(&w, id); bw_ue(&w, 0);
	bw_u(&w, 1, g->cabac); bw_u(&w, 1, 0); bw_ue(&w, 0);
	bw_ue(&w, g->refs - 1 < 0 ? 0 : g->refs - 1); bw_ue(&w, 0);      /* default active refs: l0 = refs, l1 = 1 */
	bw_u(&w, 1, g->wp_p); bw_u(&w, 2, g->wp_b);
	bw_se(&w, init_qp - 26); bw_se(&w, 0);
	bw_se(&w, g->cqp_fixed ? g->cqp[0] : rnd(g, 9) - 4);
	bw_u(&w, 1, 1); bw_u(&w, 1, 0); bw_u(&w, 1, 0);
	bw_u(&w, 1, g->t8x8_mode);
	bw_u(&w, 1, g->scaling >= 2);
	if (g->scaling >= 2) put_scaling_matrix(g, &w, 6 + 2 * g->t8x8_mode);
	bw_se(&w, g->cqp_fixed ? g->cqp[1] : rnd(g, 9) - 4);
	bw_trailing(&w);
	e264_emit_nal(out, 3, 8, w.buf, w.pos / 8); free(w.buf);
}

/* ------------------------------------------------------------------------------------------ */
/* macroblock chooser                                                                           */
/* ------------------------------------------------------------------------------------------ */
/* --levels big: magnitudes spread over every power of two up to the 8-bit bound (7.4.5.3.2: -2^15 .. 2^15-1), so that CAVLC
 * takes level_prefix 15, 16 and above and CABAC long Exp-Golomb suffixes; now and then exactly -32768 or 32767 */
static int big_level(GenState *g) {
	int r = rnd(g, 16);
	if (r == 0) return -32768;
	if (r == 1) return 32767;
	int b = rnd(g, 16), m = (1 << b) + rnd(g, 1 << b);   /* [2^b, 2^(b+1)) */
	if (m > 32767) m = 32767;
	return rnd(g, 2) ? -m : m;
}
static void gen_block(GenState *g, int16_t *blk, int n, int first, const uint8_t *scan, int rich) {
	/* a few low-frequency-biased coefficients */
	int cnt = 1 + rnd(g, rich ? 6 : 3);
	for (int i = 0; i < cnt; i++) {
		int k = first + rnd(g, 1 + rnd(g, n - first));
		int lv = laplace(g, 2); if (lv == 0) lv = rnd(g, 2) ? 1 : -1;
		if (rnd(g, 40) == 0) lv *= 1 + rnd(g, 12);
		if (g->levels_big && rnd(g, 4) == 0) lv = big_level(g);
		blk[scan[k]] = (int16_t)lv;
	}
}
static const uint8_t scan_id4[4] = {0, 1, 2, 3};

static int legal_i4(int mode, int un) {
	switch (mode) {
	case 0: case 3: case 7: return !(un & 2);
	case 1: case 8: return !(un & 1);
	case 2: return 1;
	default: return !(un & 11);
	}
}
static int legal_i16(int mode, int un) { return mode == 0 ? !(un & 2) : mode == 1 ? !(un & 1) : mode == 2 ? 1 : !(un & 11); }
static int legal_chroma(int mode, int un) { return mode == 0 ? 1 : mode == 1 ? !(un & 1) : mode == 2 ? !(un & 2) : !(un & 11); }

/* fill residual staging, return cbp; is_i16: returns cbp with luma 0/15 */
static int gen_residual(GenState *g, SliceCtx *s, int t8, int is_i16, int intra) {
	int16_t *c = s->gen_coefs;
	memset(c, 0, sizeof(s->gen_coefs));
	int dens = g->density * (intra ? 2 : 1); if (dens > 95) dens = 95;
	int cbp = 0;
	if (is_i16) {
		if (pct(g, 70)) gen_block(g, c, 16, 0, h264_zigzag4x4, 1);
		if (pct(g, dens)) { for (int b = 0; b < 16; b++) if (pct(g, 50)) gen_block(g, c + 16 + 16 * b, 16, 1, h264_zigzag4x4, 0); }
		int any = 0; for (int i = 16; i < 272; i++) any |= c[i];
		cbp = any ? 15 : 0;
	} else if (t8) {
		for (int i = 0; i < 4; i++) if (pct(g, dens)) { gen_block(g, c + 16 + 64 * i, 64, 0, h264_zigzag8x8, 1); cbp |= 1 << i; }
	} else {
		for (int i = 0; i < 4; i++) if (pct(g, dens)) {
			for (int j = 0; j < 4; j++) if (pct(g, 55)) gen_block(g, c + 16 + 16 * (4 * i + j), 16, 0, h264_zigzag4x4, 0);
			int any = 0; for (int k = 0; k < 64; k++) any |= c[16 + 64 * i + k];
			if (any) cbp |= 1 << i;
		}
	}
	if (pct(g, dens)) {
		for (int pl = 0; pl < 2; pl++) if (pct(g, 70)) gen_block(g, c + 272 + 4 * pl, 4, 0, scan_id4, 0);
		if (pct(g, 40)) for (int j = 0; j < 8; j++) if (pct(g, 40)) gen_block(g, c + 280 + 16 * j, 16, 1, h264_zigzag4x4, 0);
		int ac = 0, dc = 0;
		for (int i = 280; i < 408; i++) ac |= c[i];
		for (int i = 272; i < 280; i++) dc |= c[i];
		cbp |= (ac ? 2 : dc ? 1 : 0) << 4;
	}
	return cbp;
}

/* a wanted motion vector for the block at 4x4 position (x4,y4) of the current MB, size w4 x h4 */
static void gen_mv(GenState *g, SliceCtx *s, int x4, int y4, int w4, int h4, int base[2], int16_t out[2]) {
	int X = s->mbx * 16 + x4 * 4, Y = s->mby * 16 + y4 * 4, W = s->w_mbs * 16, H = s->h_mbs * 16;
	int mvx = base[0] + laplace(g, 3), mvy = base[1] + laplace(g, 3);
	if (rnd(g, 4) == 0) { mvx &= ~3; mvy &= ~3; }                 /* some integer-pel vectors */
	int m = g->mvrange;                                           /* allowed overshoot beyond the picture, in pixels */
	int lo = (-m - X) * 4, hi = (W + m - X - w4 * 4) * 4;
	mvx = mvx < lo ? lo : mvx > hi ? hi : mvx;
	lo = (-m - Y) * 4; hi = (H + m - Y - h4 * 4) * 4;
	mvy = mvy < lo ? lo : mvy > hi ? hi : mvy;
	out[0] = (int16_t)mvx; out[1] = (int16_t)mvy;
}

/* --pcm-extreme: one 16x16 luma and two 8x8 chroma planes of a PCM macroblock at the ends of the sample range, so that the
 * intra predictors (8x8 reference filter, plane, DC) and the interpolation filters of the next pictures read extreme
 * neighbourhoods: a 0/255 step, a ramp over the full range, a 0/255 checker, or random bits (bytes or 0/255) */
static void gen_pcm_extreme(GenState *g, uint8_t *pcm) {
	int kind = rnd(g, 4), dir = rnd(g, 3), flip = rnd(g, 2) ? 255 : 0, at = 1 + rnd(g, 15), period = 1 + rnd(g, 2), bytes = rnd(g, 2);
	for (int i = 0; i < 384; i++) {
		int n = i < 256 ? 16 : 8, j = i < 256 ? i : (i - 256) & 63, x = j % n, y = j / n;
		int t = dir == 0 ? x : dir == 1 ? y : (x + y) / 2;   /* position across the pattern, 0..n-1 */
		int v;
		if (kind == 0) v = t * 16 / n < at ? 0 : 255;
		else if (kind == 1) v = t * 255 / (n - 1);
		else if (kind == 2) v = ((x / period + y / period) & 1) ? 255 : 0;
		else v = bytes ? rnd(g, 256) : rnd(g, 2) * 255;
		pcm[i] = (uint8_t)(v ^ flip);
	}
}

static void gen_choose_intra(GenState *g, SliceCtx *s, MbSyn *m, int base) {
	int r = rnd(g, 100);
	int un16 = sx_unavail16(s);
	do m->chroma_mode = rnd(g, 4); while (!legal_chroma(m->chroma_mode, un16));
	if (g->pcm_pm && rnd(g, 1000) < g->pcm_pm) {
		m->mb_type = base + 25;
		int v = rnd(g, 256);
		if (g->pcm_checker) {   /* 0/255 checkerboards: the most extreme input of the 6-tap filters (int16 corner cases of the reference) */
			/* period-3 pattern H L H | H L H in both directions: every +tap of (1,-5,20,20,-5,1) on 255, every -tap on 0 */
			int phx = rnd(g, 3), phy = rnd(g, 3);
			for (int i = 0; i < 256; i++) m->pcm[i] = (uint8_t)((((((i & 15) + phx) % 3 == 1) == ((((i >> 4) + phy) % 3) == 1)) ? 255 : 0) ^ (rnd(g, 32) ? 0 : rnd(g, 4)));
			for (int i = 256; i < 384; i++) m->pcm[i] = (uint8_t)((((i & 7) + ((i >> 3) & 7) + phx) & 1) ? 255 : 0);
		} else if (g->pcm_extreme) gen_pcm_extreme(g, m->pcm);
		else
		for (int i = 0; i < 384; i++) m->pcm[i] = (uint8_t)(rnd(g, 8) ? v + rnd(g, 9) - 4 : rnd(g, 256));
		return;
	}
	if (r < 30) {   /* Intra16x16 */
		int mode; do mode = rnd(g, 4); while (!legal_i16(mode, un16));
		int cbp = gen_residual(g, s, 0, 1, 1);
		m->mb_type = base + 1 + mode + 4 * (cbp >> 4) + 12 * ((cbp & 15) != 0);
		m->cbp = cbp;
	} else {
		m->mb_type = base;
		m->t8x8 = g->t8x8_mode && pct(g, g->t8x8_pct);
		if (m->t8x8) for (int i = 0; i < 4; i++) { int un = sx_unavail8x8(s, i), mode; do mode = rnd(g, 9); while (!legal_i4(mode, un)); m->ipm[4 * i] = mode; }
		else for (int b = 0; b < 16; b++) { int un = sx_unavail4x4(s, b), mode; do mode = rnd(g, 9); while (!legal_i4(mode, un)); m->ipm[b] = mode; }
		/* favour the predicted mode sometimes so that prev_intra_pred_mode_flag = 1 is exercised: handled
		 * naturally when the random mode equals the prediction */
		m->cbp = gen_residual(g, s, m->t8x8, 0, 1);
	}
}

static void gen_choose_mb(GenState *g, SliceCtx *s, MbSyn *m, int allow_skip) {
	memset(m, 0, sizeof(*m));
	int st = s->slice_type;
	if (g->qp_walk) {   /* --qp-walk: any delta of -26..25, often landing on QP_Y 0 or 51; QP_Y wraps modulo 52 (7.4.5) */
		int r = rnd(g, 8), d = r == 0 ? -s->qp : r == 1 ? 51 - s->qp : r < 5 ? rnd(g, 52) - 26 : 0;
		m->qp_delta = d > 25 ? d - 52 : d < -26 ? d + 52 : d;
	} else {
		m->qp_delta = rnd(g, 3) == 0 ? rnd(g, 5) - 2 : 0;
		/* keep QP inside [qp0-8, qp0+10] (touches both 8x8 dequant branches when qp0 ~ 30) */
		int q = s->qp + m->qp_delta;
		if (q < g->qp0 - 8 || q > g->qp0 + 10 || q < 0 || q > 51) m->qp_delta = 0;
	}
	if (st == SLICE_I) { gen_choose_intra(g, s, m, 0); return; }
	if (allow_skip && pct(g, g->skip_pct)) { m->skip = 1; return; }
	if (pct(g, g->intra_pct)) { gen_choose_intra(g, s, m, st == SLICE_P ? 5 : 23); return; }
	/* base vector: left neighbour's (smooth field) or the global drift */
	int base[2][2];
	for (int l = 0; l < 2; l++) {
		if (s->recA && s->recA->ref_idx[l][1] >= 0 && rnd(g, 4)) { base[l][0] = s->recA->mv[l][5][0]; base[l][1] = s->recA->mv[l][5][1]; }
		else { base[l][0] = g->drift[0] * (l ? -1 : 1); base[l][1] = g->drift[1] * (l ? -1 : 1); }
	}
	int no_sub8 = 1, direct16 = 0;
	const int infer8 = !g->direct4x4;
	if (st == SLICE_P) {
		int r = rnd(g, 100);
		m->mb_type = r < 35 ? 0 : r < 50 ? 1 : r < 65 ? 2 : 3;
		int np = m->mb_type == 0 ? 1 : m->mb_type == 3 ? 4 : 2;
		for (int p = 0; p < np; p++) m->ref_idx[0][p] = rnd(g, s->num_ref[0]);
		if (m->mb_type == 0) gen_mv(g, s, 0, 0, 4, 4, base[0], m->mv[0][0]);
		else if (m->mb_type == 1) { gen_mv(g, s, 0, 0, 4, 2, base[0], m->mv[0][0]); gen_mv(g, s, 0, 2, 4, 2, base[0], m->mv[0][8]); }
		else if (m->mb_type == 2) { gen_mv(g, s, 0, 0, 2, 4, base[0], m->mv[0][0]); gen_mv(g, s, 2, 0, 2, 4, base[0], m->mv[0][4]); }
		else for (int i = 0; i < 4; i++) {
			int sh = rnd(g, 100) < 50 ? 0 : 1 + rnd(g, 3);
			m->sub_type[i] = sh; if (sh) no_sub8 = 0;
			int x0 = (i & 1) * 2, y0 = (i >> 1) * 2;
			for (int j = 0; j < 4; j++) gen_mv(g, s, x0 + (j & 1), y0 + (j >> 1), sh == 0 || sh == 1 ? 2 : 1, sh == 0 || sh == 2 ? 2 : 1, base[0], m->mv[0][4 * i + j]);
		}
	} else {
		int r = rnd(g, 100);
		if (r < 15) { m->mb_type = 0; direct16 = 1; if (!infer8) no_sub8 = 0; }   /* 7.3.5: B_Direct_16x16 may use the 8x8 transform only with direct_8x8_inference_flag */
		else if (r < 45) m->mb_type = 1 + rnd(g, 3);
		else if (r < 75) m->mb_type = 4 + rnd(g, 18);
		else m->mb_type = 22;
		if (m->mb_type >= 1 && m->mb_type <= 21) {
			int shape = m->mb_type <= 3 ? 0 : 1 + ((m->mb_type - 4) & 1);
			int np = shape ? 2 : 1;
			for (int p = 0; p < np; p++) for (int l = 0; l < 2; l++) {
				m->ref_idx[l][p] = rnd(g, s->num_ref[l]);
				int x4 = shape == 2 ? p * 2 : 0, y4 = shape == 1 ? p * 2 : 0, w4 = shape == 2 ? 2 : 4, h4 = shape == 1 ? 2 : 4;
				gen_mv(g, s, x4, y4, w4, h4, base[l], m->mv[l][e264_blk_z(x4, y4)]);
			}
		} else if (m->mb_type == 22) {
			for (int i = 0; i < 4; i++) {
				int t = rnd(g, 100) < 25 ? 0 : 1 + rnd(g, 12);
				m->sub_type[i] = t;
				if (t == 0) { if (!infer8) no_sub8 = 0; }
				else if (sx_b_sub_shape[t]) no_sub8 = 0;
				int sh = sx_b_sub_shape[t], x0 = (i & 1) * 2, y0 = (i >> 1) * 2;
				for (int l = 0; l < 2; l++) {
					m->ref_idx[l][i] = rnd(g, s->num_ref[l]);
					for (int j = 0; j < 4; j++) gen_mv(g, s, x0 + (j & 1), y0 + (j >> 1), sh == 0 || sh == 1 ? 2 : 1, sh == 0 || sh == 2 ? 2 : 1, base[l], m->mv[l][4 * i + j]);
				}
			}
		}
	}
	(void)direct16;
	int t8 = g->t8x8_mode && no_sub8 && pct(g, g->t8x8_pct);
	m->cbp = gen_residual(g, s, t8, 0, 0);
	m->t8x8 = t8 && (m->cbp & 15);
	if (t8 && !(m->cbp & 15)) { /* no luma: flag not sent; staging already empty for luma */ }
}

/* ------------------------------------------------------------------------------------------ */
/* pictures                                                                                     */
/* ------------------------------------------------------------------------------------------ */
typedef struct PicPlan { int type; int idr; int is_ref; int frame_num; int poc; } PicPlan;   /* type: 0 P, 1 B, 2 I */

/* --wp-range full: one picture's explicit weight table.  Weights -128..127 (both ends forced now and then), offsets
 * -128..127, luma and chroma logWD 0..7; about a quarter of the entries take the inferred 2^logWD and offset 0 (their flag is
 * then 0, so 128 at logWD 7 in P pictures).  B pictures (7.4.3.2): every weight is coded at logWD 7, and each list-1 weight
 * keeps -128 <= w0 + w1 <= (logWD == 7 ? 127 : 128) with every list-0 weight in use, now and then at either bound. */
static int wp_full_value(GenState *g, int mid) { int r = rnd(g, 8); return r == 0 ? -128 : r == 1 ? 127 : r == 2 ? mid : rnd(g, 256) - 128; }
static void gen_wp_full(GenState *g, int is_b, int n0, int *lwd, int *cwd, int16_t w[2][16][3], int16_t o[2][16][3]) {
	*lwd = rnd(g, 8); *cwd = rnd(g, 8);
	for (int l = 0; l < 2; l++) for (int i = 0; i < 16; i++) for (int c = 0; c < 3; c += c ? 2 : 1) {
		const int wd = c ? *cwd : *lwd, n = c ? 2 : 1, infer = !(is_b && wd == 7) && rnd(g, 4) == 0;
		for (int k = c; k < c + n; k++) {
			int wk = wp_full_value(g, 1 << wd);
			w[l][i][k] = (int16_t)(infer ? 1 << wd : wk > 127 ? 127 : wk);
			o[l][i][k] = (int16_t)(infer ? 0 : wp_full_value(g, 0));
		}
	}
	if (!is_b) return;
	for (int c = 0; c < 3; c++) {
		int mn = 127, mx = -128, top = (c ? *cwd : *lwd) == 7 ? 127 : 128;
		for (int i = 0; i < n0; i++) { if (w[0][i][c] < mn) mn = w[0][i][c]; if (w[0][i][c] > mx) mx = w[0][i][c]; }
		const int lo = -128 - mn > -128 ? -128 - mn : -128, hi = top - mx < 127 ? top - mx : 127;
		for (int i = 0; i < 16; i++) {
			int r = rnd(g, 4), v = r == 0 ? lo : r == 1 ? hi : w[1][i][c];
			w[1][i][c] = (int16_t)(v < lo ? lo : v > hi ? hi : v);
		}
	}
}

/* returns 1 when the picture carried memory_management_control_operation 5 (frame_num and POC restart after it) */
/* --mvc: the frame slot number the second view's records give the inter-view reference (no picture of its own view uses it) */
#define IV_SLOT (E264_MAX_SLOTS - 1)
static const GenPic *gen_pic(const GenState *g, int slot) { return slot == IV_SLOT ? g->base : &g->dpb[slot]; }

static int encode_picture(GenState *g, ByteBuf *out, const PicPlan *pp, int idr_pic_id) {
	int nmb = g->W * g->H;
	const int anchor = g->au_anchor;   /* --mvc: an anchor access unit, whose second view predicts from the base view only */
	/* free DPB slot for this picture */
	int slot = -1;
	for (int i = 0; i < E264_MAX_SLOTS; i++) if (!g->dpb[i].used) { slot = i; break; }
	GenPic *cp = &g->dpb[slot];
	if (!cp->recs) cp->recs = (E264MbRec *)calloc((size_t)nmb, sizeof(E264MbRec));
	memset(cp->recs, 0, (size_t)nmb * sizeof(E264MbRec));
	memset(g->mbi, 0, (size_t)nmb * sizeof(MbInfo));
	cp->frame_num = pp->frame_num; cp->poc = pp->poc; cp->uid = g->next_uid++;
	if (pp->idr) for (int i = 0; i < E264_MAX_SLOTS; i++) g->dpb[i].used = 0;
	for (int i = 0; i < E264_MAX_SLOTS; i++) cp->slot_uid[i] = (g->dpb[i].used || i == slot) ? g->dpb[i].uid : -1;
	if (g->view) cp->slot_uid[IV_SLOT] = g->base->uid;

	/* reference lists exactly as 8.2.4.2 builds them for our simple GOPs (all short-term) */
	int l0[16], l1[16], n0 = 0, n1 = 0;
	if (pp->type != 2) {
		int idx[E264_MAX_SLOTS], n = 0;
		for (int i = 0; i < E264_MAX_SLOTS; i++) if (g->dpb[i].used) idx[n++] = i;
		if (pp->type == 0) {
			for (int i = 1; i < n; i++) for (int j = i; j > 0 && g->dpb[idx[j]].frame_num > g->dpb[idx[j - 1]].frame_num; j--) { int t = idx[j]; idx[j] = idx[j - 1]; idx[j - 1] = t; }
			for (int i = 0; i < n; i++) l0[n0++] = idx[i];
		} else {
			int bf[16], af[16], nb = 0, na = 0;
			for (int i = 0; i < n; i++) { if (g->dpb[idx[i]].poc < pp->poc) bf[nb++] = idx[i]; else af[na++] = idx[i]; }
			for (int i = 1; i < nb; i++) for (int j = i; j > 0 && g->dpb[bf[j]].poc > g->dpb[bf[j - 1]].poc; j--) { int t = bf[j]; bf[j] = bf[j - 1]; bf[j - 1] = t; }
			for (int i = 1; i < na; i++) for (int j = i; j > 0 && g->dpb[af[j]].poc < g->dpb[af[j - 1]].poc; j--) { int t = af[j]; af[j] = af[j - 1]; af[j - 1] = t; }
			for (int i = 0; i < nb; i++) l0[n0++] = bf[i];
			for (int i = 0; i < na; i++) l0[n0++] = af[i];
			for (int i = 0; i < na; i++) l1[n1++] = af[i];
			for (int i = 0; i < nb; i++) l1[n1++] = bf[i];
		}
	}
	/* the second view's lists end with the inter-view reference (H.8.2.1); an anchor's holds nothing else */
	const int nt0 = n0, nt1 = n1;
	if (g->view) { if (anchor) n0 = 0; l0[n0++] = IV_SLOT; if (pp->type == 1) l1[n1++] = IV_SLOT; }
	if (pp->type == 1 && n1 > 1 && l0[0] == l1[0]) { int t = l1[0]; l1[0] = l1[1]; l1[1] = t; }
	int num_ref[2] = {n0 < 1 ? 1 : n0, n1 < 1 ? 1 : n1};
	if (pp->type == 1 && !g->view) { if (num_ref[0] > 2) num_ref[0] = 2; if (num_ref[1] > 2) num_ref[1] = 2; }
	if (g->view && !g->base_inter_view) { num_ref[0] = nt0; num_ref[1] = nt1; }   /* a base view that is no inter-view reference (B: both lists hold a temporal picture first) */
	/* --temporal: a P second view is the co-located picture of the B second views after it, and temporal direct needs every
	 * picture it predicts from in their list 0 (8.4.1.2.3).  Its inter-view reference goes to the front (list modification)
	 * and it leaves out the picture the sliding window drops when it is marked. */
	const int iv_front = g->view && !anchor && g->temporal && pp->type == 0;
	if (iv_front) {
		for (int i = n0 - 1; i > 0; i--) l0[i] = l0[i - 1];
		l0[0] = IV_SLOT; num_ref[0] = 1 + (nt0 >= g->refs ? g->refs - 1 : nt0);
	}
	g->drift[0] = laplace(g, 6); g->drift[1] = laplace(g, 4);
	g->cur_is_b = pp->type == 1;

	/* --dpb: plan this picture's reference marking (8.2.5.4) on a copy of the DPB model; every operation targets a
	 * picture that exists, and at most refs-1 other references remain so that the picture itself fits */
	int mmco[40][3], n_mmco = 0, idr_long = 0, cur_long = -1, did_op5 = 0;
	int m_used[E264_MAX_SLOTS], m_long[E264_MAX_SLOTS], m_idx[E264_MAX_SLOTS], m_max = g->max_long_idx_plus1;
	for (int i = 0; i < E264_MAX_SLOTS; i++) { m_used[i] = g->dpb[i].used && i != slot; m_long[i] = g->dpb[i].is_long; m_idx[i] = g->dpb[i].long_idx; }
	if (g->dpb_mode && pp->idr) { idr_long = g->refs > 1 && rnd(g, 4) == 0;   /* with one reference frame the reference decoder asserts (edge264_headers.c:1099) */ m_max = idr_long ? 1 : 0; cur_long = idr_long ? 0 : -1; }
	if (g->dpb_mode && !pp->idr && pp->type == 0 && pp->is_ref && !(g->view && anchor)) {
		const int maxfn = 1 << g->log2_max_frame_num, cur = pp->frame_num & (maxfn - 1);
#define DIFF(i) (cur - (((g->dpb[i].frame_num & (maxfn - 1)) > cur) ? (g->dpb[i].frame_num & (maxfn - 1)) - maxfn : (g->dpb[i].frame_num & (maxfn - 1))))
#define PICK(cond, out) do { int c_[E264_MAX_SLOTS], n_ = 0; for (int i = 0; i < E264_MAX_SLOTS; i++) if (m_used[i] && (cond)) c_[n_++] = i; out = n_ ? c_[rnd(g, n_)] : -1; } while (0)
#define DROP_IDX(k) do { for (int i = 0; i < E264_MAX_SLOTS; i++) if (m_used[i] && m_long[i] && m_idx[i] == (k)) m_used[i] = 0; } while (0)
		int cnt0 = 0, nshort0 = 0, t;
		for (int i = 0; i < E264_MAX_SLOTS; i++) if (m_used[i]) { cnt0++; nshort0 += !m_long[i]; }
		const int op5 = g->mmco5 && g->gop == 1 && pp->frame_num >= 3 && rnd(g, 12) == 0;   /* --mmco5 only: the reference reports one FrameId twice after such a picture (observed), so these streams are not in the parity suite */   /* 8.2.5.4: everything else leaves, this picture restarts frame_num and POC at 0 */
		const int adaptive = !op5 && (rnd(g, 2) || (cnt0 >= g->refs && nshort0 == 0));   /* the sliding window needs a short-term picture to drop */
		if (op5) { mmco[0][0] = 5; n_mmco = 1; did_op5 = 1; for (int i = 0; i < E264_MAX_SLOTS; i++) m_used[i] = 0; m_max = 0; }
		/* short-term pictures about to alias in frame_num must go in any case */
		for (int i = 0; i < E264_MAX_SLOTS && !op5; i++) if (m_used[i] && !m_long[i] && pp->frame_num - g->dpb[i].frame_num >= maxfn - 3) { mmco[n_mmco][0] = 1; mmco[n_mmco][1] = DIFF(i) - 1; n_mmco++; m_used[i] = 0; }
		if (adaptive || n_mmco) {
			if (rnd(g, 3) == 0) { m_max = rnd(g, g->refs + 1); mmco[n_mmco][0] = 4; mmco[n_mmco][1] = m_max; n_mmco++; for (int i = 0; i < E264_MAX_SLOTS; i++) if (m_used[i] && m_long[i] && m_idx[i] >= m_max) m_used[i] = 0; }
			if (g->refs > 1 && m_max > 0 && rnd(g, 2)) { PICK(!m_long[i], t); if (t >= 0) { int k = rnd(g, m_max); DROP_IDX(k); mmco[n_mmco][0] = 3; mmco[n_mmco][1] = DIFF(t) - 1; mmco[n_mmco][2] = k; n_mmco++; m_long[t] = 1; m_idx[t] = k; } }
			if (rnd(g, 3) == 0) { PICK(!m_long[i], t); if (t >= 0) { mmco[n_mmco][0] = 1; mmco[n_mmco][1] = DIFF(t) - 1; n_mmco++; m_used[t] = 0; } }
			if (rnd(g, 4) == 0) { PICK(m_long[i], t); if (t >= 0) { mmco[n_mmco][0] = 2; mmco[n_mmco][1] = m_idx[t]; n_mmco++; m_used[t] = 0; } }
			for (;;) {   /* room for the current picture */
				int cnt = 0; for (int i = 0; i < E264_MAX_SLOTS; i++) cnt += m_used[i];
				if (cnt < g->refs) break;
				int old = -1; for (int i = 0; i < E264_MAX_SLOTS; i++) if (m_used[i] && !m_long[i] && (old < 0 || g->dpb[i].frame_num < g->dpb[old].frame_num)) old = i;
				if (old >= 0) { mmco[n_mmco][0] = 1; mmco[n_mmco][1] = DIFF(old) - 1; n_mmco++; m_used[old] = 0; }
				else { PICK(m_long[i], t); mmco[n_mmco][0] = 2; mmco[n_mmco][1] = m_idx[t]; n_mmco++; m_used[t] = 0; }
			}
			if (g->refs > 1 && m_max > 0 && rnd(g, 4) == 0) { int k = rnd(g, m_max); DROP_IDX(k); mmco[n_mmco][0] = 6; mmco[n_mmco][1] = k; n_mmco++; cur_long = k; }
		}
#undef DIFF
#undef PICK
#undef DROP_IDX
	}

	int rows_per_slice = (g->H + g->slices - 1) / g->slices;
	int16_t w_tab[2][16][3], o_tab[2][16][3]; int lwd = 0, cwd = 0, w_ready = 0; uint8_t w_sent[2][16]; memset(w_sent, 0, sizeof(w_sent));
	for (int sl = 0; sl * rows_per_slice < g->H; sl++) {
		/* --mixed-slices: later slices of a P picture may be I slices, of a B picture I or P slices (7.4.3: slice types of one
		 * picture are independent) */
		int st = pp->type;
		if (g->mixed && sl > 0 && pp->type != 2 && rnd(g, 3) == 0) st = (pp->type == 1 && rnd(g, 2)) ? 0 : 2;
		int first_mb = sl * rows_per_slice * g->W;
		int last_mb = (sl + 1) * rows_per_slice * g->W; if (last_mb > nmb) last_mb = nmb;
		int pps_id = st == 2 ? 0 : st == 0 ? 1 : 2;
		BitWriter w; bw_init(&w, 1 << 16);
		/* nal_unit_header_mvc_extension: non_idr_flag, priority_id 0, view_id, temporal_id 0, anchor_pic_flag, inter_view_flag
		 * (the second view is no one's reference), reserved_one_bit */
		const uint32_t mvc_hdr = (uint32_t)!pp->idr << 22 | (uint32_t)g->view << 6 | (uint32_t)anchor << 2 | (uint32_t)(!g->view && g->base_inter_view) << 1 | 1;
		if (g->view) bw_u(&w, 24, mvc_hdr);
		bw_ue(&w, first_mb);
		bw_ue(&w, st + (rnd(g, 2) ? 5 : 0));
		bw_ue(&w, pps_id);
		bw_u(&w, g->log2_max_frame_num, pp->frame_num & ((1 << g->log2_max_frame_num) - 1));
		if (pp->idr) bw_ue(&w, idr_pic_id);
		if (g->poc_type == 0) bw_u(&w, g->log2_max_poc_lsb, pp->poc & ((1 << g->log2_max_poc_lsb) - 1));
		int direct_spatial = !g->temporal;
		if (st != 2) {
			if (st == 1) bw_u(&w, 1, direct_spatial);
			bw_u(&w, 1, 1);   /* num_ref_idx_active_override_flag */
			bw_ue(&w, num_ref[0] - 1);
			if (st == 1) bw_ue(&w, num_ref[1] - 1);
			if ((g->view && anchor && !pp->idr) || iv_front) {   /* the inter-view reference to the front: a non-IDR anchor uses it alone */
				bw_u(&w, 1, 1); bw_ue(&w, 5); bw_ue(&w, 0); bw_ue(&w, 3);
			} else if (g->dpb_mode && st == 0 && n0 > 0 && rnd(g, 2)) {   /* ref_pic_list_modification (7.3.3.1, 8.2.4.3): move existing pictures to the front */
				bw_u(&w, 1, 1); g->stat_rplm++;
				const int maxfn = 1 << g->log2_max_frame_num;
				int pred = pp->frame_num & (maxfn - 1), nops = 1 + rnd(g, num_ref[0] < 3 ? num_ref[0] : 3), view_pred = -1;
				for (int k = 0; k < nops; k++) {
					const int ti = l0[rnd(g, n0)];
					if (ti == IV_SLOT) {   /* H.8.2.2.3: idc 5 adds abs_diff_view_idx_minus1 + 1 to the view index prediction (-1 first), idc 4 subtracts it, modulo the one inter-view reference */
						if (!g->base_inter_view) continue;
						bw_ue(&w, view_pred < 0 ? 5 : 4); bw_ue(&w, 0); view_pred = 0;
						continue;
					}
					const GenPic *t = &g->dpb[ti];
					if (t->is_long) { bw_ue(&w, 2); bw_ue(&w, t->long_idx); continue; }
					const int nowrap = t->frame_num & (maxfn - 1);   /* picNumL0NoWrap of a frame is its frame_num */
					if (nowrap == pred) continue;
					if (nowrap < pred) { bw_ue(&w, 0); bw_ue(&w, pred - nowrap - 1); } else { bw_ue(&w, 1); bw_ue(&w, nowrap - pred - 1); }
					pred = nowrap;
				}
				bw_ue(&w, 3);
			} else bw_u(&w, 1, 0);   /* ref_pic_list_modification_flag_l0 */
			if (st == 1) bw_u(&w, 1, 0);
			int wp = st == 0 ? g->wp_p : g->wp_b;
			if (wp == 1) {
				if (!w_ready && g->wp_full) { w_ready = 1; gen_wp_full(g, pp->type == 1, num_ref[0], &lwd, &cwd, w_tab, o_tab); }
				if (!w_ready) { w_ready = 1;
					lwd = rnd(g, pp->type == 1 ? 7 : 8); cwd = rnd(g, pp->type == 1 ? 7 : 8);   /* logWD 7 + inferred weight 128 is only legal for uni-prediction */
					for (int l = 0; l < 2; l++) for (int i = 0; i < 16; i++) for (int c = 0; c < 3; c++) {
						int wd = c ? cwd : lwd;
						int r = rnd(g, 10);
						w_tab[l][i][c] = (int16_t)(r < 2 ? (wd == 7 ? 127 : 1 << wd) : rnd(g, 72) - 16);   /* coded values stay in -128..127 */
						if (pp->type == 1 && w_tab[l][i][c] > 63) w_tab[l][i][c] = 63;                       /* bi-pred: w0 + w1 <= 127 */
						o_tab[l][i][c] = (int16_t)(rnd(g, 41) - 20);
					}
				}
				bw_ue(&w, lwd); bw_ue(&w, cwd);
				for (int l = 0; l <= (st == 1); l++) for (int i = 0; i < num_ref[l]; i++) {
					int lf, cf;
					if (g->wp_full) {   /* the table holds the inferred values where a flag is to be 0 */
						lf = !(w_tab[l][i][0] == (1 << lwd) && o_tab[l][i][0] == 0);
						cf = !(w_tab[l][i][1] == (1 << cwd) && o_tab[l][i][1] == 0 && w_tab[l][i][2] == (1 << cwd) && o_tab[l][i][2] == 0);
					} else {
						lf = rnd(g, 4) != 0; cf = rnd(g, 4) != 0;
						if (w_sent[l][i]) { lf = !(w_tab[l][i][0] == (1 << lwd) && o_tab[l][i][0] == 0); cf = 1; }
					}
					if (!lf) { w_tab[l][i][0] = (int16_t)(1 << lwd); o_tab[l][i][0] = 0; }
					if (!cf) for (int c = 1; c < 3; c++) { w_tab[l][i][c] = (int16_t)(1 << cwd); o_tab[l][i][c] = 0; }
					bw_u(&w, 1, lf); if (lf) { bw_se(&w, w_tab[l][i][0]); bw_se(&w, o_tab[l][i][0]); }
					bw_u(&w, 1, cf); if (cf) for (int c = 1; c < 3; c++) { bw_se(&w, w_tab[l][i][c]); bw_se(&w, o_tab[l][i][c]); }
					w_sent[l][i] = 1;
				}
			}
		}
		if (pp->is_ref) {
			if (pp->idr) { bw_u(&w, 1, 0); bw_u(&w, 1, g->dpb_mode && idr_long); }
			else if (n_mmco) {   /* dec_ref_pic_marking( ) with adaptive_ref_pic_marking_mode_flag = 1 (7.3.3.3) */
				bw_u(&w, 1, 1);
				for (int k = 0; k < n_mmco; k++) {
					const int op = mmco[k][0];
					bw_ue(&w, op);
					if (op == 1 || op == 3) bw_ue(&w, mmco[k][1]);        /* difference_of_pic_nums_minus1 */
					if (op == 2) bw_ue(&w, mmco[k][1]);                   /* long_term_pic_num */
					if (op == 3) bw_ue(&w, mmco[k][2]);                   /* long_term_frame_idx */
					if (op == 4) bw_ue(&w, mmco[k][1]);                   /* max_long_term_frame_idx_plus1 */
					if (op == 6) bw_ue(&w, mmco[k][1]);                   /* long_term_frame_idx */
				}
				bw_ue(&w, 0);
			}
			else bw_u(&w, 1, 0);
		}
		int cabac_init_idc = rnd(g, 3);
		if (g->cabac && st != 2) bw_ue(&w, cabac_init_idc);
		int slice_qp = g->qp0 + rnd(g, 7) - 3;
		if (g->qp_walk) { int r = rnd(g, 4); slice_qp = r == 0 ? 0 : r == 1 ? 51 : rnd(g, 52); }
		if (slice_qp < 0) slice_qp = 0;
		if (slice_qp > 51) slice_qp = 51;
		int pic_init_qp = g->qp0;
		bw_se(&w, slice_qp - pic_init_qp);
		int idc = g->deblock;
		const int off = g->deblock_off == 2 || (g->deblock_off == 1 && !pp->is_ref && !(g->mvc && !g->view && g->base_inter_view));   /* an inter-view reference counts as a reference (edge264_mvc.h) */
		bw_ue(&w, off ? 1 : idc);
		if (idc != 1) {   /* the offsets are drawn either way, so that the rest of the stream does not change */
			const int a = rnd(g, 13) - 6, b = rnd(g, 13) - 6;
			if (!off) { bw_se(&w, a); bw_se(&w, b); }
		}

		/* slice data through the shared writer */
		SliceCtx *s = (SliceCtx *)calloc(1, sizeof(SliceCtx));
		MbSyn syn;
		s->cabac = g->cabac; s->bw = &w; s->syn = &syn;
		s->w_mbs = g->W; s->h_mbs = g->H;
		s->slice_type = st; s->slice_id = sl + 1; s->slice_idx = sl;
		s->num_ref[0] = num_ref[0]; s->num_ref[1] = num_ref[1];
		s->direct_spatial = direct_spatial; s->direct_8x8_inference = !g->direct4x4; s->transform_8x8_mode = g->t8x8_mode;
		s->qp = slice_qp; s->deblock_idc = idc; s->cur_poc = pp->poc;
		s->mbi = g->mbi; s->recs = cp->recs; s->coefs = g->pool; s->coef_cap = (uint32_t)nmb * 408; s->n_coefs = 0;
		memset(s->ref_slot, -1, sizeof(s->ref_slot));
		for (int i = 0; i < n0 && i < 16; i++) { s->ref_slot[0][i] = (int8_t)l0[i]; s->ref_uid[0][i] = gen_pic(g, l0[i])->uid; s->ref_poc[0][i] = gen_pic(g, l0[i])->poc; }
		for (int i = 0; i < n1 && i < 16; i++) { s->ref_slot[1][i] = (int8_t)l1[i]; s->ref_uid[1][i] = gen_pic(g, l1[i])->uid; s->ref_poc[1][i] = gen_pic(g, l1[i])->poc; }
		if (st == 1 && n1 > 0) { s->col_recs = gen_pic(g, l1[0])->recs; s->col_slot_uid = gen_pic(g, l1[0])->slot_uid; }
		s->skip_run = 0;
		if (g->cabac) {
			while (w.pos & 7) bw_u(&w, 1, 1);   /* cabac_alignment_one_bit */
			cabac_init_states(s->ce.state, st == 2 ? 0 : 1 + cabac_init_idc, slice_qp);
			cabac_enc_start(&s->ce, &w);
		}
		for (int a = first_mb; a < last_mb; a++) {
			s->mbaddr = a; s->mbx = a % g->W; s->mby = a / g->W;
			sx_set_neighbours(s);   /* the chooser looks at availability before sx_one_mb recomputes it */
			memset(s->cur, 0, sizeof(MbInfo)); s->cur->slice_id = (uint16_t)s->slice_id;
			gen_choose_mb(g, s, &syn, 1);
			sx_one_mb(s);
			if (s->error) { fprintf(stderr, "gen264: internal error %d at mb %d\n", s->error, a); exit(3); }
			if (g->cabac) cabac_enc_terminate(&s->ce, a == last_mb - 1);
		}
		if (g->cabac) bw_align_zero(&w);   /* the arithmetic coder's last bit is the rbsp_stop_one_bit */
		else { if (s->skip_run > 0) bw_ue(&w, s->skip_run); bw_trailing(&w); }
		if (g->mvc && !g->view) {   /* prefix NAL unit of the base view slice: its nal_unit_header_mvc_extension alone */
			const uint8_t prefix[3] = {(uint8_t)(mvc_hdr >> 16), (uint8_t)(mvc_hdr >> 8), (uint8_t)mvc_hdr};
			e264_emit_nal(out, pp->is_ref ? 2 + pp->idr : 0, 14, prefix, 3);
		}
		e264_emit_nal(out, pp->is_ref ? 2 + pp->idr : 0, g->view ? 20 : pp->idr ? 5 : 1, w.buf, w.pos / 8);
		free(w.buf); free(s);
	}
	for (int k = 0; k < n_mmco; k++) g->stat_mmco[mmco[k][0]]++;
	if (getenv("GEN264_DEBUG")) { fprintf(stderr, "pic uid %d type %d idr %d frame_num %d poc %d refs %d:", cp->uid, pp->type, pp->idr, pp->frame_num, pp->poc, n0); for (int k = 0; k < n_mmco; k++) fprintf(stderr, " mmco%d(%d,%d)", mmco[k][0], mmco[k][1], mmco[k][2]); fprintf(stderr, "%s\n", idr_long ? " long-term IDR" : ""); }
	g->stat_idr_long += idr_long;
	g->last_pic = cp;
	/* marking: the planned memory-management operations, or the sliding window (8.2.5.3) */
	if (pp->is_ref) {
		if (n_mmco || (g->dpb_mode && pp->idr)) {
			for (int i = 0; i < E264_MAX_SLOTS; i++) if (i != slot) { g->dpb[i].used = m_used[i]; g->dpb[i].is_long = m_long[i]; g->dpb[i].long_idx = m_idx[i]; }
			g->max_long_idx_plus1 = m_max;
			cp->used = 1; cp->is_long = cur_long >= 0; cp->long_idx = cur_long >= 0 ? cur_long : 0;
			if (did_op5) { cp->frame_num = 0; cp->poc = 0; }
		} else {
			cp->used = 1; cp->is_long = 0; cp->long_idx = 0;
			int n = 0; for (int i = 0; i < E264_MAX_SLOTS; i++) n += g->dpb[i].used;
			while (n > g->refs) {
				int best = -1;
				for (int i = 0; i < E264_MAX_SLOTS; i++) if (g->dpb[i].used && !g->dpb[i].is_long && i != slot && (best < 0 || g->dpb[i].frame_num < g->dpb[best].frame_num)) best = i;
				if (best < 0) break;
				g->dpb[best].used = 0; n--;
			}
		}
	}
	return did_op5;
}

/* --mvc: the coding state of the other view (its pictures, generator and long-term index bound) becomes the current one */
static void switch_view(GenState *g) {
	uint64_t r = g->rng; g->rng = g->rng_view; g->rng_view = r;
	int m = g->max_long_idx_plus1; g->max_long_idx_plus1 = g->max_long_view; g->max_long_view = m;
	g->view ^= 1; g->dpb = g->views[g->view];
}

/* one access unit: its base view picture, then with --mvc its second view (same type, frame_num, POC and nal_ref_idc; an I
 * base view gets a P second view).  Returns encode_picture's result for the base view. */
static int encode_au(GenState *g, ByteBuf *out, const PicPlan *pp, int idr_pic_id) {
	g->au_anchor = pp->idr || pp->type == 2;
	if (!g->mvc) return encode_picture(g, out, pp, idr_pic_id);
	switch_view(g);
	g->base_inter_view = pp->is_ref || rnd(g, 2);   /* a non-reference base view may still be an inter-view reference */
	switch_view(g);
	const int r = encode_picture(g, out, pp, idr_pic_id);
	g->base = g->last_pic;
	switch_view(g);
	PicPlan q = *pp;
	if (q.type == 2) q.type = 0;
	encode_picture(g, out, &q, idr_pic_id);
	switch_view(g);
	return r;
}

static int argi(int argc, char **argv, const char *name, int def) {
	for (int i = 1; i + 1 < argc; i++) if (!strcmp(argv[i], name)) return atoi(argv[i + 1]);
	return def;
}
static int argf(int argc, char **argv, const char *name) { for (int i = 1; i < argc; i++) if (!strcmp(argv[i], name)) return 1; return 0; }

int main(int argc, char **argv) {
	GenState *g = (GenState *)calloc(1, sizeof(GenState));
	const char *outp = NULL, *gop = "I";
	for (int i = 1; i + 1 < argc; i++) { if (!strcmp(argv[i], "-o")) outp = argv[i + 1]; if (!strcmp(argv[i], "--gop")) gop = argv[i + 1]; }
	if (!outp) { fprintf(stderr, "usage: gen264 -o out.264 [options] (see the file header)\n"); return 2; }
	g->W = argi(argc, argv, "-W", 120); g->H = argi(argc, argv, "-H", 68); g->frames = argi(argc, argv, "-n", 8);
	g->rng = 0x9E3779B97F4A7C15ull ^ ((uint64_t)argi(argc, argv, "-s", 1) * 0xD1B54A32D192ED03ull); rnd64(g);
	g->cabac = !argf(argc, argv, "--cavlc");
	g->gop = !strcmp(gop, "I") ? 0 : !strcmp(gop, "IP") ? 1 : 2;
	g->idr_period = argi(argc, argv, "--idr", 30);
	g->refs = argi(argc, argv, "--refs", g->gop ? 2 : 1);
	g->t8x8_pct = argi(argc, argv, "--t8x8", 40); g->t8x8_mode = g->t8x8_pct > 0;
	g->scaling = argi(argc, argv, "--scaling", 0);
	g->wp = argi(argc, argv, "--wp", 0); g->wp_p = g->wp == 1; g->wp_b = g->wp;
	g->slices = argi(argc, argv, "--slices", 1);
	g->deblock = argi(argc, argv, "--deblock", 0);
	g->density = argi(argc, argv, "--density", 25);
	g->qp0 = argi(argc, argv, "--qp", 28);
	g->temporal = argf(argc, argv, "--temporal");
	g->pcm_pm = argi(argc, argv, "--pcm", 2);
	g->pcm_checker = argf(argc, argv, "--pcm-checker");
	g->crop_bottom = argi(argc, argv, "--crop-bottom", (g->H * 16) % 1080 == 8 ? 8 : 0);
	g->level = argi(argc, argv, "--level", g->W * g->H > 36864 ? 62 : g->W * g->H > 8704 ? 51 : 40);
	g->mvrange = argi(argc, argv, "--mvrange", 24);
	g->intra_pct = argi(argc, argv, "--intra-pct", 10);
	g->skip_pct = argi(argc, argv, "--skip-pct", 15);
	g->crop_left = argi(argc, argv, "--crop-left", 0); g->crop_right = argi(argc, argv, "--crop-right", 0); g->crop_top = argi(argc, argv, "--crop-top", 0);
	g->direct4x4 = argf(argc, argv, "--direct4x4"); g->nonref_p = argf(argc, argv, "--nonref-p"); g->extra_nals = argf(argc, argv, "--extra-nals");
	g->bref = argf(argc, argv, "--bref");
	g->i_period = argi(argc, argv, "--i-period", 0);
	g->no_vui = argf(argc, argv, "--no-vui"); g->reorder = argi(argc, argv, "--reorder", -1);
	if (g->reorder > 16) { fprintf(stderr, "gen264: --reorder takes 0..16\n"); return 2; }
	for (int i = 1; i + 1 < argc; i++) if (!strcmp(argv[i], "--deblock-off")) {
		g->deblock_off = !strcmp(argv[i + 1], "nonref") ? 1 : !strcmp(argv[i + 1], "all") ? 2 : -1;
		if (g->deblock_off < 0) { fprintf(stderr, "gen264: --deblock-off takes nonref or all\n"); return 2; }
	}
	g->mixed = argf(argc, argv, "--mixed-slices"); g->ps_update = argf(argc, argv, "--ps-update");
	g->dpb_mode = argf(argc, argv, "--dpb"); g->mmco5 = argf(argc, argv, "--mmco5"); g->poc_type = argi(argc, argv, "--poc-type", 0);
	g->log2_max_frame_num = g->dpb_mode ? 4 : 8; g->log2_max_poc_lsb = 10;
	for (int i = 1; i + 1 < argc; i++) {
		if (!strcmp(argv[i], "--wp-range")) g->wp_full = !strcmp(argv[i + 1], "full");
		if (!strcmp(argv[i], "--levels")) g->levels_big = !strcmp(argv[i + 1], "big");
		if (!strcmp(argv[i], "--cqp-offset")) g->cqp_fixed = sscanf(argv[i + 1], "%d,%d", &g->cqp[0], &g->cqp[1]) == 2;
	}
	g->qp_walk = argf(argc, argv, "--qp-walk"); g->pcm_extreme = argf(argc, argv, "--pcm-extreme");
	g->dpb = g->views[0];
	for (int i = 1; i < argc; i++) if (!strcmp(argv[i], "--mvc")) {
		g->mvc = 1;
		const uint64_t seed = i + 1 < argc && argv[i + 1][0] >= '0' && argv[i + 1][0] <= '9' ? strtoull(argv[i + 1], NULL, 10) : 1;
		g->rng_view = 0x6A09E667F3BCC909ull ^ (seed * 0xD1B54A32D192ED03ull);
	}
	/* --mmco5, and --bref or --dpb beside --temporal, would make second views whose co-located pictures predict from
	 * pictures no longer in the list 0 of the B pictures after them (8.4.1.2.3) */
	if (g->mvc && (g->mmco5 || (g->temporal && (g->bref || g->dpb_mode)))) { fprintf(stderr, "gen264: --mvc does not combine with --mmco5, nor --temporal with --bref or --dpb\n"); return 2; }
	if (g->cqp_fixed && (g->cqp[0] < -12 || g->cqp[0] > 12 || g->cqp[1] < -12 || g->cqp[1] > 12)) { fprintf(stderr, "gen264: --cqp-offset takes two offsets in -12..12\n"); return 2; }
	if ((g->dpb_mode && g->gop == 0) || (g->poc_type && g->gop != 1)) { fprintf(stderr, "gen264: --dpb needs --gop IP or IPB, --poc-type needs --gop IP\n"); return 2; }
	if (g->slices > g->H) g->slices = g->H;
	if (g->refs < 1) g->refs = 1;
	if (g->refs > 16) g->refs = 16;
	sx_init_tables();
	int nmb = g->W * g->H;
	g->mbi = (MbInfo *)calloc((size_t)nmb, sizeof(MbInfo));
	g->pool = (int16_t *)calloc((size_t)nmb * 408 + 1024, sizeof(int16_t));
	ByteBuf out = {0, 0, 0};
	int frame_num = 0, idr_id = 0, disp = 0, since_idr = 0, since_i = 0;
	/* coding order.  gop 0: IDR every picture; gop 1: IDR P P P ...; gop 2: IDR P B B P B B ... (B not referenced) */
	for (int k = 0; k < g->frames;) {
		int need_idr = k == 0 || since_idr >= g->idr_period;
		if (g->gop == 0 || need_idr) {
			write_sps(g, &out, 0);
			for (int id = 0; id < 3; id++) write_pps(g, &out, id, g->qp0);
			PicPlan p = {2, 1, 1, 0, 0};
			frame_num = 0; disp = 0; since_idr = 0;
			encode_au(g, &out, &p, idr_id++ & 0xffff);
			frame_num = 1; disp = 1; since_idr = 1; since_i = 1; k++;
			continue;
		}
		if (g->ps_update && rnd(g, 4) == 0) { if (rnd(g, 3) == 0) write_sps(g, &out, 0); for (int id = 0; id < 3; id++) write_pps(g, &out, id, g->qp0); }
		if (g->extra_nals) {
			if (rnd(g, 2)) { uint8_t aud[1] = {(uint8_t)(rnd(g, 3) << 5 | 0x10)}; e264_emit_nal(&out, 0, 9, aud, 1); }
			if (rnd(g, 3) == 0) { uint8_t sei[40]; int n = 2 + rnd(g, 30); sei[0] = 5; sei[1] = (uint8_t)n; for (int i = 0; i < n; i++) sei[2 + i] = (uint8_t)rnd(g, 256); sei[2 + n] = 0x80; e264_emit_nal(&out, 0, 6, sei, 3 + n); }
			if (rnd(g, 4) == 0) { uint8_t fil[24]; int n = 1 + rnd(g, 20); for (int i = 0; i < n; i++) fil[i] = 0xff; fil[n] = 0x80; e264_emit_nal(&out, 0, 12, fil, n + 1); }
		}
		const int i_pic = g->i_period > 0 && since_i >= g->i_period;   /* --i-period: this anchor is a non-IDR I picture */
		if (i_pic) since_i = 0;
		if (g->gop == 1) {
			const int is_ref = i_pic || !(g->nonref_p && g->poc_type == 0 && !g->dpb_mode && rnd(g, 3) == 0);
			PicPlan p = {i_pic ? 2 : 0, 0, is_ref, frame_num, disp * 2};
			if (encode_au(g, &out, &p, 0)) { frame_num = 0; disp = 0; }
			if (is_ref) frame_num++;
			disp++; since_idr++; since_i++; k++;
			continue;
		}
		/* IPB: next anchor P at display disp+2 (or fewer if the sequence ends), then the B pictures before it */
		int nb = 2;
		if (k + 1 + nb > g->frames) nb = g->frames - k - 1;
		if (since_idr + 1 + nb > g->idr_period) nb = g->idr_period - since_idr - 1 < 0 ? 0 : g->idr_period - since_idr - 1;
		PicPlan p = {i_pic ? 2 : 0, 0, 1, frame_num, (disp + nb) * 2};
		encode_au(g, &out, &p, 0);
		frame_num++; k++;
		for (int b = 0; b < nb; b++) {
			int used = 0, nshort = 0;
			for (int i = 0; i < E264_MAX_SLOTS; i++) if (g->dpb[i].used) { used++; nshort += !g->dpb[i].is_long; }
			const int can_ref = used < g->refs || nshort > 0;   /* the sliding window needs a short-term picture to drop */
			PicPlan q = {1, 0, g->bref && b == 0 && nb == 2 && can_ref, frame_num, (disp + b) * 2}; encode_au(g, &out, &q, 0); if (q.is_ref) frame_num++; k++;
		}
		disp += nb + 1; since_idr += nb + 1; since_i += nb + 1;
	}
	FILE *f = fopen(outp, "wb");
	if (!f) { perror(outp); return 2; }
	fwrite(out.p, 1, out.n, f); fclose(f);
	fprintf(stderr, "gen264: %d frames %dx%d, %zu bytes (%.1f bits/MB)\n", g->frames, g->W * 16, g->H * 16, out.n, 8.0 * out.n / ((double)g->frames * nmb));
	if (g->dpb_mode) fprintf(stderr, "gen264: --dpb: %d slices with list modification, memory-management ops 1..6: %d %d %d %d %d %d, %d long-term IDR\n", g->stat_rplm, g->stat_mmco[1], g->stat_mmco[2], g->stat_mmco[3], g->stat_mmco[4], g->stat_mmco[5], g->stat_mmco[6], g->stat_idr_long);
	return 0;
}
