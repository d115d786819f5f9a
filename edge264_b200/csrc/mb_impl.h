/* mb_impl.h — second half of the shared slice-data code: motion-vector prediction (8.4.1),
 * direct modes, macroblock_layer() and the slice_data() loop.  Same two-direction convention as
 * syntax_impl.h.  Reference counterparts: edge264_mvpred.c:44-515 (prediction, P_Skip, direct),
 * edge264_slice.c:783-1849 (macroblock parsing) — restated from the standard, no pixel work. */
#ifndef E264B_MB_IMPL_H
#define E264B_MB_IMPL_H
#include "syntax_impl.h"

#ifdef E264_ENCODER
/* what the chooser (tools/gen264.c) decided for the macroblock being written */
typedef struct MbSyn {
	int skip;
	int mb_type;              /* numbering of the slice type (P: 0..4 then 5+I; B: 0..22 then 23+I; I: 0..25) */
	int t8x8;
	int sub_type[4];
	int ref_idx[2][4];        /* per partition */
	int16_t mv[2][16][2];     /* wanted absolute mv, indexed by z of the (sub-)partition's top-left 4x4 */
	int ipm[16];              /* wanted Intra4x4PredMode per z (Intra8x8: at z = 4*i8) */
	int chroma_mode, cbp, qp_delta;
	uint8_t pcm[384];
} MbSyn;
#define SYN(f) (s->syn->f)
#else
#define SYN(f) 0
#endif

typedef struct NbMv { int avail, ref; int mv[2]; } NbMv;

/* ---- neighbour cache (dec.h MvCache) ---- */
static const uint8_t sx_mc_of_z[16] = {   /* cache index of luma4x4BlkIdx z */
	MC_IDX(0, 0), MC_IDX(1, 0), MC_IDX(0, 1), MC_IDX(1, 1), MC_IDX(2, 0), MC_IDX(3, 0), MC_IDX(2, 1), MC_IDX(3, 1),
	MC_IDX(0, 2), MC_IDX(1, 2), MC_IDX(0, 3), MC_IDX(1, 3), MC_IDX(2, 2), MC_IDX(3, 2), MC_IDX(2, 3), MC_IDX(3, 3)};
/* bit wi (0: w4 = 1, 1: w4 = 2, 2: w4 = 4) of entry z: the block right of and above a partition of that width starting at
 * z lies inside this macroblock but later in decoding order, or right of the macroblock in its own row: neighbour C is
 * not available and D takes its place (6.4.11.7) */
static uint8_t sx_c_later[16];
static void sx_init_c_later(void) {
	for (int z = 0; z < 16; z++) {
		int x4 = e264_blk_x(z), y4 = e264_blk_y(z), m = 0;
		for (int wi = 0; wi < 3; wi++) {
			int cx = x4 + (1 << wi), cy = y4 - 1;
			if (cy >= 0 && (cx >= 4 || e264_blk_z(cx, cy) > z)) m |= 1 << wi;
		}
		sx_c_later[z] = (uint8_t)m;
	}
}

static inline void sx_cache_nb(SliceCtx *s, int l, int idx, const MbInfo *m, const E264MbRec *r, int z) {
	MvCache *c = &s->mc;
	if (!m) { c->mv[l][idx] = 0; c->ref[l][idx] = -2; c->mvd[l][idx] = 0; return; }
	int ref = r->ref_idx[l][z >> 2];
	c->ref[l][idx] = (int8_t)ref;
	c->mv[l][idx] = ref >= 0 ? ((const uint32_t *)r->mv[l])[z] : 0;
	c->mvd[l][idx] = ((const uint16_t *)m->mvd[l])[z];
}
/* the four neighbours 16x16 prediction looks at (P_Skip, spatial direct, 16x16 partitions): A0, B0, C, D */
static inline void sx_cache_corners(SliceCtx *s, int nl) {
	for (int l = 0; l < nl; l++) {
		sx_cache_nb(s, l, MC_IDX(-1, 0), s->A, s->recA, 5);
		sx_cache_nb(s, l, MC_IDX(0, -1), s->B, s->recB, 10);
		sx_cache_nb(s, l, MC_IDX(4, -1), s->C, s->recC, 10);
		sx_cache_nb(s, l, MC_IDX(-1, -1), s->D, s->recD, 15);
	}
}
static inline void sx_cache_fill(SliceCtx *s, int nl) {
	MvCache *c = &s->mc;
	sx_cache_corners(s, nl);
	for (int l = 0; l < nl; l++) {
		sx_cache_nb(s, l, MC_IDX(-1, 1), s->A, s->recA, 7); sx_cache_nb(s, l, MC_IDX(-1, 2), s->A, s->recA, 13); sx_cache_nb(s, l, MC_IDX(-1, 3), s->A, s->recA, 15);
		sx_cache_nb(s, l, MC_IDX(1, -1), s->B, s->recB, 11); sx_cache_nb(s, l, MC_IDX(2, -1), s->B, s->recB, 14); sx_cache_nb(s, l, MC_IDX(3, -1), s->B, s->recB, 15);
		for (int y = 0; y < 4; y++) {
			int i = MC_IDX(0, y);
			c->mv[l][i] = c->mv[l][i + 1] = c->mv[l][i + 2] = c->mv[l][i + 3] = c->mv[l][i + 4] = 0;
			c->ref[l][i] = c->ref[l][i + 1] = c->ref[l][i + 2] = c->ref[l][i + 3] = -1; c->ref[l][i + 4] = -2;   /* x4 = 4 in the own row: not decoded yet */
			c->mvd[l][i] = c->mvd[l][i + 1] = c->mvd[l][i + 2] = c->mvd[l][i + 3] = 0;
		}
	}
}
/* blocks derived in direct mode were written to the record: mirror them (they are neighbours of what follows) */
static inline void sx_cache_from_rec(SliceCtx *s, int mask8) {
	MvCache *c = &s->mc; const E264MbRec *r = s->rec;
	for (int l = 0; l < 2; l++) for (int z = 0; z < 16; z++) if ((mask8 >> (z >> 2)) & 1) {
		c->mv[l][sx_mc_of_z[z]] = ((const uint32_t *)r->mv[l])[z]; c->ref[l][sx_mc_of_z[z]] = r->ref_idx[l][z >> 2];
	}
}
/* interior -> record / MbInfo at the end of an inter macroblock */
static inline void sx_cache_flush(SliceCtx *s, int nl) {
	const MvCache *c = &s->mc;
	for (int l = 0; l < nl; l++) {
		uint32_t *mv = (uint32_t *)s->rec->mv[l]; uint16_t *mvd = (uint16_t *)s->cur->mvd[l];
		for (int z = 0; z < 16; z++) { mv[z] = c->mv[l][sx_mc_of_z[z]]; mvd[z] = c->mvd[l][sx_mc_of_z[z]]; }
	}
}
static inline int sx_median(int a, int b, int c) { int mx = a > b ? a : b, mn = a < b ? a : b; return c > mx ? mx : c < mn ? mn : c; }

/* 8.4.1.3: prediction for the partition whose top-left 4x4 is (x4,y4), w4 wide; the cache holds its neighbourhood.
 * shape: 0 generic, 1 = 16x8, 2 = 8x16 (directional rules) */
static inline void sx_mvpred(SliceCtx *s, int list, int x4, int y4, int w4, int ref, int shape, int mvp[2]) {
	const MvCache *c = &s->mc;
	const int8_t *rf = c->ref[list]; const uint32_t *mv = c->mv[list];
	const int idx = MC_IDX(x4, y4);
	int ic = idx - 8 + w4;
	if (rf[ic] == -2 || ((sx_c_later[e264_blk_z(x4, y4)] >> (w4 >> 1)) & 1)) ic = idx - 9;
	const int ra = rf[idx - 1], rb = rf[idx - 8], rc = rf[ic];
	uint32_t pick;
	if (shape == 1 && (y4 == 0 ? rb == ref : ra == ref)) pick = y4 == 0 ? mv[idx - 8] : mv[idx - 1];
	else if (shape == 2 && (x4 == 0 ? ra == ref : rc == ref)) pick = x4 == 0 ? mv[idx - 1] : mv[ic];
	else if (rb == -2 && rc == -2 && ra != -2) pick = mv[idx - 1];
	else {
		const int ea = ra == ref, eb = rb == ref, ec = rc == ref;
		if (ea + eb + ec == 1) pick = ea ? mv[idx - 1] : eb ? mv[idx - 8] : mv[ic];
		else {
			const uint32_t a = mv[idx - 1], b = mv[idx - 8], cc = mv[ic];
			mvp[0] = sx_median((int16_t)a, (int16_t)b, (int16_t)cc);
			mvp[1] = sx_median((int16_t)(a >> 16), (int16_t)(b >> 16), (int16_t)(cc >> 16));
			return;
		}
	}
	mvp[0] = (int16_t)pick; mvp[1] = (int16_t)(pick >> 16);
}

static inline void sx_cache_rect32(uint32_t *a, int idx, int w4, int h4, uint32_t v) { for (int y = 0; y < h4; y++) for (int x = 0; x < w4; x++) a[idx + y * 8 + x] = v; }
static inline void sx_cache_rect16(uint16_t *a, int idx, int w4, int h4, uint16_t v) { for (int y = 0; y < h4; y++) for (int x = 0; x < w4; x++) a[idx + y * 8 + x] = v; }
/* z-order makes 16x16, 16x8 and 8x8 partitions contiguous runs of the per-4x4 arrays (record side: skip and direct) */
static inline void sx_fill_mv(SliceCtx *s, int list, int x4, int y4, int w4, int h4, int mvx, int mvy) {
	uint32_t v = (uint16_t)mvx | ((uint32_t)(uint16_t)mvy << 16);
	uint32_t *dst = (uint32_t *)s->rec->mv[list];
	if (w4 == 4 && h4 == 4) { for (int z = 0; z < 16; z++) dst[z] = v; return; }
	if (w4 == 4 && h4 == 2) { int z0 = y4 * 4; for (int z = z0; z < z0 + 8; z++) dst[z] = v; return; }
	if (w4 == 2 && h4 == 2) { int z0 = e264_blk_z(x4, y4); dst[z0] = dst[z0 + 1] = dst[z0 + 2] = dst[z0 + 3] = v; return; }
	for (int y = y4; y < y4 + h4; y++) for (int x = x4; x < x4 + w4; x++) dst[e264_blk_z(x, y)] = v;
}
/* reference index of an 8x8 quadrant: record and cache */
static inline void sx_set_ref(SliceCtx *s, int list, int i8, int ref) {
	s->rec->ref_idx[list][i8] = (int8_t)ref;
	s->rec->ref_pic[list][i8] = ref >= 0 ? s->ref_slot[list][ref & 31] : -1;
	int8_t *rf = s->mc.ref[list] + MC_IDX((i8 & 1) * 2, (i8 >> 1) * 2);
	rf[0] = rf[1] = rf[8] = rf[9] = (int8_t)ref;
}

/* P_Skip (8.4.1.1) */
static void sx_p_skip_motion(SliceCtx *s) {
	int mvp[2] = {0, 0};
	sx_cache_corners(s, 1);
	const MvCache *c = &s->mc;
	const int ia = MC_IDX(-1, 0), ib = MC_IDX(0, -1);
	if (s->A && s->B && !(c->ref[0][ia] == 0 && c->mv[0][ia] == 0) && !(c->ref[0][ib] == 0 && c->mv[0][ib] == 0))
		sx_mvpred(s, 0, 0, 0, 4, 0, 0, mvp);
	for (int i = 0; i < 4; i++) {
		s->rec->ref_idx[0][i] = 0; s->rec->ref_pic[0][i] = s->ref_slot[0][0];
		s->rec->ref_idx[1][i] = -1; s->rec->ref_pic[1][i] = -1;
	}
	sx_fill_mv(s, 0, 0, 0, 4, 4, mvp[0], mvp[1]);
}

/* co-located 4x4 block info for direct prediction (8.4.1.2.1, frame pictures only) */
static inline int sx_col(SliceCtx *s, int z, int *ref_idx, int mv[2], int *ref_slot) {
	if (!s->col_recs) return 0;
	const E264MbRec *c = s->col_recs + s->mbaddr;
	if (c->kind != MBK_INTER) return 0;
	int l = c->ref_idx[0][z >> 2] >= 0 ? 0 : 1;
	if (c->ref_idx[l][z >> 2] < 0) return 0;
	*ref_idx = c->ref_idx[l][z >> 2]; *ref_slot = c->ref_pic[l][z >> 2];
	mv[0] = c->mv[l][z][0]; mv[1] = c->mv[l][z][1];
	return 1;
}
static inline int sx_minpos(int a, int b) { return (a >= 0 && b >= 0) ? (a < b ? a : b) : (a > b ? a : b); }

/* B direct prediction for the 8x8 blocks selected by mask8 (8.4.1.2.2 spatial / 8.4.1.2.3 temporal) */
static void sx_direct_motion(SliceCtx *s, int mask8) {
	static const uint8_t corner[4] = {0, 5, 10, 15};
	if (s->direct_spatial) {
		int ref[2], mvp[2][2] = {{0, 0}, {0, 0}};
		const MvCache *c = &s->mc;     /* corners filled by the caller */
		for (int l = 0; l < 2; l++) {
			int ic = MC_IDX(4, -1);
			if (c->ref[l][ic] == -2) ic = MC_IDX(-1, -1);
			int ra = c->ref[l][MC_IDX(-1, 0)], rb = c->ref[l][MC_IDX(0, -1)], rc = c->ref[l][ic];
			ref[l] = sx_minpos(ra < 0 ? -1 : ra, sx_minpos(rb < 0 ? -1 : rb, rc < 0 ? -1 : rc));
		}
		if (ref[0] < 0 && ref[1] < 0) ref[0] = ref[1] = 0;
		else for (int l = 0; l < 2; l++) if (ref[l] >= 0) sx_mvpred(s, l, 0, 0, 4, ref[l], 0, mvp[l]);
		/* note: mvpred above reads only neighbours OUTSIDE the current macroblock (16x16 geometry) */
		for (int i8 = 0; i8 < 4; i8++) {
			if (!((mask8 >> i8) & 1)) continue;
			for (int l = 0; l < 2; l++) sx_set_ref(s, l, i8, ref[l]);
			for (int j = 0; j < 4; j++) {
				int z = i8 * 4 + j;
				int cz = s->direct_8x8_inference ? corner[i8] : z;
				int cref, cmv[2], cslot;
				int col_zero = !s->ref_long[1][0] && sx_col(s, cz, &cref, cmv, &cslot) && cref == 0 &&
				               cmv[0] >= -1 && cmv[0] <= 1 && cmv[1] >= -1 && cmv[1] <= 1;
				for (int l = 0; l < 2; l++) {
					int zero = ref[l] < 0 || (ref[l] == 0 && col_zero);
					s->rec->mv[l][z][0] = (int16_t)(zero ? 0 : mvp[l][0]);
					s->rec->mv[l][z][1] = (int16_t)(zero ? 0 : mvp[l][1]);
				}
			}
		}
	} else {
		for (int i8 = 0; i8 < 4; i8++) {
			if (!((mask8 >> i8) & 1)) continue;
			for (int j = 0; j < 4; j++) {
				int z = i8 * 4 + j;
				int cz = s->direct_8x8_inference ? corner[i8] : z;
				int cref, cmv[2] = {0, 0}, cslot, r0 = 0, m0[2] = {0, 0}, m1[2] = {0, 0};
				if (sx_col(s, cz, &cref, cmv, &cslot)) {
					int32_t uid = (cslot >= 0 && cslot < E264_MAX_SLOTS) ? s->col_slot_uid[cslot] : -1;
					for (int k = 0; k < s->num_ref[0]; k++) if (s->ref_uid[0][k] == uid) { r0 = k; break; }
					int tb = s->cur_poc - s->ref_poc[0][r0], td = s->ref_poc[1][0] - s->ref_poc[0][r0];
					tb = tb < -128 ? -128 : tb > 127 ? 127 : tb; td = td < -128 ? -128 : td > 127 ? 127 : td;
					if (s->ref_long[0][r0] || td == 0) { m0[0] = cmv[0]; m0[1] = cmv[1]; }
					else {
						int tx = (16384 + (td < 0 ? -td : td) / 2) / td;
						int dsf = (tb * tx + 32) >> 6; dsf = dsf < -1024 ? -1024 : dsf > 1023 ? 1023 : dsf;
						m0[0] = (dsf * cmv[0] + 128) >> 8; m0[1] = (dsf * cmv[1] + 128) >> 8;
						m1[0] = m0[0] - cmv[0]; m1[1] = m0[1] - cmv[1];
					}
				}
				if (j == 0 || !s->direct_8x8_inference || 1) { sx_set_ref(s, 0, i8, r0); sx_set_ref(s, 1, i8, 0); }
				s->rec->mv[0][z][0] = (int16_t)m0[0]; s->rec->mv[0][z][1] = (int16_t)m0[1];
				s->rec->mv[1][z][0] = (int16_t)m1[0]; s->rec->mv[1][z][1] = (int16_t)m1[1];
			}
		}
	}
}

/* chroma QPs and record flags common to every macroblock */
static inline int sx_qpc(SliceCtx *s, int qpy, int pl) {
	int q = qpy + s->chroma_qp_offset[pl];
	return h264_qpc[q < 0 ? 0 : q > 51 ? 51 : q];
}
static inline void sx_finish_rec(SliceCtx *s, int qp_for_deblock) {
	E264MbRec *r = s->rec;
	r->qp[0] = (uint8_t)qp_for_deblock; r->qp[1] = (uint8_t)sx_qpc(s, qp_for_deblock, 0); r->qp[2] = (uint8_t)sx_qpc(s, qp_for_deblock, 1);
	r->slice_idx = (uint8_t)s->slice_idx;
	if (s->deblock_idc != 1) {
		r->flags |= MBF_DEBLOCK;
		if (s->mbx > 0 && (s->deblock_idc == 0 || s->A)) r->flags |= MBF_EDGE_L;
		if (s->mby > 0 && (s->deblock_idc == 0 || s->B)) r->flags |= MBF_EDGE_T;
	}
}

static void sx_skip_mb(SliceCtx *s) {
	MbInfo *m = s->cur; E264MbRec *r = s->rec;
	m->is_skip = 1;
	r->kind = MBK_INTER; r->flags |= MBF_SKIP;
	memset(m->ipm, 2, 16);
	if (s->slice_type == SLICE_P) sx_p_skip_motion(s);
	else { m->is_direct = 1; m->direct8 = 15; if (s->direct_spatial) sx_cache_corners(s, 2); sx_direct_motion(s, 15); }
	s->last_qp_delta_nz = 0;
	r->coef_off = s->n_coefs;
	sx_finish_rec(s, s->qp);
}

/* B macroblock types 1..21: prediction use of the two partitions, bit0 = L0, bit1 = L1 */
static const uint8_t sx_b_part_pred[9][2] = {{1, 1}, {2, 2}, {1, 2}, {2, 1}, {1, 3}, {2, 3}, {3, 1}, {3, 2}, {3, 3}};
static const uint8_t sx_b_sub_pred[13] = {0, 1, 2, 3, 1, 1, 2, 2, 3, 3, 1, 2, 3};
static const uint8_t sx_b_sub_shape[13] = {0, 0, 0, 0, 1, 2, 1, 2, 1, 2, 3, 3, 3};   /* 0 8x8, 1 8x4, 2 4x8, 3 4x4 */

/* mvd_lX (9.3.2.3 UEG3, 9.3.3.1.1.7) on the register-resident engine; absum = |mvd| of the neighbours A and B */
#define SE_EGK_BYP_R(k0, v) ({ int k_ = (k0), val_ = 0, v_ = (v); (void)v_; \
	while (AE_BYP_R(ENCV(v_ >= (1 << k_)))) { val_ += 1 << k_; v_ -= ENCV(1 << k_); if (++k_ > 24) { s->error = 1; break; } } \
	while (k_--) val_ += AE_BYP_R(ENCV((v_ >> k_) & 1)) << k_; \
	val_; })
#define SE_MVD_R(comp, absum, v) ({ const int base_ = (comp) ? 47 : 40, sum_ = (absum), w_ = (v); (void)w_; \
	const int a_ = ENCV(w_ < 0 ? -w_ : w_); (void)a_; int n_ = 0; \
	if (AE_R(base_ + (sum_ < 3 ? 0 : sum_ > 32 ? 2 : 1), ENCV(a_ > 0))) { \
		int ctx_ = base_ + 3; n_ = 1; \
		while (n_ < 9 && AE_R(ctx_, ENCV(a_ > n_))) { if (n_ < 4) ctx_++; n_++; } \
		if (n_ >= 9) n_ = 9 + SE_EGK_BYP_R(3, ENCV(a_ - 9)); \
		if (AE_BYP_R(ENCV(w_ < 0))) n_ = -n_; \
	} \
	n_; })

/* mvd + prediction for one (sub-)partition */
static void sx_mv_part(SliceCtx *s, int list, int x4, int y4, int w4, int h4, int ref, int shape) {
	int mvp[2];
	sx_mvpred(s, list, x4, y4, w4, ref, shape, mvp);
	MvCache *c = &s->mc;
	const int idx = MC_IDX(x4, y4);
	const unsigned na = c->mvd[list][idx - 1], nb = c->mvd[list][idx - 8];
	const int sx = (int)(na & 255) + (int)(nb & 255), sy = (int)(na >> 8) + (int)(nb >> 8);
	int z = e264_blk_z(x4, y4); (void)z;
	int dx, dy;
	if (!s->cabac) {
		dx = VLC_SE(ENCV(SYN(mv[list][z][0]) - mvp[0]));
		dy = VLC_SE(ENCV(SYN(mv[list][z][1]) - mvp[1]));
	} else {
		CR_BEGIN
		dx = SE_MVD_R(0, sx, ENCV(SYN(mv[list][z][0]) - mvp[0]));
		dy = SE_MVD_R(1, sy, ENCV(SYN(mv[list][z][1]) - mvp[1]));
		CR_OUT
	}
	int ax = dx < 0 ? -dx : dx, ay = dy < 0 ? -dy : dy;
	if (ax > 255) ax = 255;
	if (ay > 255) ay = 255;
	sx_cache_rect32(c->mv[list], idx, w4, h4, (uint16_t)(mvp[0] + dx) | ((uint32_t)(uint16_t)(mvp[1] + dy) << 16));
	sx_cache_rect16(c->mvd[list], idx, w4, h4, (uint16_t)(ax | (ay << 8)));
}

static void sx_intra_common_tail(SliceCtx *s, int is_i16, int cbp_known, int cbp);

static void sx_macroblock(SliceCtx *s) {
	MbInfo *m = s->cur; E264MbRec *r = s->rec;
	int st = s->slice_type;
	int mbt = st == SLICE_I ? se_mb_type_intra(s, ENCV(SYN(mb_type)), 3, 1) : st == SLICE_P ? se_mb_type_P(s, ENCV(SYN(mb_type))) : se_mb_type_B(s, ENCV(SYN(mb_type)));
	int ityp = st == SLICE_I ? mbt : st == SLICE_P ? mbt - 5 : mbt - 23;   /* >= 0: intra */
	r->coef_off = s->n_coefs;
	for (int l = 0; l < 2; l++) for (int i = 0; i < 4; i++) { r->ref_idx[l][i] = -1; r->ref_pic[l][i] = -1; }
	memset(m->ipm, 2, 16);
	if (ityp > 25 || (st == SLICE_P && mbt > 30) || (st == SLICE_B && mbt > 48)) { s->error = 1; return; }

	if (ityp >= 0) {
		m->is_intra = 1; s->n_intra++;
		if (ityp == 25) {   /* I_PCM (7.3.5: pcm_alignment_zero_bit, 384 samples) */
			m->is_pcm = 1; r->kind = MBK_IPCM;
			int16_t *dst = sx_pool_take(s, 192, 0);
#ifdef E264_ENCODER
			memcpy(dst, s->syn->pcm, 384);
			bw_align_zero(s->bw);
			bw_bytes(s->bw, s->syn->pcm, 384);
			if (s->cabac) cabac_enc_start(&s->ce, s->bw);
#else
			if (s->cabac) {
				const uint8_t *p = cabac_dec_aligned_pos(&s->cd);
				if (p + 384 > s->cd.end) { s->error = 1; return; }
				memcpy(dst, p, 384);
				cabac_dec_start(&s->cd, p + 384, s->cd.end);
			} else {
				s->br.pos = (s->br.pos + 7) & ~(size_t)7;
				if ((s->br.pos >> 3) + 384 > s->br.size) { s->error = 1; return; }
				memcpy(dst, s->br.buf + (s->br.pos >> 3), 384);
				s->br.pos += 384 * 8;
			}
			if (s->luma_only) memset((uint8_t *)dst + 256, 128, 128);   /* luma only: the chroma samples are 128 (edge264_luma.h) */
#endif
			m->cbp = 0x2f; m->cbf_dc = 7; m->cbf_luma = 0xffff; m->cbf_cb = m->cbf_cr = 15;
			memset(m->tc, 16, 24);
			s->last_qp_delta_nz = 0;
			sx_finish_rec(s, 0);      /* deblocking sees qP = 0 for I_PCM (8.7.2.2); QP_Y prediction chain is unchanged */
			return;
		}
		int cbp;
		if (ityp == 0) {
			int t8 = s->transform_8x8_mode ? se_transform_8x8_flag(s, ENCV(SYN(t8x8))) : 0;
			m->t8x8 = (uint8_t)t8;
			if (t8) {
				r->kind = MBK_I8x8; r->flags |= MBF_T8x8;
				for (int i8 = 0; i8 < 4; i8++) {
					int pred = sx_pred_intra_mode(s, (i8 & 1) * 2, (i8 >> 1) * 2);
					int want = ENCV(SYN(ipm[i8 * 4]));
					int rem = se_intra_pred_mode(s, ENCV(want == pred ? -1 : want < pred ? want : want - 1));
					int mode = rem < 0 ? pred : rem + (rem >= pred), un = sx_unavail8x8(s, i8);
					if (!e264_intra_mode_legal(MBK_I8x8, mode, un)) { s->error = 1; mode = 2; }   /* reads a neighbour that is not there: DC */
					memset(m->ipm + i8 * 4, mode, 4);
					r->modes[i8] = IMODE(mode, un);
				}
			} else {
				r->kind = MBK_I4x4;
				for (int b = 0; b < 16; b++) {
					int pred = sx_pred_intra_mode(s, e264_blk_x(b), e264_blk_y(b));
					int want = ENCV(SYN(ipm[b]));
					int rem = se_intra_pred_mode(s, ENCV(want == pred ? -1 : want < pred ? want : want - 1));
					int mode = rem < 0 ? pred : rem + (rem >= pred), un = sx_unavail4x4(s, b);
					if (!e264_intra_mode_legal(MBK_I4x4, mode, un)) { s->error = 1; mode = 2; }
					m->ipm[b] = (int8_t)mode;
					r->modes[b] = IMODE(mode, un);
				}
			}
		} else {
			m->is_i16 = 1; r->kind = MBK_I16x16;
			int mode = (ityp - 1) & 3;
			if (!e264_intra_mode_legal(MBK_I16x16, mode, sx_unavail16(s))) { s->error = 1; mode = 2; }
			r->i16_mode = IMODE(mode, sx_unavail16(s));
		}
		int cm = se_intra_chroma_pred_mode(s, ENCV(SYN(chroma_mode)));
		if (cm > 3) { s->error = 1; return; }
		if (!e264_intra_mode_legal(-1, cm, sx_unavail16(s))) { s->error = 1; cm = 0; }
		m->chroma_pred_mode = (uint8_t)cm;
		r->chroma_mode = IMODE(cm, sx_unavail16(s));
		if (ityp == 0) cbp = se_coded_block_pattern(s, ENCV(SYN(cbp)), 1);
		else cbp = (((ityp - 1) >> 2) % 3) << 4 | ((ityp - 1) >= 12 ? 15 : 0);
		m->cbp = (uint8_t)cbp;
		sx_intra_common_tail(s, ityp != 0, 1, cbp);
		return;
	}

	/* ---- inter ---- */
	r->kind = MBK_INTER;
	int is_b = st == SLICE_B;
	const int nl = is_b ? 2 : 1;
	int no_sub8 = 1;      /* noSubMbPartSizeLessThan8x8Flag */
	if (is_b && mbt == 0) {                    /* B_Direct_16x16 */
		m->is_direct = 1; m->direct8 = 15;
		if (s->direct_spatial) sx_cache_corners(s, 2);
		sx_direct_motion(s, 15);
		no_sub8 = s->direct_8x8_inference;
	} else if ((!is_b && mbt >= 3) || (is_b && mbt == 22)) {   /* 8x8 sub-macroblocks */
		int sub[4], pred8[4], shape8[4];
		for (int i = 0; i < 4; i++) {
			sub[i] = is_b ? se_sub_mb_type_B(s, ENCV(SYN(sub_type[i]))) : se_sub_mb_type_P(s, ENCV(SYN(sub_type[i])));
			if (sub[i] > (is_b ? 12 : 3)) { s->error = 1; return; }
			pred8[i] = is_b ? sx_b_sub_pred[sub[i]] : 1;
			shape8[i] = is_b ? sx_b_sub_shape[sub[i]] : sub[i];
			if (is_b && sub[i] == 0) { m->direct8 |= 1 << i; if (!s->direct_8x8_inference) no_sub8 = 0; }
			else if (shape8[i]) no_sub8 = 0;
		}
		sx_cache_fill(s, nl);
		if (m->direct8) { sx_direct_motion(s, m->direct8); sx_cache_from_rec(s, m->direct8); }
		for (int l = 0; l < 2; l++) for (int i = 0; i < 4; i++) {
			if (!(pred8[i] & (1 << l))) continue;
			int ref = 0;
			if (s->num_ref[l] > 1 && !(!is_b && mbt == 4)) ref = se_ref_idx(s, l, i, ENCV(SYN(ref_idx[l][i])));
			if (ref >= s->num_ref[l]) { s->error = 1; ref = 0; }
			sx_set_ref(s, l, i, ref);
		}
		for (int l = 0; l < 2; l++) for (int i = 0; i < 4; i++) {
			if (!(pred8[i] & (1 << l))) continue;
			int x0 = (i & 1) * 2, y0 = (i >> 1) * 2, ref = r->ref_idx[l][i];
			switch (shape8[i]) {
			case 0: sx_mv_part(s, l, x0, y0, 2, 2, ref, 0); break;
			case 1: sx_mv_part(s, l, x0, y0, 2, 1, ref, 0); sx_mv_part(s, l, x0, y0 + 1, 2, 1, ref, 0); break;
			case 2: sx_mv_part(s, l, x0, y0, 1, 2, ref, 0); sx_mv_part(s, l, x0 + 1, y0, 1, 2, ref, 0); break;
			default: for (int j = 0; j < 4; j++) sx_mv_part(s, l, x0 + (j & 1), y0 + (j >> 1), 1, 1, ref, 0);
			}
		}
		sx_cache_flush(s, nl);
	} else {
		/* 16x16, 16x8, 8x16 */
		int shape, p0, p1;
		if (!is_b) { shape = mbt; p0 = p1 = 1; }
		else if (mbt <= 3) { shape = 0; p0 = p1 = mbt; }
		else { shape = 1 + ((mbt - 4) & 1); p0 = sx_b_part_pred[(mbt - 4) >> 1][0]; p1 = sx_b_part_pred[(mbt - 4) >> 1][1]; }
		int nparts = shape ? 2 : 1;
		int pp[2] = {p0, p1}, refs[2][2] = {{-1, -1}, {-1, -1}};
		sx_cache_fill(s, nl);
		for (int l = 0; l < 2; l++) for (int p = 0; p < nparts; p++) {
			if (!(pp[p] & (1 << l))) continue;
			int ref = 0;
			int i8 = shape == 0 ? 0 : shape == 1 ? p * 2 : p;
			if (s->num_ref[l] > 1) ref = se_ref_idx(s, l, i8, ENCV(SYN(ref_idx[l][p])));
			if (ref >= s->num_ref[l]) { s->error = 1; ref = 0; }
			refs[l][p] = ref;
			if (shape == 0) for (int i = 0; i < 4; i++) sx_set_ref(s, l, i, ref);
			else if (shape == 1) { sx_set_ref(s, l, p * 2, ref); sx_set_ref(s, l, p * 2 + 1, ref); }
			else { sx_set_ref(s, l, p, ref); sx_set_ref(s, l, p + 2, ref); }
		}
		for (int l = 0; l < 2; l++) for (int p = 0; p < nparts; p++) {
			if (!(pp[p] & (1 << l))) continue;
			if (shape == 0) sx_mv_part(s, l, 0, 0, 4, 4, refs[l][p], 0);
			else if (shape == 1) sx_mv_part(s, l, 0, p * 2, 4, 2, refs[l][p], 1);
			else sx_mv_part(s, l, p * 2, 0, 2, 4, refs[l][p], 2);
		}
		sx_cache_flush(s, nl);
	}
	int cbp = se_coded_block_pattern(s, ENCV(SYN(cbp)), 0);
	m->cbp = (uint8_t)cbp;
	if ((cbp & 15) && s->transform_8x8_mode && no_sub8) {
		m->t8x8 = (uint8_t)se_transform_8x8_flag(s, ENCV(SYN(t8x8)));
		if (m->t8x8) r->flags |= MBF_T8x8;
	}
	sx_intra_common_tail(s, 0, 1, cbp);
}

/* mb_qp_delta + residual + record completion (shared by intra and inter macroblocks) */
static void sx_intra_common_tail(SliceCtx *s, int is_i16, int cbp_known, int cbp) {
	(void)cbp_known;
	if (cbp || is_i16) {
		int d = se_mb_qp_delta(s, ENCV(SYN(qp_delta)));
		if (d < -26 || d > 25) { s->error = 1; d = 0; }
		s->last_qp_delta_nz = d != 0;
		s->qp = (s->qp + d + 52) % 52;
		sx_residual(s, is_i16, cbp);
	} else {
		s->last_qp_delta_nz = 0;
		s->rec->coded = 0;
	}
	sx_finish_rec(s, s->qp);
}

/* one macroblock of slice_data(); returns 1 when the slice ends after it */
static int sx_one_mb(SliceCtx *s) {
	s->mbx = s->mbaddr % s->w_mbs; s->mby = s->mbaddr / s->w_mbs;
	sx_set_neighbours(s);
	memset(s->cur, 0, sizeof(MbInfo)); s->cur->slice_id = (uint16_t)s->slice_id;
	memset(s->rec, 0, sizeof(E264MbRec));
	int skip = 0;
	if (s->slice_type != SLICE_I) {
		if (s->cabac) skip = se_mb_skip_flag(s, ENCV(SYN(skip)));
		else {
#ifdef E264_ENCODER
			skip = SYN(skip);
			if (skip) s->skip_run++; else { bw_ue(s->bw, s->skip_run); s->skip_run = 0; }
#else
			if (s->skip_run == -1) { s->skip_run = (int)br_ue(&s->br); if (s->skip_run == 0) s->skip_run = -2; }
			if (s->skip_run > 0) { skip = 1; s->skip_run--; if (s->skip_run == 0) s->skip_run = br_more_rbsp_data(&s->br) ? -2 : -3; }
			else s->skip_run = -1;   /* -2: a coded macroblock follows, then a new run is read */
#endif
		}
	}
	if (skip) sx_skip_mb(s); else sx_macroblock(s);
	if (s->error) return 1;
	if (s->cabac) {
#ifdef E264_ENCODER
		return 0;    /* the writer terminates explicitly (it knows the last macroblock) */
#else
		return cabac_terminate(&s->cd);
#endif
	}
#ifndef E264_ENCODER
	if (skip) return s->skip_run == -3;
	return !br_more_rbsp_data(&s->br);
#else
	return 0;
#endif
}
#endif
