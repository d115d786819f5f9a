/* syntax_impl.h — slice_data() / macroblock_layer() of ITU-T H.264 (7.3.4, 7.3.5) written ONCE and
 * compiled in two directions:
 *   - default:            PARSER  (product): bitstream -> E264MbRec records + coefficient pool
 *   - -DE264_ENCODER:     WRITER  (tools/gen264.c, test infrastructure): random syntax -> bitstream,
 *                         producing the same records as a by-product
 * Every syntax-element routine has the form  v = se_xxx(s, v): the parser ignores the argument and
 * returns what it read, the writer emits the argument and returns it.  Context-index derivations
 * (9.3.3.1.1) and neighbour bookkeeping are therefore shared, and the reference decoder (compiled as
 * the oracle) arbitrates that this shared understanding is the standard's.
 *
 * Replaces the reference's parse_slice_data / parse_{I,P,B}_mb / parse_*_residual and the MV
 * prediction they call (reference: edge264_slice.c:82-1849, edge264_mvpred.c:44-515), minus every
 * pixel operation: where the reference calls its decode_intra, decode_inter and add_idct functions
 * from inside the parser, this code only fills the record. */
#ifndef E264B_SYNTAX_IMPL_H
#define E264B_SYNTAX_IMPL_H
#include "dec.h"

#ifdef E264_ENCODER
#define ENCV(x)      (x)
#define AE(ctx, v)   cabac_enc_bin(&s->ce, (ctx), (v))
#define AE_BYP(v)    cabac_enc_bypass(&s->ce, (v))
#define AE_TERM(v)   cabac_enc_terminate(&s->ce, (v))
#define VLC_UE(v)    (bw_ue(s->bw, (uint32_t)(v)), (int)(v))
#define VLC_SE(v)    (bw_se(s->bw, (v)), (int)(v))
#define VLC_U(n, v)  (bw_u(s->bw, (n), (uint32_t)(v)), (int)(v))
#else
#define ENCV(x)      0
#define AE(ctx, v)   cabac_bin(&s->cd, (ctx))
#define AE_BYP(v)    cabac_bypass(&s->cd)
#define AE_TERM(v)   cabac_terminate(&s->cd)
#define VLC_UE(v)    ((int)br_ue(&s->br))
#define VLC_SE(v)    ((int)br_se(&s->br))
#define VLC_U(n, v)  ((int)br_u(&s->br, (n)))
#endif

/* register-resident CABAC state for the residual parser (parser direction only) */
#ifdef E264_ENCODER
#define CR_BEGIN
#define CR_OUT
#define CR_IN
#define AE_R(ctx, v)  AE(ctx, v)
#define AE_BYP_R(v)   AE_BYP(v)
#else
#define CR_BEGIN      CabacRegs cr = cabac_regs_load(&s->cd); CabacState *const cst = s->cd.state;
#define CR_OUT        cabac_regs_store(&s->cd, &cr);
#define CR_IN         cr = cabac_regs_load(&s->cd);
#define AE_R(ctx, v)  cabac_r_bin(&cr, cst, (ctx))
#define AE_BYP_R(v)   cabac_r_bypass(&cr)
#endif

enum { SLICE_P = 0, SLICE_B = 1, SLICE_I = 2 };

/* ------------------------------------------------------------------------------------------ */
/* neighbour helpers                                                                            */
/* ------------------------------------------------------------------------------------------ */
static inline void sx_set_neighbours(SliceCtx *s) {
	int a = s->mbaddr, w = s->w_mbs;
	MbInfo *m = s->mbi + a; E264MbRec *r = s->recs + a;
	s->cur = m; s->rec = r;
	int sid = s->slice_id;
	int hasA = s->mbx > 0 && m[-1].slice_id == sid;
	int hasB = s->mby > 0 && m[-w].slice_id == sid;
	int hasC = s->mby > 0 && s->mbx < w - 1 && m[-w + 1].slice_id == sid;
	int hasD = s->mby > 0 && s->mbx > 0 && m[-w - 1].slice_id == sid;
	s->A = hasA ? m - 1 : NULL;      s->recA = hasA ? r - 1 : NULL;
	s->B = hasB ? m - w : NULL;      s->recB = hasB ? r - w : NULL;
	s->C = hasC ? m - w + 1 : NULL;  s->recC = hasC ? r - w + 1 : NULL;
	s->D = hasD ? m - w - 1 : NULL;  s->recD = hasD ? r - w - 1 : NULL;
}

/* locate the 4x4 block at (x4,y4) relative to the current MB (each in -1..4).
 * returns 0 and *mi=NULL when outside the slice/picture or to the right (not yet decoded) */
static inline int sx_locate(SliceCtx *s, int x4, int y4, MbInfo **mi, E264MbRec **rec) {
	MbInfo *m; E264MbRec *r;
	if (y4 < 0) {
		if (x4 < 0) { m = s->D; r = s->recD; }
		else if (x4 < 4) { m = s->B; r = s->recB; }
		else { m = s->C; r = s->recC; }
	} else if (x4 < 0) { m = s->A; r = s->recA; }
	else if (x4 >= 4) { m = NULL; r = NULL; }
	else { m = s->cur; r = s->rec; }
	*mi = m; *rec = r;
	return e264_blk_z(x4 & 3, y4 & 3);
}

/* unavailability bits (A=1,B=2,C=4,D=8) of the neighbours of an Intra4x4 block (6.4.11.4) */
static inline int sx_unavail4x4(SliceCtx *s, int b) {
	int x = e264_blk_x(b), y = e264_blk_y(b), u = 0;
	if (x == 0 && !s->A) u |= 1;
	if (y == 0 && !s->B) u |= 2;
	if (y == 0) { if (x < 3 ? !s->B : !s->C) u |= 4; }
	else if (x == 3 || e264_blk_z(x + 1, y - 1) > b) u |= 4;
	if (x == 0 && y == 0) { if (!s->D) u |= 8; }
	else if (x == 0) { if (!s->A) u |= 8; }
	else if (y == 0) { if (!s->B) u |= 8; }
	return u;
}
static inline int sx_unavail8x8(SliceCtx *s, int i) {
	int u = 0;
	if (!(i & 1) && !s->A) u |= 1;
	if (!(i & 2) && !s->B) u |= 2;
	if (i == 0 ? !s->B : i == 1 ? !s->C : i == 3) u |= 4;
	if (i == 0 ? !s->D : i == 1 ? !s->B : i == 2 ? !s->A : 0) u |= 8;
	return u;
}
static inline int sx_unavail16(SliceCtx *s) { return (s->A ? 0 : 1) | (s->B ? 0 : 2) | (s->D ? 0 : 8); }

/* predIntra4x4PredMode / predIntra8x8PredMode (8.3.1.1, 8.3.2.1) for the block whose top-left 4x4 is (x4,y4) */
static inline int sx_pred_intra_mode(SliceCtx *s, int x4, int y4) {
	MbInfo *ma, *mb; E264MbRec *r;
	int za = sx_locate(s, x4 - 1, y4, &ma, &r);
	int zb = sx_locate(s, x4, y4 - 1, &mb, &r);
	if (!ma || !mb) return 2;
	int a = ma->is_intra ? ma->ipm[za] : 2;   /* inter neighbours predict DC (constrained_intra_pred_flag == 0) */
	int bm = mb->is_intra ? mb->ipm[zb] : 2;
	return a < bm ? a : bm;
}

/* ------------------------------------------------------------------------------------------ */
/* CABAC / CAVLC syntax elements                                                                */
/* ------------------------------------------------------------------------------------------ */
static int se_mb_skip_flag(SliceCtx *s, int v) {
	int ctx = (s->slice_type == SLICE_P ? 11 : 24) + (s->A && !s->A->is_skip) + (s->B && !s->B->is_skip);
	return AE(ctx, v);
}

/* I macroblock types: 0 = I_NxN, 1..24 = I_16x16_<pred>_<chroma>_<ac>, 25 = I_PCM (Table 7-11) */
static int se_mb_type_intra(SliceCtx *s, int v, int base, int intra_slice) {
	if (!s->cabac) return VLC_UE(v);
	if (intra_slice) {
		int inc = (s->A && !(s->A->is_intra && !s->A->is_i16 && !s->A->is_pcm)) + (s->B && !(s->B->is_intra && !s->B->is_i16 && !s->B->is_pcm));
		if (!AE(base + inc, ENCV(v != 0))) return 0;
		base += 2;
	} else {
		if (!AE(base, ENCV(v != 0))) return 0;
	}
	if (AE_TERM(ENCV(v == 25))) return 25;
	int t = ENCV(v - 1);   /* 0..23: pred = t&3, chroma = (t>>2)%3, ac = t>=12 */
	int ac = AE(base + 1, ENCV(t >= 12));
	int chroma = 0;
	if (AE(base + 2, ENCV((t >> 2) % 3 != 0)))
		chroma = 1 + AE(base + 2 + intra_slice, ENCV((t >> 2) % 3 == 2));
	int pred = AE(base + 3 + intra_slice, ENCV((t >> 1) & 1)) << 1;
	pred |= AE(base + 3 + 2 * intra_slice, ENCV(t & 1));
	return 1 + pred + 4 * chroma + 12 * ac;
}
/* P: 0..4 inter (Table 7-13), 5.. = 5 + intra type */
static int se_mb_type_P(SliceCtx *s, int v) {
	if (!s->cabac) { int t = VLC_UE(v); (void)t; return t; }
	if (!AE(14, ENCV(v >= 5))) {
		if (!AE(15, ENCV(v == 1 || v == 2))) return 3 * AE(16, ENCV(v == 3));
		return 2 - AE(17, ENCV(v == 1));
	}
	return 5 + se_mb_type_intra(s, ENCV(v - 5), 17, 0);
}
/* B: 0..22 inter (Table 7-14), 23.. = 23 + intra type */
static int se_mb_type_B(SliceCtx *s, int v) {
	if (!s->cabac) return VLC_UE(v);
	int inc = (s->A && !s->A->is_direct) + (s->B && !s->B->is_direct);
	if (!AE(27 + inc, ENCV(v != 0))) return 0;
	if (!AE(27 + 3, ENCV(v > 2))) return 1 + AE(27 + 5, ENCV(v == 2));
	/* 4-bit code `bits` (MSB first): 0..7 -> types 3..10; 13 -> intra; 14 -> 11; 15 -> 22; 8..12 -> 5th bit, types 12..21 */
	int bits_e = 0;
#ifdef E264_ENCODER
	if (v >= 3 && v <= 10) bits_e = v - 3;
	else if (v >= 23) bits_e = 13;
	else if (v == 11) bits_e = 14;
	else if (v == 22) bits_e = 15;
	else bits_e = (v + 4) >> 1;   /* 12..21 -> (bits<<1|b) - 4 = v  => bits = (v+4)>>1 in 8..12 */
#endif
	int bits = AE(27 + 4, ENCV((bits_e >> 3) & 1)) << 3;
	bits |= AE(27 + 5, ENCV((bits_e >> 2) & 1)) << 2;
	bits |= AE(27 + 5, ENCV((bits_e >> 1) & 1)) << 1;
	bits |= AE(27 + 5, ENCV(bits_e & 1));
	if (bits < 8) return bits + 3;
	if (bits == 13) return 23 + se_mb_type_intra(s, ENCV(v - 23), 32, 0);
	if (bits == 14) return 11;
	if (bits == 15) return 22;
	bits = (bits << 1) | AE(27 + 5, ENCV((v + 4) & 1));
	return bits - 4;
}
static int se_sub_mb_type_P(SliceCtx *s, int v) {   /* 0: 8x8, 1: 8x4, 2: 4x8, 3: 4x4 */
	if (!s->cabac) return VLC_UE(v);
	if (AE(21, ENCV(v == 0))) return 0;
	if (!AE(22, ENCV(v != 1))) return 1;
	if (AE(23, ENCV(v == 2))) return 2;
	return 3;
}
static int se_sub_mb_type_B(SliceCtx *s, int v) {   /* Table 7-18: 0 direct, 1 L0_8x8, 2 L1_8x8, 3 Bi_8x8, 4..12 */
	if (!s->cabac) return VLC_UE(v);
	if (!AE(36, ENCV(v != 0))) return 0;
	if (!AE(37, ENCV(v > 2))) return 1 + AE(39, ENCV(v == 2));
	int type = 3;
	if (AE(38, ENCV(v >= 7))) {
		if (AE(39, ENCV(v >= 11))) return 11 + AE(39, ENCV(v == 12));
		type += 4;
	}
	type += 2 * AE(39, ENCV(((v - type) >> 1) & 1));
	type += AE(39, ENCV((v - type) & 1));
	return type;
}
static int se_ref_idx(SliceCtx *s, int list, int i8, int v) {
	if (!s->cabac) {
		if (s->num_ref[list] == 2) return 1 ^ VLC_U(1, ENCV(v ^ 1));
		return VLC_UE(v);
	}
	/* ctxIdxInc from the 8x8 blocks left of / above partition i8 (9.3.3.1.1.6) */
	MbInfo *m; E264MbRec *r; int inc = 0;
	int x4 = (i8 & 1) * 2, y4 = (i8 >> 1) * 2;
	int z = sx_locate(s, x4 - 1, y4, &m, &r);
	if (m && !m->is_intra && !m->is_skip && !((m->direct8 >> (z >> 2)) & 1) && r->ref_idx[list][z >> 2] > 0) inc += 1;
	z = sx_locate(s, x4, y4 - 1, &m, &r);
	if (m && !m->is_intra && !m->is_skip && !((m->direct8 >> (z >> 2)) & 1) && r->ref_idx[list][z >> 2] > 0) inc += 2;
	int ref = 0, ctx = 54 + inc;
	while (AE(ctx, ENCV(ref < v))) {
		ref++;
		ctx = 54 + ((ctx - 54) >> 2) + 4;
		if (ref >= 32) { s->error = 1; break; }
	}
	return ref;
}
static int se_egk_bypass(SliceCtx *s, int k, int v) {
	int val = 0;
	while (AE_BYP(ENCV(v >= (1 << k)))) {
		val += 1 << k;
#ifdef E264_ENCODER
		v -= 1 << k;
#endif
		if (++k > 24) { s->error = 1; break; }
	}
	while (k--) val += AE_BYP(ENCV((v >> k) & 1)) << k;
	return val;
}
static int se_coded_block_pattern(SliceCtx *s, int v, int is_intra) {
	if (!s->cabac) {
#ifdef E264_ENCODER
		bw_ue(s->bw, is_intra ? h264_cbp_to_code_intra[v] : h264_cbp_to_code_inter[v]);
		return v;
#else
		unsigned c = br_ue(&s->br);
		if (c > 47) { s->error = 1; return 0; }
		return is_intra ? h264_code_to_cbp_intra[c] : h264_code_to_cbp_inter[c];
#endif
	}
	/* luma: 4 bins, ctxIdxInc from the cbp bits of the 8x8 blocks to the left / above (9.3.3.1.1.4) */
	int cbp = 0;
	int cbpA = s->A ? (s->A->is_pcm ? 0x2f : s->A->cbp) : 0x2f;   /* unavailable or I_PCM: condTerm 0 */
	int cbpB = s->B ? (s->B->is_pcm ? 0x2f : s->B->cbp) : 0x2f;
	for (int i = 0; i < 4; i++) {
		int a = (i & 1) ? (cbp >> (i - 1)) & 1 : (cbpA >> (i + 1)) & 1;
		int b = (i & 2) ? (cbp >> (i - 2)) & 1 : (cbpB >> (i + 2)) & 1;
		cbp |= AE(73 + !a + 2 * !b, ENCV((v >> i) & 1)) << i;
	}
	int ca = cbpA >> 4, cb = cbpB >> 4;
	if (!s->A) ca = 0;
	if (!s->B) cb = 0;
	if (AE(77 + (ca != 0) + 2 * (cb != 0), ENCV((v >> 4) != 0)))
		cbp |= (1 + AE(77 + 4 + (ca == 2) + 2 * (cb == 2), ENCV((v >> 4) == 2))) << 4;
	return cbp;
}
static int se_mb_qp_delta(SliceCtx *s, int v) {
	if (!s->cabac) return VLC_SE(v);
	int k = ENCV(v > 0 ? 2 * v - 1 : -2 * v);
	int val = 0, ctx = 60 + (s->last_qp_delta_nz != 0);
	while (AE(ctx, ENCV(val < k))) {
		ctx = 60 + 2 + ((ctx - 60) >> 1);
		if (++val > 104) { s->error = 1; break; }
	}
	return (val & 1) ? (val + 1) >> 1 : -(val >> 1);
}
static int se_intra_chroma_pred_mode(SliceCtx *s, int v) {
	if (!s->cabac) return VLC_UE(v);
	int inc = (s->A && s->A->is_intra && !s->A->is_pcm && s->A->chroma_pred_mode != 0)
	        + (s->B && s->B->is_intra && !s->B->is_pcm && s->B->chroma_pred_mode != 0);
	if (!AE(64 + inc, ENCV(v > 0))) return 0;
	if (!AE(64 + 3, ENCV(v > 1))) return 1;
	return 2 + AE(64 + 3, ENCV(v > 2));
}
/* returns -1 for "use predicted mode", else rem_intra_pred_mode 0..7 */
static int se_intra_pred_mode(SliceCtx *s, int v) {
	if (!s->cabac) {
		if (VLC_U(1, ENCV(v < 0))) return -1;
		return VLC_U(3, ENCV(v));
	}
	if (AE(68, ENCV(v < 0))) return -1;
	int m = AE(69, ENCV(v & 1));
	m |= AE(69, ENCV((v >> 1) & 1)) << 1;
	m |= AE(69, ENCV((v >> 2) & 1)) << 2;
	return m;
}
static int se_transform_8x8_flag(SliceCtx *s, int v) {
	if (!s->cabac) return VLC_U(1, v);
	return AE(399 + (s->A && s->A->t8x8) + (s->B && s->B->t8x8), v);
}

/* ------------------------------------------------------------------------------------------ */
/* residual blocks                                                                              */
/* ------------------------------------------------------------------------------------------ */
/* CABAC residual_block_cabac (7.3.5.3.3): `blk` is the raster block in the pool (pre-zeroed by the
 * parser / pre-filled by the writer); scan[k] maps coefficient k (0..n-1) to its raster slot.
 * has_cbf: whether coded_block_flag is transmitted.  Returns the number of non-zero levels.
 * The body is force-inlined with a constant ctxBlockCat so that each category gets its own tight
 * significance loop (the per-coefficient context selection folds away). */
static inline __attribute__((always_inline)) int residual_block_cabac_cat(SliceCtx *s, const int cat, int cbf_inc, int has_cbf, int16_t *blk, const uint8_t *scan, const int n) {
	int last_e = -1;
#ifdef E264_ENCODER
	for (int k = 0; k < n; k++) if (blk[scan[k]]) last_e = k;
#endif
	CR_BEGIN
	if (has_cbf && !AE_R(h264_cat_cbf[cat] + cbf_inc, ENCV(last_e >= 0))) { CR_OUT return 0; }
	uint64_t sigmask = 0;
	const int sig_base = h264_cat_sig[cat], last_base = h264_cat_last[cat];
	int k;
	for (k = 0; k < n - 1; k++) {
		const int si = cat == 5 ? h264_sig8x8_inc[k] : cat == 3 ? (k < 2 ? k : 2) : k;
		if (AE_R(sig_base + si, ENCV(blk[scan[k]] != 0))) {
			sigmask |= (uint64_t)1 << k;
			const int li = cat == 5 ? h264_last8x8_inc[k] : cat == 3 ? (k < 2 ? k : 2) : k;
			if (AE_R(last_base + li, ENCV(k == last_e))) break;
		}
	}
	if (k == n - 1) sigmask |= (uint64_t)1 << (n - 1);
	const int nsig = __builtin_popcountll(sigmask);
	const int abs_base = h264_cat_abs[cat], cap = 4 - (cat == 3);
	int gt1 = 0, eq1 = 0;
	while (sigmask) {
		const int pos = 63 - __builtin_clzll(sigmask);
		sigmask &= ~((uint64_t)1 << pos);
		int16_t *dst = blk + scan[pos];
		int a = ENCV((*dst < 0 ? -*dst : *dst) - 1);
		int absm1;
		if (!AE_R(abs_base + (gt1 ? 0 : (1 + eq1 > 4 ? 4 : 1 + eq1)), ENCV(a > 0))) { absm1 = 0; eq1++; }
		else {
			int ctx = abs_base + 5 + (gt1 < cap ? gt1 : cap), cnt = 1;
			while (cnt < 14 && AE_R(ctx, ENCV(a > cnt))) cnt++;
			absm1 = cnt;
			if (cnt == 14) { CR_OUT absm1 = 14 + se_egk_bypass(s, 0, ENCV(a - 14)); CR_IN }
			gt1++;
		}
		int neg = AE_BYP_R(ENCV(*dst < 0));
		int lv = neg ? -(absm1 + 1) : absm1 + 1;
#ifndef E264_ENCODER
		*dst = (int16_t)lv;
#else
		(void)lv;
#endif
	}
	CR_OUT
	return nsig;
}
static __attribute__((noinline)) int residual_block_cabac(SliceCtx *s, int cat, int cbf_inc, int has_cbf, int16_t *blk, const uint8_t *scan, int n) {
	switch (cat) {
	case 0: return residual_block_cabac_cat(s, 0, cbf_inc, 1, blk, scan, 16);
	case 1: return residual_block_cabac_cat(s, 1, cbf_inc, 1, blk, scan, 15);
	case 2: return residual_block_cabac_cat(s, 2, cbf_inc, 1, blk, scan, 16);
	case 3: return residual_block_cabac_cat(s, 3, cbf_inc, 1, blk, scan, 4);
	case 4: return residual_block_cabac_cat(s, 4, cbf_inc, 1, blk, scan, 15);
	default: return residual_block_cabac_cat(s, 5, cbf_inc, 0, blk, scan, 64);
	}
	(void)has_cbf; (void)n;
}

/* --- CAVLC residual_block_cavlc (7.3.5.3.2, 9.2) --- */
#ifndef E264_ENCODER
typedef struct VlcLut { uint16_t l1[256]; uint16_t l2[24][256]; int n2; } VlcLut;
/* entry: (value << 5) | len for len 1..16;  in l1 an entry with bit 15 set = index of the l2 table */
static VlcLut vl_coeff_token[5], vl_total_zeros[15], vl_total_zeros_dc[3], vl_run_before[7];
static int vlc_ready;
static void vlc_add(VlcLut *t, int len, unsigned code, int value) {
	if (len == 0) return;
	if (len <= 8) {
		unsigned lo = code << (8 - len);
		for (unsigned i = 0; i < (1u << (8 - len)); i++) t->l1[lo + i] = (uint16_t)((value << 5) | len);
	} else {
		unsigned top = code >> (len - 8);
		if (!(t->l1[top] & 0x8000)) t->l1[top] = (uint16_t)(0x8000 | t->n2++);
		uint16_t *sub = t->l2[t->l1[top] & 0xff];
		unsigned rest = len - 8, lo = (code & ((1u << rest) - 1)) << (8 - rest);
		for (unsigned i = 0; i < (1u << (8 - rest)); i++) sub[lo + i] = (uint16_t)((value << 5) | len);
	}
}
static void vlc_build_all(void) {
	if (vlc_ready) return;
	for (int c = 0; c < 5; c++) for (int i = 0; i < 68; i++) vlc_add(&vl_coeff_token[c], h264_coeff_token[c][i].len, h264_coeff_token[c][i].code, i);
	for (int t = 0; t < 15; t++) for (int i = 0; i < 16 - t; i++) vlc_add(&vl_total_zeros[t], h264_total_zeros4x4[t][i].len, h264_total_zeros4x4[t][i].code, i);
	for (int t = 0; t < 3; t++) for (int i = 0; i < 4 - t; i++) vlc_add(&vl_total_zeros_dc[t], h264_total_zeros2x2[t][i].len, h264_total_zeros2x2[t][i].code, i);
	for (int t = 0; t < 7; t++) for (int i = 0; i < (t < 6 ? t + 2 : 15); i++) vlc_add(&vl_run_before[t], h264_run_before[t][i].len, h264_run_before[t][i].code, i);
	vlc_ready = 1;
}
static inline int vlc_get(SliceCtx *s, const VlcLut *t) {
	uint32_t p = br_peek32(&s->br);
	uint16_t e = t->l1[p >> 24];
	if (e & 0x8000) e = t->l2[e & 0xff][(p >> 16) & 0xff];
	if ((e & 31) == 0) { s->error = 1; s->br.pos += 1; return 0; }
	s->br.pos += e & 31;
	return e >> 5;
}
#endif

/* nC: -1 for chroma DC, otherwise the predicted number of coefficients.  Returns TotalCoeff. */
static int residual_block_cavlc(SliceCtx *s, int nC, int16_t *blk, const uint8_t *scan, int n) {
	int cls = nC < 0 ? 4 : nC < 2 ? 0 : nC < 4 ? 1 : nC < 8 ? 2 : 3;
	int level[16], run[16];
#ifdef E264_ENCODER
	int idx[16], total = 0;
	for (int k = 0; k < n; k++) if (blk[scan[k]]) { idx[total] = k; total++; }
	/* reversed order: level[0] is the highest-frequency coefficient */
	for (int i = 0; i < total; i++) level[i] = blk[scan[idx[total - 1 - i]]];
	int t1 = 0;
	while (t1 < 3 && t1 < total && (level[t1] == 1 || level[t1] == -1)) t1++;
	const H264Vlc *ct = &h264_coeff_token[cls][total * 4 + t1];
	bw_u(s->bw, ct->len, ct->code);
	if (total == 0) return 0;
	int suffix_len = (total > 10 && t1 < 3) ? 1 : 0;
	for (int i = 0; i < total; i++) {
		if (i < t1) { bw_u(s->bw, 1, level[i] < 0); continue; }
		int a = level[i] < 0 ? -level[i] : level[i];
		int code = 2 * a - 2 + (level[i] < 0);
		if (i == t1 && t1 < 3) code -= 2;
		int prefix, sfx_size = suffix_len, sfx;
		if (suffix_len == 0 && code >= 14 && code < 30) { prefix = 14; sfx = code - 14; sfx_size = 4; }
		else if (code >= (15 << (suffix_len ? suffix_len : 1)) ) {
			/* escape: level_prefix >= 15 */
			int c2 = code - (15 << suffix_len) - (suffix_len == 0 ? 15 : 0);
			prefix = 15;
			while (c2 >= (1 << (prefix - 3)) ) { c2 -= 1 << (prefix - 3); prefix++; }
			/* levelCode = (Min(15,prefix) << suffixLength) + suffix (+15 if prefix>=15 && suffixLength==0) (+ (1<<(prefix-3)) - 4096 if prefix>=16) */
			sfx = c2; sfx_size = prefix - 3;
		} else { prefix = code >> suffix_len; sfx = code & ((1 << suffix_len) - 1); }
		bw_u(s->bw, prefix, 0); bw_u(s->bw, 1, 1);
		if (sfx_size) bw_u(s->bw, sfx_size, sfx);
		if (suffix_len == 0) suffix_len = 1;
		if (a > (3 << (suffix_len - 1)) && suffix_len < 6) suffix_len++;
	}
	int zeros_left = 0;
	if (total < n) {
		zeros_left = idx[total - 1] + 1 - total;
		const H264Vlc *tz = nC < 0 ? &h264_total_zeros2x2[total - 1][zeros_left] : &h264_total_zeros4x4[total - 1][zeros_left];
		bw_u(s->bw, tz->len, tz->code);
	}
	for (int i = total - 1; i > 0 && zeros_left > 0; i--) {
		int rb = idx[i] - idx[i - 1] - 1;
		const H264Vlc *r = &h264_run_before[(zeros_left > 7 ? 7 : zeros_left) - 1][rb];
		bw_u(s->bw, r->len, r->code);
		zeros_left -= rb;
	}
	(void)run;
	return total;
#else
	int tok = vlc_get(s, &vl_coeff_token[cls]);
	int total = tok >> 2, t1 = tok & 3;
	if (total == 0) return 0;
	if (total > n) { s->error = 1; return 0; }
	int suffix_len = (total > 10 && t1 < 3) ? 1 : 0;
	for (int i = 0; i < total; i++) {
		if (i < t1) { level[i] = br_u1(&s->br) ? -1 : 1; continue; }
		uint32_t p = br_peek32(&s->br);
		int prefix = p ? __builtin_clz(p) : 32;
		if (prefix > 25) { s->error = 1; return 0; }
		s->br.pos += prefix + 1;
		int code = (prefix < 15 ? prefix : 15) << suffix_len;
		int sfx_size = suffix_len;
		if (prefix == 14 && suffix_len == 0) sfx_size = 4;
		if (prefix >= 15) sfx_size = prefix - 3;
		if (sfx_size) code += br_u(&s->br, sfx_size);
		if (prefix >= 15 && suffix_len == 0) code += 15;
		if (prefix >= 16) code += (1 << (prefix - 3)) - 4096;
		if (i == t1 && t1 < 3) code += 2;
		level[i] = (code & 1) ? (-code - 1) >> 1 : (code + 2) >> 1;
		if (suffix_len == 0) suffix_len = 1;
		int a = level[i] < 0 ? -level[i] : level[i];
		if (a > (3 << (suffix_len - 1)) && suffix_len < 6) suffix_len++;
	}
	int zeros_left = 0;
	if (total < n) zeros_left = vlc_get(s, nC < 0 ? &vl_total_zeros_dc[total - 1] : &vl_total_zeros[total - 1]);
	for (int i = 0; i < total - 1; i++) {
		run[i] = zeros_left > 0 ? vlc_get(s, &vl_run_before[(zeros_left > 7 ? 7 : zeros_left) - 1]) : 0;
		zeros_left -= run[i];
		if (zeros_left < 0) { s->error = 1; return 0; }
	}
	run[total - 1] = zeros_left;
	int pos = -1;
	for (int i = total - 1; i >= 0; i--) {
		pos += run[i] + 1;
		if (pos >= n) { s->error = 1; return 0; }
		blk[scan[pos]] = (int16_t)level[i];
	}
	return total;
#endif
}

/* ------------------------------------------------------------------------------------------ */
/* coefficient pool                                                                             */
/* ------------------------------------------------------------------------------------------ */
/* The parser takes zeroed pool space and rewinds when the block turns out empty.  The writer gets
 * its levels from a fixed-layout staging area filled by the chooser (gen_coefs: luma DC at 0, luma
 * 4x4 block b at 16+16b or 8x8 block i at 16+64i, chroma DC at 272, chroma AC block j at 280+16j)
 * and copies them into the pool the same way, so both directions produce identical records. */
static inline int16_t *sx_pool_take(SliceCtx *s, int n, int staging_off) {
	if (s->n_coefs + (uint32_t)n > s->coef_cap) { s->error = 2; s->n_coefs = s->coef_cap - 408u; }   /* unreachable after the per-macroblock check of the slice loop; stays inside the buffer regardless */
	int16_t *p = s->coefs + s->n_coefs;
	s->n_coefs += n;
#ifndef E264_ENCODER
	(void)staging_off;
	memset(p, 0, (size_t)n * sizeof(int16_t));
#else
	memcpy(p, s->gen_coefs + staging_off, (size_t)n * sizeof(int16_t));
#endif
	return p;
}

static const uint8_t sx_scan_dc2x2[4] = {0, 1, 2, 3};
static uint8_t sx_scan_ac[15];          /* zigzag positions 1..15 */
static uint8_t sx_scan8x8_cavlc[4][16]; /* zigzag8x8[4k+i] */
static void sx_init_c_later(void);
static void sx_init_tables(void) {
	cabac_build_tables();
	sx_init_c_later();
	for (int k = 0; k < 15; k++) sx_scan_ac[k] = h264_zigzag4x4[k + 1];
	for (int i = 0; i < 4; i++) for (int k = 0; k < 16; k++) sx_scan8x8_cavlc[i][k] = h264_zigzag8x8[4 * k + i];
#ifndef E264_ENCODER
	vlc_build_all();
#endif
}

/* CAVLC nC of a luma block (z) / chroma block (plane 0/1, idx 0..3) from the left/top blocks (9.2.1) */
static int sx_nC_luma(SliceCtx *s, int b) {
	MbInfo *ma, *mb; E264MbRec *r;
	int x = e264_blk_x(b), y = e264_blk_y(b);
	int za = sx_locate(s, x - 1, y, &ma, &r), zb = sx_locate(s, x, y - 1, &mb, &r);
	int na = ma ? ma->tc[za] : 0, nb = mb ? mb->tc[zb] : 0;
	return (ma && mb) ? (na + nb + 1) >> 1 : na + nb;
}
static int sx_nC_chroma(SliceCtx *s, int pl, int i) {
	int x = i & 1, y = i >> 1;
	MbInfo *ma = x ? s->cur : s->A, *mb = y ? s->cur : s->B;
	int na = ma ? ma->tc[16 + pl * 4 + (y * 2 + (x ^ 1))] : 0;
	int nb = mb ? mb->tc[16 + pl * 4 + ((y ^ 1) * 2 + x)] : 0;
	return (ma && mb) ? (na + nb + 1) >> 1 : na + nb;
}
/* CABAC coded_block_flag ctxIdxInc helpers (9.3.3.1.1.9): value for an unavailable neighbour */
static inline int sx_cbf_na(SliceCtx *s) { return s->cur->is_intra; }
/* z-index of the block left of / above block b inside the same macroblock (valid when x>0 / y>0) */
static const uint8_t sx_left_z[16]  = {0, 0, 0, 2, 1, 4, 3, 6, 0, 8, 0, 10, 9, 12, 11, 14};
static const uint8_t sx_above_z[16] = {0, 0, 0, 1, 0, 0, 4, 5, 2, 3, 8, 9, 6, 7, 12, 13};
/* The same, macroblock at a time: bits 0-15 = coded_block_flags of this macroblock so far (z-order), bits 16-19 =
 * the left neighbour's right column by row, bits 20-23 = the top neighbour's bottom row by column (each already
 * resolved for unavailable / I_PCM neighbours); sx_cbf_la/tb give the bit to test for block b. */
static const uint8_t sx_cbf_la[16] = {16, 0, 17, 2, 1, 4, 3, 6, 18, 8, 19, 10, 9, 12, 11, 14};
static const uint8_t sx_cbf_tb[16] = {20, 21, 0, 1, 22, 23, 4, 5, 2, 3, 8, 9, 6, 7, 12, 13};
static inline uint32_t sx_cbf_luma_border(SliceCtx *s) {
	const uint32_t na = (uint32_t)sx_cbf_na(s);
	uint32_t left = na * 15u, top = na * 15u;
	if (s->A) { const uint32_t c = s->A->cbf_luma; left = s->A->is_pcm ? 15u : ((c >> 5) & 1) | ((c >> 7) & 1) << 1 | ((c >> 13) & 1) << 2 | ((c >> 15) & 1) << 3; }
	if (s->B) { const uint32_t c = s->B->cbf_luma; top = s->B->is_pcm ? 15u : ((c >> 10) & 1) | ((c >> 11) & 1) << 1 | ((c >> 14) & 1) << 2 | ((c >> 15) & 1) << 3; }
	return left << 16 | top << 20;
}
static int sx_cbf_inc_luma(SliceCtx *s, int b) {
	const int x = e264_blk_x(b), y = e264_blk_y(b);
	int a, bb;
	if (x) a = (s->cur->cbf_luma >> sx_left_z[b]) & 1;
	else a = s->A ? (s->A->is_pcm ? 1 : (s->A->cbf_luma >> e264_blk_z(3, y)) & 1) : sx_cbf_na(s);
	if (y) bb = (s->cur->cbf_luma >> sx_above_z[b]) & 1;
	else bb = s->B ? (s->B->is_pcm ? 1 : (s->B->cbf_luma >> e264_blk_z(x, 3)) & 1) : sx_cbf_na(s);
	return a + 2 * bb;
}
static int sx_cbf_inc_chroma_ac(SliceCtx *s, int pl, int i) {
	int x = i & 1, y = i >> 1;
	MbInfo *ma = x ? s->cur : s->A, *mb = y ? s->cur : s->B;
	int a = ma ? (ma->is_pcm ? 1 : ((pl ? ma->cbf_cr : ma->cbf_cb) >> (y * 2 + (x ^ 1))) & 1) : sx_cbf_na(s);
	int b = mb ? (mb->is_pcm ? 1 : ((pl ? mb->cbf_cr : mb->cbf_cb) >> ((y ^ 1) * 2 + x)) & 1) : sx_cbf_na(s);
	return a + 2 * b;
}
static int sx_cbf_inc_dc(SliceCtx *s, int bit) {
	int a = s->A ? (s->A->is_pcm ? 1 : (s->A->cbf_dc >> bit) & 1) : sx_cbf_na(s);
	int b = s->B ? (s->B->is_pcm ? 1 : (s->B->cbf_dc >> bit) & 1) : sx_cbf_na(s);
	return a + 2 * b;
}

/* residual( ) for one macroblock (7.3.5.3): luma according to the macroblock kind, then chroma */
static void sx_residual(SliceCtx *s, int is_i16, int cbp) {
	MbInfo *m = s->cur; E264MbRec *r = s->rec;
	uint32_t coded = 0;
	if (is_i16) {
		int16_t *blk = sx_pool_take(s, 16, 0);
		int n = s->cabac ? residual_block_cabac(s, 0, sx_cbf_inc_dc(s, 0), 1, blk, h264_zigzag4x4, 16)
		                 : residual_block_cavlc(s, sx_nC_luma(s, 0), blk, h264_zigzag4x4, 16);
		if (n) { coded |= CODED_Y_DC; m->cbf_dc |= 1; } else s->n_coefs -= 16;
	}
	uint32_t cbf_ext = (s->cabac && !m->t8x8 && (cbp & 15)) ? sx_cbf_luma_border(s) : 0;
	for (int i8 = 0; i8 < 4; i8++) {
		if (!((cbp >> i8) & 1)) continue;
		if (m->t8x8) {
			int16_t *blk = sx_pool_take(s, 64, 16 + 64 * i8);
			int n = 0;
			if (s->cabac) {
				n = residual_block_cabac(s, 5, 0, 0, blk, h264_zigzag8x8, 64);
				if (n) m->cbf_luma |= 15 << (i8 * 4);
			} else {
				for (int i = 0; i < 4; i++) {
					int t = residual_block_cavlc(s, sx_nC_luma(s, i8 * 4 + i), blk, sx_scan8x8_cavlc[i], 16);
					m->tc[i8 * 4 + i] = (uint8_t)t; n += t;
				}
			}
			if (n) coded |= 15u << (i8 * 4); else s->n_coefs -= 64;
		} else {
			for (int i = 0; i < 4; i++) {
				int b = i8 * 4 + i;
				int16_t *blk = sx_pool_take(s, 16, 16 + 16 * b);
				int n;
				if (s->cabac) {
					const int inc = (int)(((cbf_ext >> sx_cbf_la[b]) & 1) + 2 * ((cbf_ext >> sx_cbf_tb[b]) & 1));
					n = is_i16 ? residual_block_cabac(s, 1, inc, 1, blk, sx_scan_ac, 15)
					           : residual_block_cabac(s, 2, inc, 1, blk, h264_zigzag4x4, 16);
					if (n) { m->cbf_luma |= 1 << b; cbf_ext |= 1u << b; }
				} else {
					n = is_i16 ? residual_block_cavlc(s, sx_nC_luma(s, b), blk, sx_scan_ac, 15)
					           : residual_block_cavlc(s, sx_nC_luma(s, b), blk, h264_zigzag4x4, 16);
					m->tc[b] = (uint8_t)n;
				}
				if (n) coded |= 1u << b; else s->n_coefs -= 16;
			}
		}
	}
	if (cbp >> 4) {
		const uint32_t chroma_off = s->n_coefs;
		int16_t *dc = sx_pool_take(s, 8, 272);
		int any = 0;
		for (int pl = 0; pl < 2; pl++) {
			int n = s->cabac ? residual_block_cabac(s, 3, sx_cbf_inc_dc(s, 1 + pl), 1, dc + 4 * pl, sx_scan_dc2x2, 4)
			                 : residual_block_cavlc(s, -1, dc + 4 * pl, sx_scan_dc2x2, 4);
			if (n) { coded |= pl ? CODED_CR_DC : CODED_CB_DC; m->cbf_dc |= 2 << pl; any = 1; }
		}
		if (!any) s->n_coefs -= 8;
		if ((cbp >> 4) == 2) {
			for (int pl = 0; pl < 2; pl++) for (int i = 0; i < 4; i++) {
				int16_t *blk = sx_pool_take(s, 16, 280 + 16 * (pl * 4 + i));
				int n;
				if (s->cabac) {
					n = residual_block_cabac(s, 4, sx_cbf_inc_chroma_ac(s, pl, i), 1, blk, sx_scan_ac, 15);
					if (n) { if (pl) m->cbf_cr |= 1 << i; else m->cbf_cb |= 1 << i; }
				} else {
					n = residual_block_cavlc(s, sx_nC_chroma(s, pl, i), blk, sx_scan_ac, 15);
					m->tc[16 + pl * 4 + i] = (uint8_t)n;
				}
				if (n) coded |= 1u << (16 + pl * 4 + i); else s->n_coefs -= 16;
			}
		}
		/* luma only: every chroma element is parsed above (the entropy state and the neighbours' cbf / tc need it), then
		 * its levels leave the pool again (they are the run's tail) and the record keeps no chroma bit */
		if (s->luma_only) { s->n_coefs = chroma_off; coded &= 0xffffu | CODED_Y_DC; }
	}
	r->coded = coded;
}
#endif
