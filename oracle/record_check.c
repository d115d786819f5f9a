/* oracle/record_check.c — TEST INFRASTRUCTURE ONLY.  The record contract of edge264_b200/csrc/records.h as a check:
 * the CPU restatement backend runs it on every submitted picture when E264_CHECK_RECORDS=1 (oracle/port_backend.c),
 * and the record fuzzer (tests/native/record_fuzz.c) runs it on every picture it generates before the device sees it. */
#include <stdarg.h>
#include <stdio.h>
#include "record_check.h"
#include "../edge264_b200/csrc/h264_tables.h"

#define MAX_SLICES 64   /* E264_MAX_SLICES (dec.h): the size of the backends' slice tables */

int e264_rec_coef_count(const E264MbRec *r) {
	if (r->kind == MBK_IPCM) return 192;
	unsigned c = r->coded;
	int n = (c & CODED_Y_DC) ? 16 : 0;
	n += (r->flags & MBF_T8x8) ? 64 * __builtin_popcount(c & 0x1111) : 16 * __builtin_popcount(c & 0xffff);
	if (c & (CODED_CB_DC | CODED_CR_DC)) n += 8;
	return n + 16 * __builtin_popcount((c >> 16) & 0xff);
}

static int fail(char *why, int why_len, int mb, const E264PicDesc *pd, const char *fmt, ...) {
	char msg[200];
	va_list ap; va_start(ap, fmt); vsnprintf(msg, sizeof(msg), fmt, ap); va_end(ap);
	if (mb < 0) snprintf(why, why_len, "picture: %s", msg);
	else snprintf(why, why_len, "mb %d (%d,%d): %s", mb, mb % pd->width_mbs, mb / pd->width_mbs, msg);
	return 1;
}
#define FAIL(...) return fail(why, why_len, __VA_ARGS__)

static int is_qpc(int v) { for (int q = 0; q < 52; q++) if (h264_qpc[q] == v) return 1; return 0; }

/* unavailability bits (A=1, B=2, C=4, D=8) that 6.4.11.4 forces for the 4x4 block z / the 8x8 block i / the macroblock
 * (i = -1) when the neighbouring macroblocks are present (have: A=1, B=2, C=4, D=8) */
static int forced4x4(int z, int have) {
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
static int forced8x8(int i, int have) {
	int u = 0;
	if (!(i & 1) && !(have & 1)) u |= 1;
	if (!(i & 2) && !(have & 2)) u |= 2;
	if (i == 0 ? !(have & 2) : i == 1 ? !(have & 4) : i == 3) u |= 4;
	if (i == 0 ? !(have & 8) : i == 1 ? !(have & 2) : i == 2 ? !(have & 1) : 0) u |= 8;
	return u;
}
static int forced16(int have) { return (have & 1 ? 0 : 1) | (have & 2 ? 0 : 2) | (have & 8 ? 0 : 8); }

static int check_slice(const E264SliceRec *s, char *msg, int len) {
	if (s->filter_offset_a < -12 || s->filter_offset_a > 12 || (s->filter_offset_a & 1) || s->filter_offset_b < -12 || s->filter_offset_b > 12 || (s->filter_offset_b & 1))
		return snprintf(msg, len, "filter offsets %d %d", s->filter_offset_a, s->filter_offset_b);
	if (s->deblock_idc > 2 || s->slice_type > 2 || s->wp_mode > 2) return snprintf(msg, len, "deblock_idc %d slice_type %d wp_mode %d", s->deblock_idc, s->slice_type, s->wp_mode);
	if (s->luma_log2_wd > 7 || s->chroma_log2_wd > 7) return snprintf(msg, len, "log2_wd %d %d", s->luma_log2_wd, s->chroma_log2_wd);
	for (int l = 0; l < 2; l++) for (int i = 0; i < 16; i++) for (int k = 0; k < 3; k++) {
		if (s->wp_w[l][i][k] < -128 || s->wp_w[l][i][k] > 128) return snprintf(msg, len, "weight [%d][%d][%d] = %d", l, i, k, s->wp_w[l][i][k]);
		if (s->wp_o[l][i][k] < -128 || s->wp_o[l][i][k] > 127) return snprintf(msg, len, "offset [%d][%d][%d] = %d", l, i, k, s->wp_o[l][i][k]);
	}
	for (int i = 0; i < 256; i++) if (s->implicit_w1[i >> 4][i & 15] < -64 || s->implicit_w1[i >> 4][i & 15] > 128) return snprintf(msg, len, "implicit_w1[%d][%d] = %d", i >> 4, i & 15, s->implicit_w1[i >> 4][i & 15]);
	for (int i = 0; i < 96; i++) if (!s->scaling4x4[i >> 4][i & 15]) return snprintf(msg, len, "scaling4x4[%d][%d] = 0", i >> 4, i & 15);
	for (int i = 0; i < 128; i++) if (!s->scaling8x8[i >> 6][i & 63]) return snprintf(msg, len, "scaling8x8[%d][%d] = 0", i >> 6, i & 63);
	return 0;
}

int e264_check_records(const E264PicDesc *pd, const E264MbRec *recs, const int16_t *coefs, const E264SliceRec *slices,
                       const uint32_t *intra_list, int n_slots, char *why, int why_len) {
	(void)coefs;   /* levels may take any int16 value */
	const int W = pd->width_mbs, H = pd->height_mbs, nmb = W * H;
	if (W < 1 || H < 1) FAIL(-1, pd, "geometry %dx%d", W, H);
	if (pd->dst_slot < 0 || pd->dst_slot >= n_slots) FAIL(-1, pd, "dst_slot %d of %d slots", pd->dst_slot, n_slots);
	if (pd->n_slices < 1 || pd->n_slices > MAX_SLICES) FAIL(-1, pd, "n_slices %d", pd->n_slices);
	if (pd->n_coefs < 0 || (pd->n_coefs & 7)) FAIL(-1, pd, "n_coefs %d", pd->n_coefs);
	for (int i = 0; i < pd->n_slices; i++) {
		char msg[160];
		if (check_slice(slices + i, msg, sizeof(msg))) FAIL(-1, pd, "slice %d: %s", i, msg);
	}
	int n_intra = 0;
	for (int a = 0; a < nmb; a++) {
		const E264MbRec *r = recs + a;
		const int mbx = a % W, mby = a / W;
		if (r->kind > MBK_INTER) FAIL(a, pd, "kind %d", r->kind);
		if (r->flags & ~(MBF_T8x8 | MBF_EDGE_L | MBF_EDGE_T | MBF_DEBLOCK | MBF_SKIP)) FAIL(a, pd, "flags %#x", r->flags);
		if (r->slice_idx >= pd->n_slices) FAIL(a, pd, "slice_idx %d of %d", r->slice_idx, pd->n_slices);
		const E264SliceRec *sr = slices + r->slice_idx;
		if (r->coded >> 27) FAIL(a, pd, "coded %#x", r->coded);
		int t8 = r->flags & MBF_T8x8;
		if (r->kind == MBK_I8x8 ? !t8 : (r->kind != MBK_INTER && t8)) FAIL(a, pd, "MBF_T8x8 %d on kind %d", !!t8, r->kind);
		if (t8) for (int i8 = 0; i8 < 4; i8++) { unsigned g = (r->coded >> (4 * i8)) & 15; if (g && g != 15) FAIL(a, pd, "8x8 block %d has luma bits %#x", i8, g); }
		if ((r->coded & CODED_Y_DC) && r->kind != MBK_I16x16) FAIL(a, pd, "CODED_Y_DC on kind %d", r->kind);
		if (r->kind == MBK_IPCM && r->coded) FAIL(a, pd, "I_PCM with coded %#x", r->coded);
		if (r->qp[0] > 51 || (r->kind == MBK_IPCM && r->qp[0])) FAIL(a, pd, "qp[0] %d on kind %d", r->qp[0], r->kind);
		if (!is_qpc(r->qp[1]) || !is_qpc(r->qp[2])) FAIL(a, pd, "chroma qp %d %d", r->qp[1], r->qp[2]);
		if (r->coef_off & 7) FAIL(a, pd, "coef_off %u", r->coef_off);
		if ((int64_t)r->coef_off + e264_rec_coef_count(r) > pd->n_coefs) FAIL(a, pd, "level run %u+%d past n_coefs %d", r->coef_off, e264_rec_coef_count(r), pd->n_coefs);

		/* neighbours present for prediction: inside the picture and in the same slice */
		int have = 0;
		if (mbx > 0 && recs[a - 1].slice_idx == r->slice_idx) have |= 1;
		if (mby > 0 && recs[a - W].slice_idx == r->slice_idx) have |= 2;
		if (mby > 0 && mbx < W - 1 && recs[a - W + 1].slice_idx == r->slice_idx) have |= 4;
		if (mby > 0 && mbx > 0 && recs[a - W - 1].slice_idx == r->slice_idx) have |= 8;
		if (r->kind == MBK_I4x4 || r->kind == MBK_I8x8 || r->kind == MBK_I16x16) {
			int nb = r->kind == MBK_I4x4 ? 16 : r->kind == MBK_I8x8 ? 4 : 1;
			for (int b = 0; b < nb; b++) {
				int m = r->kind == MBK_I16x16 ? r->i16_mode : r->modes[b];
				int forced = r->kind == MBK_I4x4 ? forced4x4(b, have) : r->kind == MBK_I8x8 ? forced8x8(b, have) : forced16(have);
				if (r->kind == MBK_I16x16 && (m >> 4) & 4) FAIL(a, pd, "Intra16x16 mode byte %#x has a C bit", m);
				if (forced & ~(m >> 4)) FAIL(a, pd, "block %d: mode byte %#x marks unavailable neighbours %#x available", b, m, forced & ~(m >> 4));
				if (!e264_intra_mode_legal(r->kind, m & 15, m >> 4)) FAIL(a, pd, "block %d: intra mode %d illegal with unavailability %#x", b, m & 15, m >> 4);
			}
			int cm = r->chroma_mode;
			if ((cm >> 4) & 4) FAIL(a, pd, "chroma mode byte %#x has a C bit", cm);
			if (forced16(have) & ~(cm >> 4)) FAIL(a, pd, "chroma mode byte %#x marks unavailable neighbours %#x available", cm, forced16(have) & ~(cm >> 4));
			if (!e264_intra_mode_legal(-1, cm & 15, cm >> 4)) FAIL(a, pd, "chroma mode %d illegal with unavailability %#x", cm & 15, cm >> 4);
		}

		/* deblocking */
		if (r->flags & MBF_DEBLOCK) {
			if (sr->deblock_idc == 1) FAIL(a, pd, "MBF_DEBLOCK in a slice with deblock_idc 1");
			int l_ok = mbx > 0 && (sr->deblock_idc == 0 || recs[a - 1].slice_idx == r->slice_idx);
			int t_ok = mby > 0 && (sr->deblock_idc == 0 || recs[a - W].slice_idx == r->slice_idx);
			if ((r->flags & MBF_EDGE_L) && !l_ok) FAIL(a, pd, "MBF_EDGE_L without a left neighbour to filter against (deblock_idc %d)", sr->deblock_idc);
			if ((r->flags & MBF_EDGE_T) && !t_ok) FAIL(a, pd, "MBF_EDGE_T without a top neighbour to filter against (deblock_idc %d)", sr->deblock_idc);
			if (sr->deblock_idc == 0 && (!(r->flags & MBF_EDGE_L) != !(mbx > 0) || !(r->flags & MBF_EDGE_T) != !(mby > 0)))
				FAIL(a, pd, "edge flags %#x with deblock_idc 0", r->flags);
			if (!pd->any_deblock) FAIL(a, pd, "MBF_DEBLOCK but any_deblock is 0");
		} else if (r->flags & (MBF_EDGE_L | MBF_EDGE_T)) FAIL(a, pd, "edge flags %#x without MBF_DEBLOCK", r->flags);

		/* references */
		for (int l = 0; l < 2; l++) for (int i8 = 0; i8 < 4; i8++) {
			int ri = r->ref_idx[l][i8], rp = r->ref_pic[l][i8];
			if (r->kind != MBK_INTER || ri < 0) {
				if (ri != -1 || rp != -1) FAIL(a, pd, "unused list %d of 8x8 block %d: ref_idx %d ref_pic %d", l, i8, ri, rp);
			} else if (ri > 15 || rp < 0 || rp >= n_slots || rp == pd->dst_slot)
				FAIL(a, pd, "list %d of 8x8 block %d: ref_idx %d ref_pic %d (dst_slot %d, %d slots)", l, i8, ri, rp, pd->dst_slot, n_slots);
		}
		if (r->kind == MBK_INTER) {
			for (int i8 = 0; i8 < 4; i8++) if (r->ref_idx[0][i8] < 0 && r->ref_idx[1][i8] < 0) FAIL(a, pd, "8x8 block %d uses no list", i8);
		} else if (n_intra >= pd->n_intra || intra_list[n_intra++] != (uint32_t)a) FAIL(a, pd, "intra_list entry %d is not this macroblock", n_intra);
	}
	if (n_intra != pd->n_intra) FAIL(-1, pd, "n_intra %d but %d intra macroblocks", pd->n_intra, n_intra);
	return 0;
}
