/* port_error_map.c — TEST INFRASTRUCTURE ONLY.  The error-map rules of E264PicDesc.err_pic / taint and E264MbRec.err in
 * plain C, restated from the feature's specification (not from the kernels): what the device's map of every frame slot
 * must hold after every picture.  Built by tests/checkers.py into the CPU backend with every optional output
 * (port_outputs_backend.c) and by tests/test_mb_errors.py into the record fuzzer's error-map driver (record_fuzz_maps.c). */
#include <stddef.h>
#include <stdint.h>
#include "../../edge264_b200/csrc/records.h"

/* ---------------------------------------------------------------------------------------- */
/* error map                                                                                  */
/* ---------------------------------------------------------------------------------------- */
/* maps = [n_slots][nmb], one byte per macroblock and frame slot.  A picture with pd->err_pic gives each macroblock
 * max(err, what its prediction reads); a picture without it leaves every map alone, and a slot outside pd->taint counts
 * as zeros.  Deblocking is not followed (it moves at most three samples across an edge).
 *   inter: every used list and 4x4 block, the 9x9 luma window at (16 mbx + 4 bx + (mvx >> 2) - 2, ...) clamped to the
 *          picture; every reference macroblock it touches
 *   intra: the neighbours the record marks available (A, B, D by the chroma mode, C by 4x4 block 5 or 8x8 block 1,
 *          never for Intra16x16), in this picture's map; none for I_PCM */
long port_cov_map[12];   /* coverage counters, printed by record_fuzz_maps.c */
static int clampi(int v, int lo, int hi) { return v < lo ? lo : v > hi ? hi : v; }
static int ref_map(const uint8_t *maps, const E264PicDesc *pd, int slot, int mbx, int mby) {
	const int nmb = pd->width_mbs * pd->height_mbs;
	if (!(pd->taint >> slot & 1)) return 0;
	return maps[(size_t)slot * nmb + mby * pd->width_mbs + mbx];
}
void port_error_map(uint8_t *maps, const E264PicDesc *pd, const E264MbRec *recs) {
	if (!pd->err_pic) return;
	const int W = pd->width_mbs, H = pd->height_mbs, nmb = W * H;
	uint8_t *cur = maps + (size_t)pd->dst_slot * nmb;
	for (int a = 0; a < nmb; a++) {
		const E264MbRec *r = recs + a;
		const int mbx = a % W, mby = a / W;
		int e = 0;
		if (r->kind == MBK_INTER) {
			for (int l = 0; l < 2; l++) for (int b = 0; b < 16; b++) {
				if (r->ref_idx[l][b >> 2] < 0) continue;
				int slot = r->ref_pic[l][b >> 2];
				int X0 = mbx * 16 + e264_blk_x(b) * 4 + (r->mv[l][b][0] >> 2) - 2, Y0 = mby * 16 + e264_blk_y(b) * 4 + (r->mv[l][b][1] >> 2) - 2;
				int x0 = clampi(X0, 0, W * 16 - 1) / 16, x1 = clampi(X0 + 8, 0, W * 16 - 1) / 16;
				int y0 = clampi(Y0, 0, H * 16 - 1) / 16, y1 = clampi(Y0 + 8, 0, H * 16 - 1) / 16;
				int blk = 0;
				for (int y = y0; y <= y1; y++) for (int x = x0; x <= x1; x++) { int v = ref_map(maps, pd, slot, x, y); if (v > blk) blk = v; }
				/* coverage: clamped at the left, right, top, bottom border; 1, 2 or 4 macroblocks touched; list 1 gives the maximum */
				port_cov_map[0] += X0 < 0; port_cov_map[1] += X0 + 8 > W * 16 - 1; port_cov_map[2] += Y0 < 0; port_cov_map[3] += Y0 + 8 > H * 16 - 1;
				port_cov_map[4 + (x1 > x0) + (y1 > y0) + ((x1 > x0) && (y1 > y0))]++;
				port_cov_map[8] += l == 1 && r->ref_idx[0][b >> 2] >= 0 && blk > e;
				port_cov_map[9] += blk == 100 && (pd->taint >> slot & 1) && ref_map(maps, pd, slot, x0, y0) == 100;
				if (blk > e) e = blk;
			}
		} else if (r->kind != MBK_IPCM) {
			int un = r->chroma_mode >> 4;
			if (!(un & 1)) e = cur[a - 1] > e ? cur[a - 1] : e;
			if (!(un & 2)) e = cur[a - W] > e ? cur[a - W] : e;
			if (!(un & 8)) e = cur[a - W - 1] > e ? cur[a - W - 1] : e;
			int c = (r->kind == MBK_I4x4 && !(r->modes[5] & 0x40)) || (r->kind == MBK_I8x8 && !(r->modes[1] & 0x40));
			if (c) { e = cur[a - W + 1] > e ? cur[a - W + 1] : e; port_cov_map[r->kind == MBK_I4x4 ? 10 : 11]++; }
		}
		cur[a] = (uint8_t)(r->err > e ? r->err : e);
	}
}
