/* mc_math.cuh — quarter-sample luma and eighth-sample chroma interpolation (8.4.2.2) of ONE 4x4 luma block (2x2 per
 * chroma plane) by ONE thread, entirely in registers.
 *
 * The thread holds the block's 9x9 reference window as nine rows of three 32-bit words (sample x = -2 of the block
 * in byte 0 of word 0).  The six-tap sums of four neighbouring samples come from two dot-product instructions each
 * (dp4a: taps 1,-5,20,20 | -5,1,0,0 against byte windows cut out with funnel shifts); the vertical cases run the same
 * code on the transposed window (byte-permute 4x4 transposes) — the interpolation is symmetric under transposition,
 * including the reference's order of passes for the centre sample (vertical first when xFrac is odd, edge264_inter.c:
 * 559-640), whose wrapping int16 combination (edge264_inter.c:4-9) is reproduced bit for bit.  The weighted combination
 * of the predictions (8.4.2.3) is here too.
 * Host-compilable: tests/mc_math_check.cpp runs these functions against the oracle's per-sample restatement, and
 * tests/test_pixel_spec.py runs the chroma interpolation and the weighting against the standard's equations in numpy. */
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define MC_FN __device__ __forceinline__
/* four unsigned bytes of a times four signed bytes of b, plus c (the CUDA intrinsic offers only the same-sign forms) */
MC_FN int mc_dp4a(uint32_t a, int b, int c) { int d; asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
MC_FN uint32_t mc_fsr(uint32_t lo, uint32_t hi, int bits) { return __funnelshift_r(lo, hi, bits); }   /* bits in 0..31 */
MC_FN uint32_t mc_prmt(uint32_t a, uint32_t b, uint32_t sel) { return __byte_perm(a, b, sel); }
#else
#define MC_FN static inline
MC_FN int mc_dp4a(uint32_t a, int b, int c) { for (int k = 0; k < 4; k++) c += (int)((a >> (8 * k)) & 255) * (int)(int8_t)((uint32_t)b >> (8 * k)); return c; }
MC_FN uint32_t mc_fsr(uint32_t lo, uint32_t hi, int bits) { return (uint32_t)((((uint64_t)hi << 32) | lo) >> (bits & 31)); }
MC_FN uint32_t mc_prmt(uint32_t a, uint32_t b, uint32_t sel) {
	uint64_t v = ((uint64_t)b << 32) | a; uint32_t r = 0;
	for (int k = 0; k < 4; k++) r |= (uint32_t)((v >> (8 * ((sel >> (4 * k)) & 7))) & 255) << (8 * k);
	return r;
}
#endif

MC_FN int mc_clip255(int v) { return v < 0 ? 0 : v > 255 ? 255 : v; }
MC_FN uint32_t mc_pack4(int a, int b, int c, int d) { return (uint32_t)a | (uint32_t)b << 8 | (uint32_t)c << 16 | (uint32_t)d << 24; }
/* four predicted samples (bytes of p) plus four int16 residuals (r01: the first two, r23: the last two), clipped; the sum
 * wraps to 16 bits first like the reference's 16-bit adds (residuals of conforming streams never make it wrap) */
MC_FN uint32_t mc_add_res4(uint32_t p, uint32_t r01, uint32_t r23) {
	return mc_pack4(mc_clip255((int16_t)((int)(p & 255u) + (int16_t)(r01 & 0xffffu))), mc_clip255((int16_t)((int)((p >> 8) & 255u) + (int16_t)(r01 >> 16))),
	                mc_clip255((int16_t)((int)((p >> 16) & 255u) + (int16_t)(r23 & 0xffffu))), mc_clip255((int16_t)((int)(p >> 24) + (int16_t)(r23 >> 16))));
}
/* rounded-up average of four bytes at once */
MC_FN uint32_t mc_avg4(uint32_t a, uint32_t b) { return (a | b) - (((a ^ b) >> 1) & 0x7f7f7f7fu); }

/* 8.4.2.3 on four packed samples in ONE form: (sat16(a * wa + b * wb + rnd) >> sh) + o, clipped.  Implicit bi-prediction:
 * wa = w0, wb = w1, rnd = 2^logWD, sh = logWD + 1, o = 0; explicit bi-prediction: the same with the offsets folded into
 * rnd = ((o0 + o1 + 1) | 1) << logWD and o = 0, saturated to int16 as the reference does (edge264_inter.c:17-29,
 * :1176-1178; it differs from the standard only at logWD 7, oracle/port_recon.c wp_bi, counted by
 * tests/test_pixel_spec.py); explicit weighting of a single prediction: wa = w, wb = 0, rnd = 2^(logWD-1) (0 when
 * logWD = 0), sh = logWD.  Only explicit bi-prediction can reach the saturation (reference edge264_inter.c:1140-1180 keeps
 * five variants). */
MC_FN uint32_t wp_word(uint32_t a, uint32_t b, int wa, int wb, int rnd, int sh, int o) {
	uint32_t r = 0;
#pragma unroll
	for (int k = 0; k < 4; k++) {
		const int pa = (a >> (8 * k)) & 255, pb = (b >> (8 * k)) & 255, s = pa * wa + pb * wb + rnd, lo = s < -32768 ? -32768 : s;
		r |= (uint32_t)mc_clip255(((lo > 32767 ? 32767 : lo) >> sh) + o) << (8 * k);
	}
	return r;
}

/* six-tap sums (1,-5,20,20,-5,1) at the four sample positions x = 0..3 of a row whose samples x = -2..9 are the
 * bytes of (w0, w1, w2): s[x] = p[x-2] - 5 p[x-1] + 20 p[x] + 20 p[x+1] - 5 p[x+2] + p[x+3] */
MC_FN void mc_tap6x4(uint32_t w0, uint32_t w1, uint32_t w2, int s[4]) {
	const int c1 = 0x1414fb01, c2 = 0x000001fb;
	s[0] = mc_dp4a(w0, c1, mc_dp4a(w1, c2, 0));
	s[1] = mc_dp4a(mc_fsr(w0, w1, 8), c1, mc_dp4a(mc_fsr(w1, w2, 8), c2, 0));
	s[2] = mc_dp4a(mc_fsr(w0, w1, 16), c1, mc_dp4a(mc_fsr(w1, w2, 16), c2, 0));
	s[3] = mc_dp4a(mc_fsr(w0, w1, 24), c1, mc_dp4a(mc_fsr(w1, w2, 24), c2, 0));
}
/* the rounded half-sample row: clip((sum + 16) >> 5), four samples packed */
MC_FN uint32_t mc_half4(uint32_t w0, uint32_t w1, uint32_t w2) {
	int s[4]; mc_tap6x4(w0, w1, w2, s);
	return mc_pack4(mc_clip255((s[0] + 16) >> 5), mc_clip255((s[1] + 16) >> 5), mc_clip255((s[2] + 16) >> 5), mc_clip255((s[3] + 16) >> 5));
}

/* transpose of a 4x4 byte block held as four row words */
MC_FN void mc_tr4(uint32_t a, uint32_t b, uint32_t c, uint32_t d, uint32_t o[4]) {
	const uint32_t t0 = mc_prmt(a, b, 0x5140), t1 = mc_prmt(c, d, 0x5140), t2 = mc_prmt(a, b, 0x7362), t3 = mc_prmt(c, d, 0x7362);
	o[0] = mc_prmt(t0, t1, 0x5410); o[1] = mc_prmt(t0, t1, 0x7632); o[2] = mc_prmt(t2, t3, 0x5410); o[3] = mc_prmt(t2, t3, 0x7632);
}
/* transpose of the 9x9 window (12x12 bytes, the bytes beyond 9 are don't-cares) */
MC_FN void mc_tr_window(const uint32_t w[9][3], uint32_t t[9][3]) {
	uint32_t o[4];
#pragma unroll
	for (int bx = 0; bx < 3; bx++)
#pragma unroll
		for (int by = 0; by < 3; by++) {
			mc_tr4(w[by * 4][bx], by * 4 + 1 < 9 ? w[by * 4 + 1][bx] : 0u, by * 4 + 2 < 9 ? w[by * 4 + 2][bx] : 0u, by * 4 + 3 < 9 ? w[by * 4 + 3][bx] : 0u, o);
#pragma unroll
			for (int k = 0; k < 4; k++) if (bx * 4 + k < 9) t[bx * 4 + k][by] = o[k];
		}
}

/* a, b, c: horizontal half samples of rows y = 0..3 (window rows 2..5), averaged with the full sample left or right of them */
MC_FN void mc_luma_h(const uint32_t w[9][3], int fx, uint32_t out[4]) {
#pragma unroll
	for (int y = 0; y < 4; y++) {
		const uint32_t b = mc_half4(w[y + 2][0], w[y + 2][1], w[y + 2][2]);
		/* full samples G at x = 0..3 are bytes 2..5 of the row, the right neighbours bytes 3..6 */
		const uint32_t g = fx == 3 ? mc_fsr(w[y + 2][0], w[y + 2][1], 24) : mc_fsr(w[y + 2][0], w[y + 2][1], 16);
		out[y] = fx == 2 ? b : mc_avg4(b, g);
	}
}
/* f, j, q (xFrac 2): centre sample with the horizontal pass first — unrounded six-tap sums of rows -2..6, then the
 * vertical pass in the reference's wrapping int16 arithmetic; f and q average it with the horizontal half sample of row
 * y (yFrac 1) or y + 1 (yFrac 3), whose sums are already there */
MC_FN void mc_luma_center(const uint32_t w[9][3], int fy, uint32_t out[4]) {
	int t[9][4];
#pragma unroll
	for (int r = 0; r < 9; r++) mc_tap6x4(w[r][0], w[r][1], w[r][2], t[r]);
#pragma unroll
	for (int y = 0; y < 4; y++) {
		int v[4];
#pragma unroll
		for (int x = 0; x < 4; x++) {
			const int af = t[y][x] + t[y + 5][x], be = t[y + 1][x] + t[y + 4][x], cd = t[y + 2][x] + t[y + 3][x];
			const int t16 = (int)(int16_t)(((af - be) >> 2) + (cd - be));
			v[x] = mc_clip255(((t16 >> 2) + cd + 32) >> 6);
		}
		uint32_t j = mc_pack4(v[0], v[1], v[2], v[3]);
		if (fy != 2) {
			/* (selects, not a computed row index: the arrays must stay in registers) */
			const int b0 = fy == 3 ? t[y + 3][0] : t[y + 2][0], b1 = fy == 3 ? t[y + 3][1] : t[y + 2][1], b2 = fy == 3 ? t[y + 3][2] : t[y + 2][2], b3 = fy == 3 ? t[y + 3][3] : t[y + 2][3];
			const uint32_t b = mc_pack4(mc_clip255((b0 + 16) >> 5), mc_clip255((b1 + 16) >> 5), mc_clip255((b2 + 16) >> 5), mc_clip255((b3 + 16) >> 5));
			j = mc_avg4(j, b);
		}
		out[y] = j;
	}
}
/* d, h, n (xFrac 0): the horizontal case of the transposed window */
MC_FN void mc_luma_v(const uint32_t w[9][3], int fy, uint32_t out[4]) {
	uint32_t t[9][3], o[4];
	mc_tr_window(w, t);
	mc_luma_h(t, fy, o);
	mc_tr4(o[0], o[1], o[2], o[3], out);
}
/* i, k (yFrac 2, xFrac odd): centre sample with the vertical pass first = the centre case of the transposed window */
MC_FN void mc_luma_center_v(const uint32_t w[9][3], int fx, uint32_t out[4]) {
	uint32_t t[9][3], o[4];
	mc_tr_window(w, t);
	mc_luma_center(t, fx, o);
	mc_tr4(o[0], o[1], o[2], o[3], out);
}
/* e, g, p, r: average of a horizontal half sample (row y or y+1) and a vertical half sample (column x or x+1) */
MC_FN void mc_luma_diag(const uint32_t w[9][3], int fx, int fy, uint32_t out[4]) {
	uint32_t t[9][3], vh[4], vt[4];
	mc_tr_window(w, t);
	/* window column 2 + x (+1 when xFrac is 3) holds the vertical half samples of output column x; selects, not computed indices */
#pragma unroll
	for (int x = 0; x < 4; x++) vh[x] = fx == 3 ? mc_half4(t[3 + x][0], t[3 + x][1], t[3 + x][2]) : mc_half4(t[2 + x][0], t[2 + x][1], t[2 + x][2]);      /* column x: samples y = 0..3 */
	mc_tr4(vh[0], vh[1], vh[2], vh[3], vt);
#pragma unroll
	for (int y = 0; y < 4; y++) out[y] = mc_avg4(fy == 3 ? mc_half4(w[3 + y][0], w[3 + y][1], w[3 + y][2]) : mc_half4(w[2 + y][0], w[2 + y][1], w[2 + y][2]), vt[y]);
}

/* interpolation class of a fraction: 0 full sample, 1 horizontal (yFrac 0), 2 vertical (xFrac 0), 3 diagonal (both odd),
 * 4 centre horizontal-first (xFrac 2), 5 centre vertical-first (yFrac 2, xFrac odd) */
MC_FN int mc_class(int fx, int fy) { return !(fx | fy) ? 0 : fy == 0 ? 1 : fx == 0 ? 2 : fx == 2 ? 4 : fy == 2 ? 5 : 3; }

/* one 4x4 luma block at fraction (fx, fy) in quarter samples */
MC_FN void mc_luma4x4(const uint32_t w[9][3], int fx, int fy, uint32_t out[4]) {
	switch (mc_class(fx, fy)) {
	case 0:
#pragma unroll
		for (int y = 0; y < 4; y++) out[y] = mc_fsr(w[y + 2][0], w[y + 2][1], 16);
		break;
	case 1: mc_luma_h(w, fx, out); break;
	case 2: mc_luma_v(w, fy, out); break;
	case 3: mc_luma_diag(w, fx, fy, out); break;
	case 4: mc_luma_center(w, fy, out); break;
	default: mc_luma_center_v(w, fx, out); break;
	}
}

/* 2x2 chroma samples of one plane: c[r] = bytes x = 0..3 of window row r (r = 0..2, x = 0..2 used), fractions in
 * eighth samples.  Returns the four samples packed (row 0: bytes 0-1, row 1: bytes 2-3). */
MC_FN uint32_t mc_chroma2x2(uint32_t c0, uint32_t c1, uint32_t c2, int fx, int fy) {
	const int wa = (8 - fx) * (8 - fy), wb = fx * (8 - fy), wc = (8 - fx) * fy, wd = fx * fy;
	const int k01 = wa | wb << 8, k23 = wc | wd << 8;                /* dp4a weights for bytes (x, x+1) of the upper / lower row */
	const uint32_t r0a = mc_prmt(c0, c1, 0x5410), r0b = mc_prmt(c0, c1, 0x6521);   /* (c0[0],c0[1],c1[0],c1[1]) and (c0[1],c0[2],c1[1],c1[2]) */
	const uint32_t r1a = mc_prmt(c1, c2, 0x5410), r1b = mc_prmt(c1, c2, 0x6521);
	const int kk = k01 | k23 << 16;
	const int v00 = (mc_dp4a(r0a, kk, 32)) >> 6, v01 = (mc_dp4a(r0b, kk, 32)) >> 6, v10 = (mc_dp4a(r1a, kk, 32)) >> 6, v11 = (mc_dp4a(r1b, kk, 32)) >> 6;
	return mc_pack4(v00, v01, v10, v11);
}
