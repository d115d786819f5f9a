/* dbk_math.cuh — the deblocking arithmetic of one edge segment or one line of samples (8.7.2), shared by the digest and
 * the sample filter of deblock_kernels.cuh.
 *   dbk_bs_pair       8.7.2.1, the boundary strength between two 4x4 luma blocks of two records
 *   dbk_line_luma     8.7.2.3 / 8.7.2.4 on one luma line p3..q3, branch-free
 *   dbk_line_chroma   the same on one chroma line p1..q1
 * Host-compilable: tests/native/dbk_math_lib.cpp builds these functions for the host, and tests/test_deblock_spec.py runs
 * them against the standard's equations in numpy (tests/spec_deblock.py). */
#pragma once
#include <stdint.h>
#include "records.h"
#include "mc_math.cuh"

#ifdef __CUDACC__
#define DBK_FN __device__ __forceinline__
#else
#define DBK_FN static inline
static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }
#endif
#ifdef __CUDA_ARCH__
#define DBK_SAD(a, b) __sad(a, b, 0)
#else
#define DBK_SAD(a, b) ((unsigned)((a) < (b) ? (b) - (a) : (a) - (b)))
#endif

DBK_FN int dbk_iabs(int v) { return v < 0 ? -v : v; }

/* 8.7.2.1 for one edge segment between 4x4 blocks bp of p and bq of q.  Every candidate outcome is computed and the result
 * is selected, so the 32 lanes of a digest (different edges, different cases) run one instruction stream; the records
 * are read whole even where they do not matter (intra macroblocks), which is harmless. */
DBK_FN bool dbk_far(uint32_t a, uint32_t b) {      /* two packed quarter-sample vectors differ by 4 or more */
	return dbk_iabs((int)(short)(a & 0xffffu) - (int)(short)(b & 0xffffu)) >= 4 || dbk_iabs((int)(short)(a >> 16) - (int)(short)(b >> 16)) >= 4;
}
DBK_FN int dbk_bs_pair(const E264MbRec *p, int bp, const E264MbRec *q, int bq, bool mb_edge) {
	const bool intra = p->kind != MBK_INTER || q->kind != MBK_INTER;
	const bool coef = (((p->coded >> bp) | (q->coded >> bq)) & 1) != 0;
	const int ip = bp >> 2, iq = bq >> 2;
	const int p0 = p->ref_idx[0][ip] < 0 ? -1 : p->ref_pic[0][ip], p1 = p->ref_idx[1][ip] < 0 ? -1 : p->ref_pic[1][ip];
	const int q0 = q->ref_idx[0][iq] < 0 ? -1 : q->ref_pic[0][iq], q1 = q->ref_idx[1][iq] < 0 ? -1 : q->ref_pic[1][iq];
	const bool same = (p0 == q0 && p1 == q1) || (p0 == q1 && p1 == q0);
	const uint32_t pm0 = *(const uint32_t *)p->mv[0][bp], pm1 = *(const uint32_t *)p->mv[1][bp];
	const uint32_t qm0 = *(const uint32_t *)q->mv[0][bq], qm1 = *(const uint32_t *)q->mv[1][bq];
	const bool f00 = dbk_far(pm0, qm0), f11 = dbk_far(pm1, qm1), f01 = dbk_far(pm0, qm1), f10 = dbk_far(pm1, qm0);
	const bool straight = f00 || f11, crossed = f01 || f10;
	/* both lists: distinct pictures pair the vectors by picture, the same picture twice needs both pairings to differ;
	 * one list: the vectors of the lists in use */
	const bool one = p0 >= 0 ? (q0 >= 0 ? f00 : f01) : (q0 >= 0 ? f10 : f11);
	const bool mv = p0 >= 0 && p1 >= 0 ? (p0 != p1 ? (p0 == q0 ? straight : crossed) : straight && crossed) : one;
	return intra ? (mb_edge ? 4 : 3) : coef ? 2 : !same ? 1 : (int)mv;
}

/* ---- sample filters on one line across an edge, samples as ints ----
 * Branch-free: a line that is not filtered runs the same arithmetic with its clipping bounds set to zero (a lone
 * warp pays ~10 cycles for every branch it resolves). */
template <bool STRONG>
DBK_FN void dbk_line_luma(int &p3, int &p2, int &p1, int &p0, int &q0, int &q1, int &q2, int &q3, int bs, int alpha, int beta, int tc0, bool any4) {
	const int ad = DBK_SAD(p0, q0);
	const bool f = bs != 0 && ad < alpha && DBK_SAD(p1, p0) < beta && DBK_SAD(q1, q0) < beta;
	const bool ap = DBK_SAD(p2, p0) < beta, aq = DBK_SAD(q2, q0) < beta;
	const int tcp = f && ap ? tc0 : 0, tcq = f && aq ? tc0 : 0;
	const int tc = f ? tc0 + (int)ap + (int)aq : 0;
	const int d = min(max((((q0 - p0) << 2) + (p1 - q1) + 4) >> 3, -tc), tc);
	const int avg = (p0 + q0 + 1) >> 1;
	int n_p1 = p1 + min(max((p2 + avg - (p1 << 1)) >> 1, -tcp), tcp);
	int n_q1 = q1 + min(max((q2 + avg - (q1 << 1)) >> 1, -tcq), tcq);
	int n_p0 = mc_clip255(p0 + d), n_q0 = mc_clip255(q0 - d);
	if (STRONG && any4) {   /* bS 4 exists only on macroblock edges; `any4` is uniform over the warp */
		const bool s4 = f && bs == 4;
		const bool small = ad < ((alpha >> 2) + 2);
		const bool sp = ap && small, sq = aq && small;
		const int s_p0 = sp ? (p2 + 2 * p1 + 2 * p0 + 2 * q0 + q1 + 4) >> 3 : (2 * p1 + p0 + q1 + 2) >> 2;
		const int s_p1 = sp ? (p2 + p1 + p0 + q0 + 2) >> 2 : p1;
		const int s_p2 = sp ? (2 * p3 + 3 * p2 + p1 + p0 + q0 + 4) >> 3 : p2;
		const int s_q0 = sq ? (p1 + 2 * p0 + 2 * q0 + 2 * q1 + q2 + 4) >> 3 : (2 * q1 + q0 + p1 + 2) >> 2;
		const int s_q1 = sq ? (p0 + q0 + q1 + q2 + 2) >> 2 : q1;
		const int s_q2 = sq ? (2 * q3 + 3 * q2 + q1 + q0 + p0 + 4) >> 3 : q2;
		n_p0 = s4 ? s_p0 : n_p0; n_p1 = s4 ? s_p1 : n_p1; p2 = s4 ? s_p2 : p2;
		n_q0 = s4 ? s_q0 : n_q0; n_q1 = s4 ? s_q1 : n_q1; q2 = s4 ? s_q2 : q2;
	}
	p0 = n_p0; p1 = n_p1; q0 = n_q0; q1 = n_q1;
}
DBK_FN void dbk_line_chroma(int p1, int &p0, int &q0, int q1, int bs, int alpha, int beta, int tc0) {
	const bool f = bs != 0 && DBK_SAD(p0, q0) < alpha && DBK_SAD(p1, p0) < beta && DBK_SAD(q1, q0) < beta;
	const int tc = f ? tc0 + 1 : 0;
	const int d = min(max((((q0 - p0) << 2) + (p1 - q1) + 4) >> 3, -tc), tc);
	const bool s4 = f && bs == 4;
	const int n_p0 = s4 ? (2 * p1 + p0 + q1 + 2) >> 2 : mc_clip255(p0 + d);
	const int n_q0 = s4 ? (2 * q1 + q0 + p1 + 2) >> 2 : mc_clip255(q0 - d);
	p0 = n_p0; q0 = n_q0;
}
