// The host build of edge264_b200/csrc/dbk_math.cuh (the device's boundary strength and line filters) as a shared library
// over arrays, for tests/test_deblock_spec.py to run against the standard's equations in numpy (built there).  Test
// infrastructure.
#include <cstdint>
#include "../../edge264_b200/csrc/dbk_math.cuh"

extern "C" {
// n luma lines, 8 samples each (p3 p2 p1 p0 q0 q1 q2 q3), filtered in place by the macroblock edges' instantiation.  The
// sample filter sets any4 whenever a line of its warp has bS 4, so a line of bS 4 always runs with it set, and a line of
// bS 1..3 runs either way: any4[i] is used where bS is not 4
void dbl_luma(int n, int32_t *s, const int32_t *bs, const int32_t *alpha, const int32_t *beta, const int32_t *tc0, const int32_t *any4) {
	for (int i = 0; i < n; i++) {
		int32_t *v = s + 8 * i;
		dbk_line_luma<true>(v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7], bs[i], alpha[i], beta[i], tc0[i], bs[i] == 4 || any4[i]);
	}
}
// the same lines through the internal edges' instantiation (no bS 4 there), for bS 1..3
void dbl_luma_internal(int n, int32_t *s, const int32_t *bs, const int32_t *alpha, const int32_t *beta, const int32_t *tc0) {
	for (int i = 0; i < n; i++) {
		int32_t *v = s + 8 * i;
		dbk_line_luma<false>(v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7], bs[i], alpha[i], beta[i], tc0[i], false);
	}
}
// n chroma lines, 4 samples each (p1 p0 q0 q1)
void dbl_chroma(int n, int32_t *s, const int32_t *bs, const int32_t *alpha, const int32_t *beta, const int32_t *tc0) {
	for (int i = 0; i < n; i++) {
		int32_t *v = s + 4 * i;
		dbk_line_chroma(v[0], v[1], v[2], v[3], bs[i], alpha[i], beta[i], tc0[i]);
	}
}
// n block pairs: bS between block bp[i] of p[i] and block bq[i] of q[i]
void dbl_bs(int n, const E264MbRec *p, const int32_t *bp, const E264MbRec *q, const int32_t *bq, const int32_t *mb_edge, int32_t *out) {
	for (int i = 0; i < n; i++) out[i] = dbk_bs_pair(p + i, bp[i], q + i, bq[i], mb_edge[i] != 0);
}
}
