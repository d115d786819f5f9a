// The host build of edge264_b200/csrc/mc_math.cuh's interpolation, weighting and residual add as a shared library over
// arrays, for tests/test_pixel_spec.py and tests/test_residual_spec.py to run against the standard's equations in numpy
// (built there).  Test infrastructure.
#include <cstdint>
#include "../../edge264_b200/csrc/mc_math.cuh"

extern "C" {
// n words: wp_word with per-word parameters
void mcl_wp_word(int n, const uint32_t *a, const uint32_t *b, const int32_t *wa, const int32_t *wb, const int32_t *rnd, const int32_t *sh, const int32_t *o, uint32_t *out) {
	for (int i = 0; i < n; i++) out[i] = wp_word(a[i], b[i], wa[i], wb[i], rnd[i], sh[i], o[i]);
}
void mcl_avg4(int n, const uint32_t *a, const uint32_t *b, uint32_t *out) {
	for (int i = 0; i < n; i++) out[i] = mc_avg4(a[i], b[i]);
}
// n 3x3 windows (three row words each, bytes 0..2 used) at eighth-sample fractions fx, fy: 2x2 samples packed per window
void mcl_chroma2x2(int n, const uint32_t *rows, const int32_t *fx, const int32_t *fy, uint32_t *out) {
	for (int i = 0; i < n; i++) out[i] = mc_chroma2x2(rows[3 * i], rows[3 * i + 1], rows[3 * i + 2], fx[i], fy[i]);
}
// n 9x9 luma windows (nine rows of three words each, sample x = -2 of the block in byte 0 of word 0) at quarter-sample
// fractions fx, fy: four row words of the 4x4 block per window
void mcl_luma4x4(int n, const uint32_t *win, const int32_t *fx, const int32_t *fy, uint32_t *out) {
	for (int i = 0; i < n; i++) mc_luma4x4((const uint32_t (*)[3])(win + 27 * i), fx[i], fy[i], out + 4 * i);
}
// n words of four predicted samples plus two words of four int16 residuals each
void mcl_add_res4(int n, const uint32_t *p, const uint32_t *r01, const uint32_t *r23, uint32_t *out) {
	for (int i = 0; i < n; i++) out[i] = mc_add_res4(p[i], r01[i], r23[i]);
}
}
