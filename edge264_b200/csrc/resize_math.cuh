/* resize_math.cuh — the arithmetic of the resized output (include/edge264_packed.h) that does not depend on how threads
 * share the work: which source samples one output sample reads along one axis, with which weights, and the single
 * rounding floor((2N + D) / 2D).  Host-compilable: tests/test_resized_output.py checks e264_rs_round against Python
 * integers, and the CPU restatement (tests/native/port_resized_backend.c) uses the same two functions.
 *
 * Along an axis of s source samples resampled to t, output sample x covers [x s, (x + 1) s) in units of 1 / t source
 * sample, and source sample i covers [i t, (i + 1) t).  Their overlap a(x, i) is t for every source sample of the span
 * but the first and the last, whose weights are t - cut_first and t - cut_last (a span of one sample: weight s).
 *
 * Rounding without a 64-bit division.  N <= 255 D, D = s_w s_h < 2^29 (the runtime refuses larger pictures), so
 * A = 2N + D < 2^38 and 2D < 2^30 are exact doubles.  With inv = fl(1 / 2D), the computed q = fl(fl(A inv) + 2^-32) is
 * within 2^-32 +- 2^-43 of the exact quotient A / 2D <= 255.5 (two or three roundings of relative error 2^-53 each).  When
 * A / 2D is an integer k, q lies strictly between k and k + 1.  Otherwise its fraction lies in [1 / 2D, 1 - 1 / 2D], and
 * 1 / 2D > 2^-30 keeps q inside the same integer interval.  So the truncation of q is floor(A / 2D), whether or not the
 * compiler fuses the multiply and the add. */
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define RS_FN __host__ __device__ __forceinline__
#else
#define RS_FN static inline
#endif

typedef struct RsSpan { int32_t first, last, cut_first, cut_last; } RsSpan;

/* the span of output sample x (0 <= x < t); x s and s t must stay below 2^31 */
RS_FN RsSpan e264_rs_span(int x, int s, int t) {
	const int lo = x * s, hi = lo + s;
	RsSpan r;
	r.first = lo / t; r.last = (hi - 1) / t;
	r.cut_first = lo - r.first * t; r.cut_last = (r.last + 1) * t - hi;
	return r;
}

/* the per-plane reciprocal of 2D */
RS_FN double e264_rs_inv(int64_t d) { return 1.0 / (double)(2 * d); }

/* floor((2n + d) / 2d) for 0 <= n <= 255 d, d < 2^29, inv = e264_rs_inv(d) */
RS_FN int e264_rs_round(int64_t n, int64_t d, double inv) { return (int)((double)(2 * n + d) * inv + 0x1p-32); }
