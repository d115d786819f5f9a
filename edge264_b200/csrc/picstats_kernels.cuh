/* picstats_kernels.cuh — e264_picstats_kernel: the picture statistics of one picture (include/edge264_picstats.h, layout
 * E264_PICSTATS_* in records.h), read from the finished frame slot.
 *
 * A warp takes one macroblock at a time, one row per lane: lanes 0..15 load the 16 luma rows as aligned 16-byte words,
 * lanes 16..23 the 8 Cb rows and lanes 24..31 the 8 Cr rows as 8-byte words (strides are multiples of 16, and Cr starts
 * half a chroma stride after Cb).  Sums of the bytes (__vsadu4 against 0) and of their squares (__dp4a of a word with
 * itself) are exact; shuffles add them over the lanes of each plane, and lanes 0, 16 and 24 store the macroblock's words.
 *
 * The histogram goes to a 3 x 256 sub-histogram per block in shared memory.  For each of its (up to) 16 samples a lane
 * forms the key plane << 8 | value; lanes with equal keys find each other with __match_any_sync and the lowest of them
 * adds the group's size.  A constant plane (a blank frame, the chroma of a luma-only picture) then costs one shared
 * atomic per key and sample position instead of 32 serialised ones, on the same code path as any other picture.  Samples
 * outside the cropping rectangle are left out through a per-lane column mask, which is all ones for a row inside it, so
 * only macroblocks on the rectangle's border lose samples.  Blocks stride over the macroblocks and load the next one
 * before counting the current.  At the end a block adds its non-zero bins to the global histogram with integer atomics:
 * exact, so the result does not depend on their order.  The global histogram must be zero before the launch.
 * Launched by the runtime after the picture's reconstruction and deblocking launches, and only for decoders that asked
 * for the statistics. */
#pragma once
#include "recon_kernels.cuh"

#define PS_WARPS 16
#define PS_THREADS (PS_WARPS * 32)

struct PicStatsArgs {
	const uint8_t *y, *c;              /* the frame slot's luma plane and chroma plane */
	int32_t stride_y, stride_c;        /* chroma rows alternate Cb, Cr inside stride_c */
	int32_t w_mbs, h_mbs;
	int32_t left, top, right, bottom;  /* the cropping rectangle, luma samples: [left, right) x [top, bottom), all even */
	uint32_t *out;                     /* E264_PICSTATS_BYTES(w_mbs * h_mbs) bytes */
};

/* row r of plane p of macroblock (mbx, mby), as a 16-byte word (chroma: the upper 8 bytes 0) */
__device__ __forceinline__ uint4 ps_load(const PicStatsArgs &A, int p, int r, int mbx, int mby) {
	if (p == 0) return __ldg((const uint4 *)(A.y + (size_t)(mby * 16 + r) * A.stride_y + mbx * 16));
	const uint2 u = __ldg((const uint2 *)(A.c + (size_t)(mby * 8 + r) * A.stride_c + mbx * 8 + (p == 2 ? A.stride_c >> 1 : 0)));
	return make_uint4(u.x, u.y, 0u, 0u);
}

__global__ void __launch_bounds__(PS_THREADS) e264_picstats_kernel(const __grid_constant__ PicStatsArgs A) {
	__shared__ uint32_t hist[3 * 256];
	const int lane = threadIdx.x & 31;
	const int p = lane < 16 ? 0 : lane < 24 ? 1 : 2, r = p ? lane & 7 : lane, sh = p ? 1 : 0, n = 16 >> sh;
	const int left = A.left >> sh, right = A.right >> sh, top = A.top >> sh, bottom = A.bottom >> sh;
	const int nmb = A.w_mbs * A.h_mbs, step = gridDim.x * PS_WARPS;
	uint32_t *sum = A.out + E264_PICSTATS_SUM / 4 + p * nmb, *sum_sq = A.out + E264_PICSTATS_SUM_SQ(nmb) / 4 + p * nmb;
	for (int i = threadIdx.x; i < 3 * 256; i += PS_THREADS) hist[i] = 0;
	__syncthreads();
	int mb = blockIdx.x * PS_WARPS + (threadIdx.x >> 5);   /* the same for the whole warp */
	uint4 v = make_uint4(0u, 0u, 0u, 0u);
	if (mb < nmb) v = ps_load(A, p, r, mb % A.w_mbs, mb / A.w_mbs);
	for (; mb < nmb; mb += step) {
		const int mby = mb / A.w_mbs, mbx = mb - mby * A.w_mbs, nx = mb + step;
		uint4 next = make_uint4(0u, 0u, 0u, 0u);
		if (nx < nmb) next = ps_load(A, p, r, nx % A.w_mbs, nx / A.w_mbs);
		/* sums over the macroblock */
		uint32_t s = __vsadu4(v.x, 0u) + __vsadu4(v.y, 0u) + __vsadu4(v.z, 0u) + __vsadu4(v.w, 0u);
		uint32_t q = __dp4a(v.x, v.x, 0u) + __dp4a(v.y, v.y, 0u) + __dp4a(v.z, v.z, 0u) + __dp4a(v.w, v.w, 0u);
#pragma unroll
		for (int o = 1; o < 8; o <<= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); q += __shfl_xor_sync(0xffffffffu, q, o); }
		const uint32_t s8 = __shfl_xor_sync(0xffffffffu, s, 8), q8 = __shfl_xor_sync(0xffffffffu, q, 8);
		if (p == 0) { s += s8; q += q8; }
		if (lane == 0 || lane == 16 || lane == 24) { sum[mb] = s; sum_sq[mb] = q; }
		/* histogram of the samples inside the cropping rectangle */
		const int x0 = mbx * n, y = mby * n + r;
		const int lo = min(max(left - x0, 0), n), hi = min(max(right - x0, 0), n);
		const uint32_t cols = y >= top && y < bottom ? ((1u << hi) - 1u) & ~((1u << lo) - 1u) : 0u;
		const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
		for (int i = 0; i < 16; i++) {
			const uint32_t key = cols >> i & 1u ? (uint32_t)p << 8 | (w[i >> 2] >> (8 * (i & 3)) & 255u) : 0xffffffffu;
			const uint32_t same = __match_any_sync(0xffffffffu, key);
			if (key != 0xffffffffu && __ffs(same) - 1 == lane) atomicAdd(&hist[key], (uint32_t)__popc(same));
		}
		v = next;
	}
	__syncthreads();
	for (int i = threadIdx.x; i < 3 * 256; i += PS_THREADS)
		if (hist[i]) atomicAdd(A.out + E264_PICSTATS_HIST / 4 + i, hist[i]);
}
