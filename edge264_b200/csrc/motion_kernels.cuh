/* motion_kernels.cuh — e264_motion_kernel: the motion export of one picture (include/edge264_motion.h, layout
 * E264_MOTION_* in records.h), derived from the picture's records already resident in HBM.
 *
 * The records hold vectors per luma4x4BlkIdx (z-order inside the macroblock) and reference slots per 8x8 block; the
 * export is raster order over the picture.  A block takes a run of MOTION_RUN adjacent macroblocks of one row: their
 * records come into shared memory with 16-byte loads, then consecutive threads write consecutive words of each output
 * row (128 contiguous bytes per warp for the vectors), so the scatter out of z-order happens in shared memory and every
 * global store is coalesced.  Launched by the runtime after the picture's reconstruction launches, and only for decoders
 * that asked for the export. */
#pragma once
#include "recon_kernels.cuh"

#define MOTION_RUN 32          /* macroblocks of one row per block */
#define MOTION_THREADS 256
#define MOTION_MAX_SLOTS 32
struct MotionIds { int32_t id[MOTION_MAX_SLOTS]; };   /* FrameId of each frame slot, -1 for an empty one */

__global__ void __launch_bounds__(MOTION_THREADS) e264_motion_kernel(const E264MbRec *recs, int w_mbs, int h_mbs, MotionIds ids, uint8_t *out) {
	__shared__ uint4 rec4[MOTION_RUN * sizeof(E264MbRec) / 16];
	__shared__ int32_t sid[MOTION_MAX_SLOTS];
	const E264MbRec *r = (const E264MbRec *)rec4;
	const int runs = (w_mbs + MOTION_RUN - 1) / MOTION_RUN;
	const int mby = blockIdx.x / runs, mbx0 = (blockIdx.x - mby * runs) * MOTION_RUN, n = min(MOTION_RUN, w_mbs - mbx0);
	const size_t nmb = (size_t)w_mbs * h_mbs;
	const uint4 *src = (const uint4 *)(recs + (size_t)mby * w_mbs + mbx0);
	for (int i = threadIdx.x; i < n * (int)(sizeof(E264MbRec) / 16); i += MOTION_THREADS) rec4[i] = __ldg(src + i);
	if (threadIdx.x == 0) {
#pragma unroll
		for (int k = 0; k < MOTION_MAX_SLOTS; k++) sid[k] = ids.id[k];   /* constant indices: the table stays in the parameter bank */
	}
	__syncthreads();
	/* vectors: 8 output rows (list l, 4x4 row by), 4 n words of each from this run */
	uint32_t *mv = (uint32_t *)(out + E264_MOTION_MV * nmb);
	for (int i = threadIdx.x; i < 32 * n; i += MOTION_THREADS) {
		const int row = i / (4 * n), x4 = i - row * 4 * n, l = row >> 2, by = row & 3;
		const E264MbRec *q = r + (x4 >> 2);
		const int z = blk_z(x4 & 3, by);
		const bool used = q->kind == MBK_INTER && q->ref_idx[l][z >> 2] >= 0;
		mv[((size_t)l * 4 * h_mbs + mby * 4 + by) * (4 * w_mbs) + mbx0 * 4 + x4] = used ? *(const uint32_t *)q->mv[l][z] : 0u;
	}
	/* reference FrameIds: 4 output rows (list l, 8x8 row y8), 2 n words of each */
	int32_t *ref = (int32_t *)(out + E264_MOTION_REF * nmb);
	for (int i = threadIdx.x; i < 8 * n; i += MOTION_THREADS) {
		const int row = i / (2 * n), x8 = i - row * 2 * n, l = row >> 1, y8 = row & 1;
		const E264MbRec *q = r + (x8 >> 1);
		const int i8 = y8 * 2 + (x8 & 1), slot = q->ref_pic[l][i8];
		const bool used = q->kind == MBK_INTER && q->ref_idx[l][i8] >= 0 && (unsigned)slot < MOTION_MAX_SLOTS;
		ref[((size_t)l * 2 * h_mbs + mby * 2 + y8) * (2 * w_mbs) + mbx0 * 2 + x8] = used ? sid[slot] : -1;
	}
	/* macroblock type and QP_Y: one byte each, warp 0 and warp 1 */
	const int t = threadIdx.x & 31;
	if (threadIdx.x < 64 && t < n) {
		const E264MbRec *q = r + t;
		const size_t a = (size_t)mby * w_mbs + mbx0 + t;
		if (threadIdx.x < 32) out[E264_MOTION_TYPE * nmb + a] = q->kind == MBK_INTER && (q->flags & MBF_SKIP) ? 5 : q->kind;
		else out[E264_MOTION_QP * nmb + a] = q->qp[0];
	}
}
