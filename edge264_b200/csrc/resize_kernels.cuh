/* resize_kernels.cuh — e264_resize_kernel: the resized output of one picture (include/edge264_packed.h, layout
 * e264_packed_layout in records.h): the cropped planes of a frame slot as I420 or NV12, resampled to any size by exact
 * area averaging (spans and rounding in resize_math.cuh).
 *
 * A 256-thread block owns a tile of RS_TW x RS_TH output samples of one plane.  The source samples the tile's spans cover
 * are staged through shared memory in chunks of at most RS_RB rows x RS_CW columns, with aligned 16-byte loads, so each
 * source byte is read from memory about once (the tiles next to it read its boundary row or column again); chunking keeps
 * every ratio inside the same launch, down to a whole 16368-sample row feeding one output sample.  For each chunk:
 *   horizontal pass  a thread per (staged row, output column): the span sum restricted to the chunk, t_w times the box
 *                    sum less the cuts of the span's first and last samples when they lie in the chunk (int32: at most
 *                    255 (s_w + 2 t_w) < 2^24);
 *   vertical pass    a warp per output row, a lane per 4 output columns: the row sums of the chunk times the rows'
 *                    weights, added in 64 bits (N < 2^36).
 * Then one rounding per sample (e264_rs_round: a per-plane double reciprocal, no division) and the stores: a warp writes
 * 128 contiguous bytes of an output row, or 256 for NV12, whose Cb and Cr words are interleaved into one 8-byte store.
 * One grid covers the planes (a block belongs to one plane).  Launched by the runtime after the picture's deblocking
 * launch, and only for decoders that asked for the resized output. */
#pragma once
#include "recon_kernels.cuh"
#include "resize_math.cuh"

#define RS_THREADS 256
#define RS_TW 128                    /* output columns of a tile: 4 per lane */
#define RS_TH (RS_THREADS / 32)      /* output rows of a tile: one per warp */
#define RS_CW 512                    /* source columns of a staged chunk */
#define RS_RB 16                     /* source rows of a staged chunk */
#define RS_SROW (RS_CW + 32)         /* bytes of a staged row: the chunk and the alignment of its ends */
#define RS_VECS (RS_SROW / 16)

struct ResizePlane {
	const uint8_t *src;            /* first cropped sample of the plane in the frame slot (NV12 chroma: of Cb) */
	uint8_t *dst;
	int32_t src_stride, dst_stride;
	int32_t sw, sh, tw, th;        /* cropped size of the source plane, size of the output plane */
	int32_t bx, first;             /* tiles per tile row; the plane's first block in the grid */
	double inv;                    /* e264_rs_inv(sw * sh) */
};
struct ResizeArgs { ResizePlane p[3]; int32_t cr_off; };   /* cr_off: from a Cb sample to its Cr sample (NV12; I420 has Cr as p[2]) */

/* NC components per plane: 1, or 2 for NV12's Cb and Cr (the second at src + cr_off, interleaved in dst) */
template <int NC> __device__ __forceinline__ void resize_plane(const ResizePlane &P, int cr_off, int b, uint8_t *stage, int32_t *hsum, RsSpan *sx) {
	const int bi = b - P.first, by = bi / P.bx, bxi = bi - by * P.bx;
	const int x0 = bxi * RS_TW, y0 = by * RS_TH, lane = threadIdx.x & 31, y = y0 + (threadIdx.x >> 5);
	const int c0 = e264_rs_span(x0, P.sw, P.tw).first, c1 = e264_rs_span(min(x0 + RS_TW, P.tw) - 1, P.sw, P.tw).last + 1;
	const int r0 = e264_rs_span(y0, P.sh, P.th).first, r1 = e264_rs_span(min(y0 + RS_TH, P.th) - 1, P.sh, P.th).last + 1;
	for (int i = threadIdx.x; i < RS_TW; i += RS_THREADS) if (x0 + i < P.tw) sx[i] = e264_rs_span(x0 + i, P.sw, P.tw);
	const RsSpan sy = e264_rs_span(min(y, P.th - 1), P.sh, P.th);
	unsigned long long acc[NC][4];
#pragma unroll
	for (int c = 0; c < NC; c++)
#pragma unroll
		for (int k = 0; k < 4; k++) acc[c][k] = 0;

	for (int rr = r0; rr < r1; rr += RS_RB) {
		const int nr = min(RS_RB, r1 - rr);
		for (int cc = c0; cc < c1; cc += RS_CW) {
			const int ce = min(cc + RS_CW, c1);
			__syncthreads();   /* the previous chunk is consumed (and sx is written) */
			for (int k = threadIdx.x; k < NC * RS_RB * RS_VECS; k += RS_THREADS) {
				const int q = k / RS_VECS, v = k - q * RS_VECS, jr = q % RS_RB;
				const uint8_t *row = P.src + (q / RS_RB) * cr_off + (size_t)(rr + jr) * P.src_stride;
				const uintptr_t a = ((uintptr_t)(row + cc) & ~(uintptr_t)15) + 16 * v;
				if (jr < nr && a < (uintptr_t)(row + ce)) *(uint4 *)(stage + q * RS_SROW + 16 * v) = __ldg((const uint4 *)a);
			}
			__syncthreads();
			for (int k = threadIdx.x; k < NC * RS_RB * RS_TW; k += RS_THREADS) {
				const int q = k / RS_TW, xi = k % RS_TW, jr = q % RS_RB;
				if (jr >= nr) continue;
				int h = 0;
				if (x0 + xi < P.tw) {
					const RsSpan s = sx[xi];
					const int lo = max(s.first, cc), hi = min(s.last, ce - 1);
					if (lo <= hi) {
						const uint8_t *row = P.src + (q / RS_RB) * cr_off + (size_t)(rr + jr) * P.src_stride;
						const uint8_t *sp = stage + q * RS_SROW + (int)((uintptr_t)(row + cc) & 15) - cc;   /* sp[i]: source column i */
						int sum = 0;
						for (int i = lo; i <= hi; i++) sum += sp[i];
						h = sum * P.tw;
						if (lo == s.first) h -= s.cut_first * sp[lo];
						if (hi == s.last) h -= s.cut_last * sp[hi];
					}
				}
				hsum[q * RS_TW + xi] = h;
			}
			__syncthreads();
			const int lo = max(sy.first, rr), hi = min(sy.last, rr + nr - 1);
			for (int j = lo; j <= hi; j++) {
				const int wgt = P.th - (j == sy.first ? sy.cut_first : 0) - (j == sy.last ? sy.cut_last : 0);
#pragma unroll
				for (int c = 0; c < NC; c++) {
					const int4 hv = *(const int4 *)(hsum + (c * RS_RB + j - rr) * RS_TW + 4 * lane);
					acc[c][0] += (long long)wgt * hv.x; acc[c][1] += (long long)wgt * hv.y;
					acc[c][2] += (long long)wgt * hv.z; acc[c][3] += (long long)wgt * hv.w;
				}
			}
		}
	}

	const int x = x0 + 4 * lane;
	if (y >= P.th || x >= P.tw) return;
	const long long d = (long long)P.sw * P.sh;
	uint32_t w[NC];
#pragma unroll
	for (int c = 0; c < NC; c++)
		w[c] = (uint32_t)e264_rs_round(acc[c][0], d, P.inv) | (uint32_t)e264_rs_round(acc[c][1], d, P.inv) << 8 |
		       (uint32_t)e264_rs_round(acc[c][2], d, P.inv) << 16 | (uint32_t)e264_rs_round(acc[c][3], d, P.inv) << 24;
	uint8_t *row = P.dst + (size_t)y * P.dst_stride + NC * x;
	if (x + 4 <= P.tw) {
		if (NC == 2) *(uint2 *)row = make_uint2(__byte_perm(w[0], w[NC - 1], 0x5140), __byte_perm(w[0], w[NC - 1], 0x7362));
		else *(uint32_t *)row = w[0];
	} else {   /* the word the plane's right edge cuts */
		for (int k = 0; x + k < P.tw; k++)
#pragma unroll
			for (int c = 0; c < NC; c++) row[NC * k + c] = (uint8_t)(w[c] >> (8 * k));
	}
}

/* FMT: E264_PACKED_I420 (planes p[0..2]) or E264_PACKED_NV12 (p[0] luma, p[1] both chroma components) */
template <int FMT> __global__ void __launch_bounds__(RS_THREADS, 2) e264_resize_kernel(const __grid_constant__ ResizeArgs A) {
	constexpr int NC = FMT == E264_PACKED_NV12 ? 2 : 1;
	__shared__ __align__(16) uint8_t stage[NC * RS_RB * RS_SROW];
	__shared__ __align__(16) int32_t hsum[NC * RS_RB * RS_TW];
	__shared__ RsSpan sx[RS_TW];
	const int b = blockIdx.x;
	if (FMT == E264_PACKED_NV12 && b >= A.p[1].first) resize_plane<NC>(A.p[1], A.cr_off, b, stage, hsum, sx);
	else resize_plane<1>(A.p[b < A.p[1].first ? 0 : b < A.p[2].first ? 1 : 2], 0, b, stage, hsum, sx);
}
