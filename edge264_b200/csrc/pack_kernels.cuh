/* pack_kernels.cuh — e264_pack_kernel: the packed output of one picture (include/edge264_packed.h, layout
 * e264_packed_layout in records.h): the cropped planes of a frame slot as I420 or NV12, box-downscaled by N = 1 << K.
 *
 * A thread makes one 32-bit word of one output row: 4 output samples, from an N-row by 4N-byte window of the source.
 * The left cropping offset makes source rows unaligned, by the same amount in every row of a plane (strides are multiples
 * of 16), so a row is read as N + 1 aligned words and brought into place with funnel shifts.  Sums stay packed: N = 2 adds
 * pairs in two 16-bit lanes per word, N = 4 and 8 add the four bytes of a word with dp4a; one rounding at the end.  A warp
 * writes 32 consecutive words of an output row.  For NV12 a thread makes the Cb and the Cr word of the same place and
 * stores them interleaved as 8 bytes.  One grid covers the planes (a block belongs to one plane); only the blocks on the
 * right and bottom borders of a plane clamp rows and take the bytewise path for a word the picture's edge cuts.
 * Launched by the runtime after the picture's deblocking launch, and only for decoders that asked for the output. */
#pragma once
#include "recon_kernels.cuh"

#define PACK_THREADS 256
#define PACK_ROWS (PACK_THREADS / 32)   /* output rows of a block: a warp per row, 32 words wide */

struct PackPlane {
	const uint8_t *src;            /* first cropped sample of the plane in the frame slot (NV12 chroma: of Cb) */
	uint8_t *dst;
	int32_t src_stride, dst_stride;
	int32_t w, h;                  /* cropped size of the source plane */
	int32_t bx, first;             /* blocks per block row; the plane's first block in the grid */
};
struct PackArgs { PackPlane p[3]; int32_t cr_off; };   /* cr_off: from a Cb sample to its Cr sample (NV12; I420 has Cr as p[2]) */

/* output samples 4 xw .. 4 xw + 3 of output row yo, as one word */
template <int K, bool EDGE> __device__ __forceinline__ uint32_t pack_word(const uint8_t *src, int stride, int w, int h, int xw, int yo) {
	constexpr int N = 1 << K;
	const int sx = xw * 4 * N;
	if (EDGE && sx + 4 * N > w) {   /* the word the right border cuts: replicate the last column */
		uint32_t out = 0;
#pragma unroll
		for (int j = 0; j < 4; j++) {
			uint32_t s = 0;
			for (int dy = 0; dy < N; dy++) {
				const uint8_t *row = src + (size_t)min(yo * N + dy, h - 1) * stride;
				for (int dx = 0; dx < N; dx++) s += row[min(sx + j * N + dx, w - 1)];
			}
			out |= ((s + (N * N >> 1)) >> (2 * K)) << (8 * j);
		}
		return out;
	}
	const uintptr_t a = (uintptr_t)src + sx;
	const unsigned mis = (unsigned)(a & 3), sh = mis * 8;
	uint32_t acc[4] = {0, 0, 0, 0};
#pragma unroll
	for (int dy = 0; dy < N; dy++) {
		int sy = yo * N + dy;
		if (EDGE) sy = min(sy, h - 1);
		const uint32_t *p = (const uint32_t *)(a - mis + (size_t)sy * stride);
		uint32_t v[N + 1];
#pragma unroll
		for (int i = 0; i < N; i++) v[i] = __ldg(p + i);
		v[N] = mis ? __ldg(p + N) : 0u;   /* an aligned row needs no word beyond its last sample */
#pragma unroll
		for (int i = 0; i < N; i++) {
			const uint32_t x = __funnelshift_r(v[i], v[i + 1], sh);
			if (K == 0) acc[0] = x;
			else if (K == 1) acc[i] += (x & 0x00ff00ffu) + ((x >> 8) & 0x00ff00ffu);
			else acc[i * 4 / N] = __dp4a(x, 0x01010101u, acc[i * 4 / N]);
		}
	}
	if (K == 0) return acc[0];
	if (K == 1) return __byte_perm(((acc[0] + 0x00020002u) >> 2) & 0x00ff00ffu, ((acc[1] + 0x00020002u) >> 2) & 0x00ff00ffu, 0x6420);
	constexpr uint32_t R = N * N >> 1;
	return ((acc[0] + R) >> (2 * K)) | ((acc[1] + R) >> (2 * K)) << 8 | ((acc[2] + R) >> (2 * K)) << 16 | ((acc[3] + R) >> (2 * K)) << 24;
}

template <int K, bool NV12_CHROMA, bool EDGE> __device__ __forceinline__ void pack_store(const PackPlane &P, int cr_off, int xw, int yo) {
	const uint32_t a = pack_word<K, EDGE>(P.src, P.src_stride, P.w, P.h, xw, yo);
	uint8_t *row = P.dst + (size_t)yo * P.dst_stride;
	if (NV12_CHROMA) {
		const uint32_t b = pack_word<K, EDGE>(P.src + cr_off, P.src_stride, P.w, P.h, xw, yo);
		*(uint2 *)(row + xw * 8) = make_uint2(__byte_perm(a, b, 0x5140), __byte_perm(a, b, 0x7362));
	} else {
		*(uint32_t *)(row + xw * 4) = a;
	}
}

template <int K, bool NV12_CHROMA> __device__ __forceinline__ void pack_plane(const PackPlane &P, int cr_off, int b) {
	constexpr int N = 1 << K;
	const int bi = b - P.first, by = bi / P.bx, bxi = bi - by * P.bx;
	const int xw = bxi * 32 + (threadIdx.x & 31), yo = by * PACK_ROWS + (threadIdx.x >> 5);
	if ((bxi + 1) * 128 * N > P.w || (by + 1) * PACK_ROWS * N > P.h) {   /* the block touches the right or the bottom border */
		if (xw * 4 * N < P.w && yo * N < P.h) pack_store<K, NV12_CHROMA, true>(P, cr_off, xw, yo);
	} else {
		pack_store<K, NV12_CHROMA, false>(P, cr_off, xw, yo);
	}
}

/* FMT: E264_PACKED_I420 (planes p[0..2]) or E264_PACKED_NV12 (p[0] luma, p[1] both chroma components) */
template <int K, int FMT> __global__ void __launch_bounds__(PACK_THREADS) e264_pack_kernel(const __grid_constant__ PackArgs A) {
	const int b = blockIdx.x;
	if (b < A.p[1].first) pack_plane<K, false>(A.p[0], 0, b);
	else if (FMT == E264_PACKED_NV12) pack_plane<K, true>(A.p[1], A.cr_off, b);
	else if (b < A.p[2].first) pack_plane<K, false>(A.p[1], 0, b);
	else pack_plane<K, false>(A.p[2], 0, b);
}
