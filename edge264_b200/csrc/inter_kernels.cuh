/* inter_kernels.cuh — inter macroblocks: inverse transform + motion compensation + weighting + residual in ONE kernel.
 *
 * The unit of prediction is always the 4x4 luma block and reference list (that is what the record carries a vector for —
 * partition shapes never reach the device): an ITEM.  A thread handles one item: it loads the item's 9x9 luma window and
 * two 3x3 chroma windows of the reference picture straight into registers (aligned 32-bit loads + funnel shifts; the
 * windows of neighbouring blocks overlap in L1/L2) and interpolates 4x4 + 2x2 + 2x2 samples with the register arithmetic of
 * mc_math.cuh (dp4a tap sums).  Items are binned by interpolation class so that a warp runs ONE class body on 32 items
 * (reference edge264_inter.c:416-1251: per-partition SIMD interpolation + five weighting schemes).
 * The macroblock's coefficient run (16..816 bytes) arrives by cp.async.bulk on an mbarrier one macroblock ahead and is
 * inverse-transformed in shared memory (residual_stage), so the residual never travels through global memory.
 * It replaces an earlier kernel that regrouped rectangles on the device, fetched windows by cp.async.bulk.tensor into shared
 * memory and produced one output sample per lane and loop iteration. */
#pragma once
#include "recon_kernels.cuh"
#include "deblock_kernels.cuh"

__device__ __forceinline__ uint32_t ldg32(const uint8_t *p) { return __ldg((const uint32_t *)p); }

/* the thread's 9x9 luma window at (X0, Y0) = top-left of the window (block position + integer vector - 2) */
__device__ __forceinline__ void mc_load_luma(const uint8_t *ref, int stride, int W, int H, int X0, int Y0, uint32_t w[9][3]) {
	if (X0 >= 0 && X0 + 9 <= W) {
		const int al = X0 & ~3, sh = (X0 & 3) * 8;
#pragma unroll
		for (int r = 0; r < 9; r++) {
			const int yy = min(max(Y0 + r, 0), H - 1);
			const uint8_t *p = ref + (size_t)yy * stride + al;
			const uint32_t a0 = ldg32(p), a1 = ldg32(p + 4), a2 = ldg32(p + 8);
			w[r][0] = __funnelshift_r(a0, a1, sh); w[r][1] = __funnelshift_r(a1, a2, sh); w[r][2] = a2 >> sh;
		}
	} else {   /* the window reaches over the left or right picture edge: samples are replicated (8.4.2.2.1) */
#pragma unroll
		for (int r = 0; r < 9; r++) {
			const int yy = min(max(Y0 + r, 0), H - 1);
			const uint8_t *p = ref + (size_t)yy * stride;
			uint32_t v[3] = {0, 0, 0};
#pragma unroll
			for (int k = 0; k < 9; k++) v[k >> 2] |= (uint32_t)__ldg(p + min(max(X0 + k, 0), W - 1)) << (8 * (k & 3));
			w[r][0] = v[0]; w[r][1] = v[1]; w[r][2] = v[2];
		}
	}
}
/* the thread's 3x3 window of one chroma plane (rows alternate Cb | Cr inside stride_c; `plane` points at the plane's column 0) */
__device__ __forceinline__ void mc_load_chroma(const uint8_t *plane, int stride, int Wc, int Hc, int X0, int Y0, uint32_t c[3]) {
	if (X0 >= 0 && X0 + 3 <= Wc) {
		const int al = X0 & ~3, sh = (X0 & 3) * 8;
#pragma unroll
		for (int r = 0; r < 3; r++) {
			const uint8_t *p = plane + (size_t)min(max(Y0 + r, 0), Hc - 1) * stride + al;
			c[r] = __funnelshift_r(ldg32(p), ldg32(p + 4), sh);
		}
	} else {
#pragma unroll
		for (int r = 0; r < 3; r++) {
			const uint8_t *p = plane + (size_t)min(max(Y0 + r, 0), Hc - 1) * stride;
			c[r] = (uint32_t)__ldg(p + min(max(X0, 0), Wc - 1)) | (uint32_t)__ldg(p + min(max(X0 + 1, 0), Wc - 1)) << 8 | (uint32_t)__ldg(p + min(max(X0 + 2, 0), Wc - 1)) << 16;
		}
	}
}

/* ---- the kernel ----
 * A block takes chunks of INTER_CHUNK consecutive macroblocks.  Per chunk:
 *   1. records into shared memory; every (macroblock, list, 4x4 block) that is predicted becomes an ITEM and is queued by
 *      interpolation class (mc_class: full, horizontal, vertical, diagonal, centre h-first, centre v-first) — warp
 *      votes give the queue positions;
 *   2. the warps take 32 items of ONE class at a time: the same instruction stream for all lanes, every lane busy —
 *      window loads, interpolation, predictions (24 bytes) into shared memory;
 *   3. a warp per macroblock: inverse transform of its coefficient run (cp.async.bulk one macroblock ahead), list-0 /
 *      list-1 combination with the slice's weighting, residual, 128-bit row stores.
 * A thread-per-block version without the binning ran every class present in a macroblock one after the other (about
 * 2000 warp instructions per macroblock on random vectors, no faster than round 1's). */
/* Block geometry: INTER_WARPS warps take INTER_CHUNK macroblocks at a time (4 per warp).  The kernel's three phases are
 * separated by block barriers, so all warps of a block execute the same part of the code: the bigger the block, the fewer
 * different parts of the kernel (5 700 instructions on sm_90a) the SM's instruction cache has to hold at a time — and a
 * 16-warp block at 128 registers per thread fills the SM's register file, so no block of another kernel shares the SM. */
#ifndef INTER_WARPS
#define INTER_WARPS 16      /* H100 (results/h100_geometry.txt), 1080p replay of 32 streams: 4 warps 13.1 k, 8 warps 16.4 k, 16 warps 19.6 k frames/s */
#endif
#ifndef INTER_CHUNK
#define INTER_CHUNK (4 * INTER_WARPS)
#endif
#define INTER_MINB0 (16 / INTER_WARPS)      /* blocks per SM at 128 registers per thread */
struct __align__(16) InterSmem {
	uint4 rec4[INTER_CHUNK][12];
	uint32_t pred[INTER_CHUNK][2][16][8];          /* [macroblock][list][luma4x4BlkIdx]: four luma rows, 2x2 Cb, 2x2 Cr, (pad: 16-byte aligned entries) */
	uint16_t queue[6][INTER_CHUNK * 32];           /* item = macroblock << 5 | list << 4 | luma4x4BlkIdx */
	int qn[6];
	WarpSmem ws[INTER_WARPS];
	uint4 trec4[INTER_CHUNK][12];                  /* deblocking digests: the records of the row above the chunk's macroblocks */
	uint4 lrec4[12];                               /* and the record left of its first macroblock */
	E264DbkMb ddg[INTER_WARPS];
	int16_t coef[INTER_WARPS][2][RES_COEF_MAX];
	unsigned long long bars[INTER_WARPS][2];
};

/* One item: the window loads are the same for every interpolation class and exist ONCE in the kernel (the six class bodies
 * used to carry their own copies: 3 000 of the kernel's 12 000 instructions, and with blocks of several pictures in
 * different phases on an SM the instruction cache, 32 KB in its first shared level, is what the warps wait for);
 * `cls` is uniform over the warp, so the switch is one resolved branch per pass. */
template <bool LUMA>   /* luma-only pictures: no chroma windows, no chroma predictions */
__device__ __forceinline__ void inter_item(const PicJob &J, InterSmem &sm, int cls, int item, int mb0, int W, int H) {
	const int m = item >> 5, l = (item >> 4) & 1, z = item & 15, bx = blk_x(z), by = blk_y(z);
	const E264MbRec *r = (const E264MbRec *)sm.rec4[m];
	const int mb = mb0 + m, mbx = mb % J.w_mbs, mby = mb / J.w_mbs;
	int slot = r->ref_pic[l][z >> 2];
	if (slot < 0 || slot >= J.n_slots) slot = J.dst_slot;
	const uint8_t *ref = J.frames + (size_t)slot * J.frame_bytes;
	const int mvx = r->mv[l][z][0], mvy = r->mv[l][z][1];
	const int fx = mvx & 3, fy = mvy & 3;
	uint32_t win[9][3], py[4];
	mc_load_luma(ref, J.stride_y, W, H, mbx * 16 + bx * 4 + (mvx >> 2) - 2, mby * 16 + by * 4 + (mvy >> 2) - 2, win);
	uint32_t cb[3], cr[3];
	if (!LUMA) {
		const uint8_t *cplane = ref + J.plane_y;
		const int cx = mbx * 8 + bx * 2 + (mvx >> 3), cy = mby * 8 + by * 2 + (mvy >> 3);
		mc_load_chroma(cplane, J.stride_c, W >> 1, H >> 1, cx, cy, cb);
		mc_load_chroma(cplane + (J.stride_c >> 1), J.stride_c, W >> 1, H >> 1, cx, cy, cr);
	}
	switch (cls) {
	case 0:
#pragma unroll
		for (int y = 0; y < 4; y++) py[y] = mc_fsr(win[y + 2][0], win[y + 2][1], 16);
		break;
	case 1: mc_luma_h(win, fx, py); break;
	case 2: mc_luma_v(win, fy, py); break;
	case 3: mc_luma_diag(win, fx, fy, py); break;
	case 4: mc_luma_center(win, fy, py); break;
	default: mc_luma_center_v(win, fx, py); break;
	}
	uint32_t *o = sm.pred[m][l][z];
	*(uint4 *)o = make_uint4(py[0], py[1], py[2], py[3]);
	if (!LUMA) *(uint2 *)(o + 4) = make_uint2(mc_chroma2x2(cb[0], cb[1], cb[2], mvx & 7, mvy & 7), mc_chroma2x2(cr[0], cr[1], cr[2], mvx & 7, mvy & 7));
}

/* LUMA: luma-only pictures (PicDesc.luma_only), which neither read nor write a chroma sample */
template <int MINB, bool LUMA>
__global__ void __launch_bounds__(INTER_WARPS * 32, MINB) e264_inter4_kernel(PicJob J) {
	TraceScope trace_(J, 1);
	reset_next_tickets(J);
	extern __shared__ __align__(16) unsigned char inter_smem_raw[];
	InterSmem &sm = *(InterSmem *)inter_smem_raw;
	const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
	WarpSmem *ws = &sm.ws[w];
	const int nmb = J.w_mbs * J.h_mbs;
	const int W = J.w_mbs * 16, H = J.h_mbs * 16;
	if (lane == 0) mbar_setup(sm.bars[w], 2);
	unsigned parity[2] = {0, 0};
	PT_DECL
	const int nchunks = (nmb + INTER_CHUNK - 1) / INTER_CHUNK;
	for (int chunk = blockIdx.x; chunk < nchunks; chunk += gridDim.x) {
		const int mb0 = chunk * INTER_CHUNK, cnt = min(INTER_CHUNK, nmb - mb0);
		__syncthreads();                               /* the previous chunk's predictions and records are no longer read */
		PT_MARK(2)      /* block barriers */
		/* ---- 1. records, queues ---- */
		for (int i = tid; i < cnt * 12; i += INTER_WARPS * 32) sm.rec4[i / 12][i % 12] = __ldg((const uint4 *)(J.recs + mb0) + i);
		if (J.dbk != nullptr) {      /* the neighbour records the digests read, loaded with the chunk's own (the top edge row has none) */
			for (int i = tid; i < cnt * 12; i += INTER_WARPS * 32) if (mb0 + i / 12 >= J.w_mbs) sm.trec4[i / 12][i % 12] = __ldg((const uint4 *)(J.recs + mb0 - J.w_mbs) + i);
			if (tid < 12 && mb0 > 0) sm.lrec4[tid] = __ldg((const uint4 *)(J.recs + mb0 - 1) + tid);
		}
		if (tid < 6) sm.qn[tid] = 0;
		PT_MARK(0)      /* records and queues */
		__syncthreads();
		PT_MARK(2)
		/* the macroblocks this warp finishes in step 3 are w, w + INTER_WARPS, ...: get the first coefficient run under way */
		auto coef_issue = [&](int m, int b) -> int {     /* 0 not inter, 1 inter, 2 inter with coefficients (copy in flight) */
			if (m >= cnt) return 0;
			const E264MbRec *r = (const E264MbRec *)sm.rec4[m];
			if (r->kind != MBK_INTER) return 0;
			if (r->coded == 0) return 1;
			coef_request(J, r, sm.coef[w][b], &sm.bars[w][b], lane);
			return 2;
		};
		int what = coef_issue(w, 0);
#pragma unroll 1
		for (int i0 = 0; i0 < cnt * 32; i0 += INTER_WARPS * 32) {
			const int item = i0 + tid, m = item >> 5, l = (item >> 4) & 1, z = item & 15;
			int cls = -1;
			if (m < cnt) {
				const E264MbRec *r = (const E264MbRec *)sm.rec4[m];
				if (r->kind == MBK_INTER && r->ref_idx[l][z >> 2] >= 0) cls = mc_class(r->mv[l][z][0] & 3, r->mv[l][z][1] & 3);
			}
			/* queue position: the lanes of one class find each other with one match instruction, their first lane reserves the
			 * run in the class queue */
			const unsigned peers = __match_any_sync(0xffffffffu, cls);
			const int leader = __ffs(peers) - 1;
			int base = 0;
			if (cls >= 0 && lane == leader) base = atomicAdd(&sm.qn[cls], __popc(peers));
			base = __shfl_sync(0xffffffffu, base, leader);
			if (cls >= 0) sm.queue[cls][base + __popc(peers & ((1u << lane) - 1))] = (uint16_t)item;
		}
		PT_MARK(0)
		__syncthreads();
		PT_MARK(2)
		/* ---- 2. one class at a time, 32 items per warp pass: the groups of all classes form one list ---- */
		{
			int total = 0;
#pragma unroll
			for (int j = 0; j < 6; j++) total += (sm.qn[j] + 31) >> 5;
#pragma unroll 1
			for (int g = w; g < total; g += INTER_WARPS) {
				int c = 0, gb = 0, acc = 0;
#pragma unroll
				for (int j = 0; j < 6; j++) { const int gj = (sm.qn[j] + 31) >> 5; if (g >= acc) { c = j; gb = acc; } acc += gj; }
				const int k = (g - gb) * 32 + lane;
				if (k < sm.qn[c]) inter_item<LUMA>(J, sm, c, sm.queue[c][k], mb0, W, H);
			}
		}
		PT_MARK(1)      /* prediction passes */
		__syncthreads();
		PT_MARK(2)
		/* ---- 3. a warp per macroblock: inverse transform, weighting, residual, store ---- */
		int b = 0;
		bool failed = false;
#pragma unroll 1
		for (int m = w; m < cnt; m += INTER_WARPS, b ^= 1) {
			const int what2 = coef_issue(m + INTER_WARPS, b ^ 1);
			/* the macroblock's deblocking digest (every macroblock, intra ones too), from the records in shared memory, while
			 * the coefficient run requested above is in flight */
			if (J.dbk != nullptr)
				dbk_digest_mb<LUMA>(J, (const E264MbRec *)sm.rec4[m], (const E264MbRec *)(m > 0 ? sm.rec4[m - 1] : sm.lrec4), (const E264MbRec *)sm.trec4[m], &sm.ddg[w], mb0 + m, lane);
			PT_MARK(3)          /* deblocking digest */
			if (what) {
				const int mb = mb0 + m, mbx = mb % J.w_mbs, mby = mb / J.w_mbs;
				const E264MbRec *r = (const E264MbRec *)sm.rec4[m];
				const E264SliceRec *sr = J.slices + r->slice_idx;
				if (what == 2) {
					if (!mbar_wait(&sm.bars[w][b], parity[b])) { if (lane == 0) atomicExch(J.err, 4u); failed = true; }
					parity[b] ^= 1;
					PT_MARK(4)  /* waiting for the coefficient run */
					if (!failed) residual_stage<LUMA>(ws, r, sr, sm.coef[w][b], lane);
					PT_MARK(5)  /* dequantisation and inverse transforms */
				}
				if (!failed) {
					/* two lanes per 4x4 block: lane z + 16 h takes luma rows 2 h and 2 h + 1 of block z and its 2x2 samples of
					 * chroma plane h (Cb, Cr) */
					const int z = lane & 15, h = lane >> 4, bx = blk_x(z), by = blk_y(z), i8 = z >> 2;
					const int r0 = r->ref_idx[0][i8], r1 = r->ref_idx[1][i8];
					uint32_t py[2] = {0, 0}, pc = 0, qy[2] = {0, 0}, qc = 0;
					if (r0 >= 0) { const uint2 a = *(const uint2 *)(sm.pred[m][0][z] + 2 * h); py[0] = a.x; py[1] = a.y; if (!LUMA) pc = sm.pred[m][0][z][4 + h]; }
					if (r1 >= 0) { const uint2 a = *(const uint2 *)(sm.pred[m][1][z] + 2 * h); qy[0] = a.x; qy[1] = a.y; if (!LUMA) qc = sm.pred[m][1][z][4 + h]; }
					const int wpm = sr->wp_mode;
					const bool bi = r0 >= 0 && r1 >= 0;
					if (!bi && r0 < 0) { py[0] = qy[0]; py[1] = qy[1]; pc = qc; }
					if (bi && wpm == WP_DEFAULT) {
						py[0] = mc_avg4(py[0], qy[0]); py[1] = mc_avg4(py[1], qy[1]); if (!LUMA) pc = mc_avg4(pc, qc);
					} else if ((bi && wpm != WP_DEFAULT) || (wpm == WP_EXPLICIT && (r0 >= 0 || r1 >= 0))) {
						/* one weighting body for every scheme: parameters of luma and of this lane's chroma plane, then three words */
						int wa[2], wb[2], o[2], sh[2], rnd[2];
						const int ll = r0 >= 0 ? 0 : 1, ri = (ll ? r1 : r0) & 15;
#pragma unroll
						for (int k = 0; k < (LUMA ? 1 : 2); k++) {
							const int c = k ? 1 + h : 0, lw = k ? sr->chroma_log2_wd : sr->luma_log2_wd;
							if (bi && wpm == WP_EXPLICIT) { wa[k] = sr->wp_w[0][r0 & 15][c]; wb[k] = sr->wp_w[1][r1 & 15][c]; o[k] = 0; sh[k] = lw + 1; rnd[k] = ((sr->wp_o[0][r0 & 15][c] + sr->wp_o[1][r1 & 15][c] + 1) | 1) * (1 << lw); }
							else if (bi) { wb[k] = sr->implicit_w1[r0 & 15][r1 & 15]; wa[k] = 64 - wb[k]; o[k] = 0; sh[k] = 6; rnd[k] = 32; }
							else { wa[k] = sr->wp_w[ll][ri][c]; wb[k] = 0; o[k] = sr->wp_o[ll][ri][c]; sh[k] = lw; rnd[k] = lw >= 1 ? 1 << (lw - 1) : 0; }
						}
						py[0] = wp_word(py[0], qy[0], wa[0], wb[0], rnd[0], sh[0], o[0]); py[1] = wp_word(py[1], qy[1], wa[0], wb[0], rnd[0], sh[0], o[0]);
						if (!LUMA) pc = wp_word(pc, qc, wa[1], wb[1], rnd[1], sh[1], o[1]);
					}
					if (what == 2) {
						const int16_t *ry = ws->res + (by * 4 + 2 * h) * 16 + bx * 4, *rc = ws->res + 256 + h * 64 + (by * 2) * 8 + bx * 2;
						const uint2 res0 = *(const uint2 *)ry, res1 = *(const uint2 *)(ry + 16);
						py[0] = mc_add_res4(py[0], res0.x, res0.y); py[1] = mc_add_res4(py[1], res1.x, res1.y);
						if (!LUMA) pc = mc_add_res4(pc, *(const uint32_t *)rc, *(const uint32_t *)(rc + 8));
					}
					*(uint32_t *)&YT(bx * 4, by * 4 + 2 * h) = py[0]; *(uint32_t *)&YT(bx * 4, by * 4 + 2 * h + 1) = py[1];
					if (!LUMA) { *(uint16_t *)&CT(h, bx * 2, by * 2) = (uint16_t)pc; *(uint16_t *)&CT(h, bx * 2, by * 2 + 1) = (uint16_t)(pc >> 16); }
				}
				__syncwarp();
				if (!failed) {
					uint8_t *Y, *C; mb_planes(J, mbx, mby, Y, C);
					store_mb<LUMA>(ws, J, Y, C, lane);
					if (lane == 0) J.flags[mb] = J.epoch;     /* visible to the intra kernel through the kernel boundary */
				}
				__syncwarp();
			}
			PT_MARK(6)      /* combination, residual, stores */
			what = what2;
		}
	}
	PT_FLUSH(16)
}

/* ---- error map of the inter macroblocks (pictures with err_pic only) ----
 * A warp per macroblock, lanes over (list, 4x4 block): the largest byte of the reference macroblocks the block's luma
 * window touches, then the record's own err.  Launched behind e264_inter4_kernel and before the intra kernels, which read
 * the bytes of inter neighbours.  A kernel of its own: each way of folding this into e264_inter4_kernel (in its step 1, 2
 * or 3, inlined or as a call) made ptxas spill there, at the 128 registers its 16-warp blocks allow, and clean pictures
 * would pay for that; here they pay nothing, the launch does not happen. */
#define MAP_WARPS 8
__global__ void __launch_bounds__(MAP_WARPS * 32) e264_inter_map_kernel(PicJob J) {
	const int lane = threadIdx.x & 31, nmb = J.w_mbs * J.h_mbs;
	uint8_t *dst = map_of(J, J.dst_slot);
	for (int mb = blockIdx.x * MAP_WARPS + (threadIdx.x >> 5); mb < nmb; mb += gridDim.x * MAP_WARPS) {
		const E264MbRec *r = J.recs + mb;
		if (r->kind != MBK_INTER) continue;
		const unsigned e = __reduce_max_sync(0xffffffffu, map_inter_block(J.maps, J.taint, J.n_slots, J.w_mbs, J.h_mbs, r, lane >> 4, lane & 15, mb % J.w_mbs, mb / J.w_mbs));
		if (lane == 0) dst[mb] = (uint8_t)max(e, (unsigned)r->err);
	}
}
