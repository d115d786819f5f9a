/* intra_kernels.cuh — intra pictures (and any picture with more intra than inter macroblocks): the reconstruction
 * wavefront as BANDS of rows.
 *
 * Intra prediction of macroblock (x, y) reads the unfiltered samples of its neighbours A (x-1, y), D, B, C (x-1..x+1, y-1)
 * (reference: decode order edge264_slice.c:1651-1849 with the predictors of edge264_intra.c:291-765): rows can run in
 * parallel two macroblocks apart.  Round 1 ran one warp per row with a global flag, a gpu-scope fence (which also
 * invalidates L1) and reloads of the record, the residual and the row above from L2 inside every step.  Here a block owns IR_ROWS consecutive rows (two warps each: one
 * inverse-transforms up to IR_SLOTS - 1 macroblocks ahead, one predicts); the bottom
 * sample row of every finished macroblock goes to the row below through a shared-memory ring with done/taken counters
 * (block-scope fences); records arrive four macroblocks ahead, coefficient runs three ahead (cp.async.bulk on an mbarrier)
 * and are inverse-transformed BEFORE the row waits for its neighbours, so a step is the prediction itself plus a
 * shared-memory hand-shake and the residual never travels through global memory.  Only the band's last row talks to the next block through global memory, with
 * a progress counter published every IR_CHUNK macroblocks.  Inter macroblocks inside such a picture were reconstructed
 * by the inter kernel before: their row warp only forwards their border samples. */
#pragma once
#include "recon_kernels.cuh"
#include "deblock_kernels.cuh"

#define IR_ROWS 8
#define IR_RING 16
#define IR_CHUNK 8
#define IR_SLOTS 4      /* macroblocks the transform warp may be ahead of the prediction warp (residual / tile slots, coefficient buffers) */
#define IR_RECS 8       /* record ring of a row */
struct __align__(16) IntraRowsSmem {
	WarpSmem ws[IR_ROWS][IR_SLOTS];                    /* macroblock x of every row in slot x % IR_SLOTS: residual from the row's transform warp, tile of its prediction warp */
	uint4 recs[IR_ROWS][IR_RECS][12];           /* records of macroblocks x-4 .. x+3 of every row */
	uint32_t ring[IR_ROWS][IR_RING][8];         /* bottom sample row of a finished macroblock: luma (4 words), Cb (2), Cr (2) */
	uint8_t ering[IR_ROWS][IR_RING];            /* and its error map byte (pictures with err_pic) */
	int16_t coef[IR_ROWS][IR_SLOTS][RES_COEF_MAX];   /* coefficient runs of macroblocks x .. x+3 of every row (cp.async.bulk) */
	unsigned long long bars[IR_ROWS][IR_SLOTS];
	uint4 drecs[IR_ROWS][12];                   /* deblocking digests of intra-only pictures: the top neighbour's record */
	E264DbkMb ddg[IR_ROWS];
	int done[IR_ROWS];                          /* macroblocks a row has put into its ring */
	int taken[IR_ROWS];                         /* the macroblock a row is working on: ring entries before it (minus one) are free */
	int ready[IR_ROWS];                         /* macroblocks whose residual (and record) the transform warp has delivered */
	int used[IR_ROWS];                          /* macroblocks the prediction warp is through with */
	int band;
};

/* The row's TRANSFORM warp: records four ahead (through a register, so the warp never waits for the load it has just
 * issued), coefficient runs three ahead (cp.async.bulk; DRAM latency is longer than one macroblock of this warp's work),
 * dequantisation and inverse transforms into the residual of slot x % IR_SLOTS, at most IR_SLOTS - 1 macroblocks ahead of
 * the prediction warp.  In a picture without inter macroblocks it also derives the row's deblocking digests (no inter
 * kernel runs that would). */
template <bool LUMA>
__device__ __forceinline__ void intra_row_transform(const PicJob &J, IntraRowsSmem &sm, int band, int w, int lane, unsigned &parbits) {
	const int W = J.w_mbs, H = J.h_mbs, nmb = W * H;
	const int mby = band * IR_ROWS + w;
	if (mby >= H) return;
	const E264MbRec *rowrecs = J.recs + (size_t)mby * W;
	const volatile unsigned *errp = J.err;
	volatile int *used = sm.used + w, *ready = sm.ready + w;
	const bool digests = J.dbk != nullptr && J.n_intra == nmb;
	constexpr int AHEAD = IR_SLOTS - 1;          /* coefficient runs in flight ahead of the macroblock being transformed */
	/* prologue: records 0 .. AHEAD in shared memory, record AHEAD + 1 in the register */
	for (int x = 0; x <= AHEAD && x < W; x++) if (lane < 12) sm.recs[w][x % IR_RECS][lane] = __ldg((const uint4 *)(rowrecs + x) + lane);
	uint4 recreg = make_uint4(0, 0, 0, 0);
	if (AHEAD + 1 < W && lane < 12) recreg = __ldg((const uint4 *)(rowrecs + AHEAD + 1) + lane);
	__syncwarp();
	auto coef_issue = [&](int x) -> bool {       /* true: a copy is in flight into buffer x % IR_SLOTS */
		const E264MbRec *rr = (const E264MbRec *)sm.recs[w][x % IR_RECS];
		if (rr->kind == MBK_INTER || rr->kind == MBK_IPCM || rr->coded == 0) return false;
		coef_request(J, rr, sm.coef[w][x % IR_SLOTS], &sm.bars[w][x % IR_SLOTS], lane);
		return true;
	};
	unsigned pending = 0;                        /* bit x % IR_SLOTS: macroblock x has a copy in flight */
	uint4 topreg = make_uint4(0, 0, 0, 0);       /* digests: the top neighbour's record, one macroblock ahead */
	if (digests && mby > 0 && lane < 12) topreg = __ldg((const uint4 *)(rowrecs - W) + lane);
	PT_DECL
	for (int x = 0; x < AHEAD && x < W; x++) if (coef_issue(x)) pending |= 1u << (x % IR_SLOTS);
#pragma unroll 1
	for (int mbx = 0; mbx < W; mbx++) {
		const int sl = mbx % IR_SLOTS;
		/* residual slot sl is free once the prediction warp is through with macroblock mbx - IR_SLOTS; the record slot written
		 * below belonged to macroblock mbx + AHEAD + 1 - IR_RECS, older still */
		if (lane == 0) {
			unsigned spins = 0; bool bad = false;
			wait_smem_ge(used, mbx - IR_SLOTS + 1, errp, spins, bad);
			if (bad) atomicExch(J.err, 1u);
			__threadfence_block();
		}
		__syncwarp();
		PT_MARK(0)      /* waiting for a free slot */
		const E264MbRec *r = (const E264MbRec *)sm.recs[w][mbx % IR_RECS];
		WarpSmem *ws = &sm.ws[w][sl];
		/* the record fetched one iteration ago goes to shared memory, the next one is requested */
		if (mbx + AHEAD + 1 < W && lane < 12) sm.recs[w][(mbx + AHEAD + 1) % IR_RECS][lane] = recreg;
		if (mbx + AHEAD + 2 < W && lane < 12) recreg = __ldg((const uint4 *)(rowrecs + mbx + AHEAD + 2) + lane);
		__syncwarp();
		if (mbx + AHEAD < W) { const int nb = (mbx + AHEAD) % IR_SLOTS; pending &= ~(1u << nb); if (coef_issue(mbx + AHEAD)) pending |= 1u << nb; }
		const int kind = r->kind;
		PT_MARK(1)      /* records, coefficient copy issued */
		if ((pending >> sl) & 1) {
			if (!mbar_wait(&sm.bars[w][sl], (parbits >> sl) & 1)) { if (lane == 0) atomicExch(J.err, 3u); }
			parbits ^= 1u << sl;
			PT_MARK(2)  /* waiting for the coefficient run */
			residual_stage<LUMA>(ws, r, J.slices + r->slice_idx, sm.coef[w][sl], lane);
		} else if (kind != MBK_INTER && kind != MBK_IPCM) clear_residual(ws, lane);
		__syncwarp();
		if (lane == 0) { __threadfence_block(); *ready = mbx + 1; }
		PT_MARK(3)      /* inverse transforms */
		if (digests) {      /* the macroblock's record and the left one are in the record ring */
			if (lane < 12) sm.drecs[w][lane] = topreg;
			if (mby > 0 && mbx + 1 < W && lane < 12) topreg = __ldg((const uint4 *)(rowrecs - W + mbx + 1) + lane);
			__syncwarp();
			dbk_digest_mb<LUMA>(J, r, (const E264MbRec *)sm.recs[w][(mbx + IR_RECS - 1) % IR_RECS], (const E264MbRec *)sm.drecs[w], &sm.ddg[w], mby * W + mbx, lane);
		}
		PT_MARK(4)      /* deblocking digest */
	}
	PT_FLUSH(0)
}

/* The row's PREDICTION warp: waits for the residual, for the row above (top-right neighbour finished) and for room in
 * its ring, predicts into the tile of slot x % IR_SLOTS, stores, hands the bottom sample row down.  LUMA: luma-only
 * pictures, no chroma sample is read, predicted, stored or handed over. */
template <bool MAPS, bool LUMA>
__device__ __forceinline__ void intra_row_walk(const PicJob &J, IntraRowsSmem &sm, int band, int w, int lane) {
	const int W = J.w_mbs, H = J.h_mbs;
	const int lrow = w, mby = band * IR_ROWS + w;
	if (mby >= H) return;
	const bool from_global = lrow == 0 && mby > 0;
	const bool from_ring = lrow > 0;
	const bool to_ring = lrow + 1 < IR_ROWS && mby + 1 < H;
	const bool to_global = lrow + 1 == IR_ROWS && mby + 1 < H;
	volatile unsigned *prog = row_progress(J, PROG_INTRA);
	const volatile unsigned *errp = J.err;
	const unsigned base = prog_base(J.epoch);
	volatile int *done_in = sm.done + (lrow > 0 ? lrow - 1 : 0), *done_out = sm.done + lrow;
	volatile int *taken_me = sm.taken + lrow, *taken_next = sm.taken + (lrow + 1 < IR_ROWS ? lrow + 1 : lrow);
	volatile int *ready = sm.ready + w, *used = sm.used + w;
	uint32_t (*ring_in)[8] = sm.ring[lrow > 0 ? lrow - 1 : 0];
	uint32_t (*ring_out)[8] = sm.ring[lrow];
	const int cpl = J.stride_c >> 1;
	int avail = 0;                                            /* macroblocks of the row above the band known to be stored */
	unsigned eleft = 0;                                       /* lane 0, err_pic: error map byte of the macroblock on the left */
	PT_DECL
#pragma unroll 1
	for (int mbx = 0; mbx < W; mbx++) {
		uint8_t *Y, *C; mb_planes(J, mbx, mby, Y, C);
		/* ---- wait: residual delivered; row above through with macroblocks up to x+1 (top-right neighbour); room in our ring ---- */
		if (lane == 0) {
			unsigned spins = 0; bool bad = false;
			wait_smem_ge(ready, mbx + 1, errp, spins, bad);
			PT_MARK(0)  /* waiting for the residual */
			const int need = min(mbx + 2, W);
			if (from_ring) wait_smem_ge(done_in, need, errp, spins, bad);
			else if (from_global && avail < need) avail = wait_row_progress(prog + mby - 1, base, need, W, errp, spins, bad);
			PT_MARK(1)  /* waiting for the row above */
			/* entry mbx - RING is still the corner sample of the row below's macroblock mbx - RING + 1 */
			if (to_ring) wait_smem_ge(taken_next, mbx - IR_RING + 2, errp, spins, bad);
			if (bad) atomicExch(J.err, 1u);
			__threadfence_block();
			*taken_me = mbx;
		}
		__syncwarp();
		const E264MbRec *r = (const E264MbRec *)sm.recs[w][mbx % IR_RECS];
		const int kind = r->kind;
		WarpSmem *ws = &sm.ws[w][mbx % IR_SLOTS];
		/* ---- the row above into the tile ---- */
		if (from_ring) {
			if (lane < 4) *(uint32_t *)&YT(4 * lane, -1) = ring_in[mbx % IR_RING][lane];
			else if (lane < 6) { if (mbx + 1 < W) *(uint32_t *)&YT(16 + 4 * (lane - 4), -1) = ring_in[(mbx + 1) % IR_RING][lane - 4]; }
			else if (lane == 6) { if (mbx > 0) YT(-1, -1) = (uint8_t)(ring_in[(mbx - 1) % IR_RING][3] >> 24); }
			else if (!LUMA && lane >= 8 && lane < 12) *(uint32_t *)&CT((lane - 8) >> 1, 4 * (lane & 1), -1) = ring_in[mbx % IR_RING][lane - 4];
			else if (!LUMA && lane == 12) { if (mbx > 0) CT(0, -1, -1) = (uint8_t)(ring_in[(mbx - 1) % IR_RING][5] >> 24); }
			else if (!LUMA && lane == 13) { if (mbx > 0) CT(1, -1, -1) = (uint8_t)(ring_in[(mbx - 1) % IR_RING][7] >> 24); }
		} else if (from_global) load_row_above<LUMA>(ws, Y - J.stride_y, C - J.stride_c, cpl, mbx > 0, mbx < W - 1, lane);
		__syncwarp();
		PT_MARK(2)      /* ring room, hand-shake, row above into the tile */
		/* ---- the macroblock ---- */
		if (kind == MBK_INTER) {   /* reconstructed by the inter kernel: fetch its right column and bottom row for the neighbours to come */
			if (lane < 16) YT(15, lane) = __ldcg(Y + (size_t)lane * J.stride_y + 15);
			else if (!LUMA) { const int j = lane - 16; CT(j >> 3, 7, j & 7) = __ldcg(C + (j >> 3) * cpl + (size_t)(j & 7) * J.stride_c + 7); }
			if (to_ring) {
				if (lane < 4) ring_out[mbx % IR_RING][lane] = __ldcg((const uint32_t *)(Y + (size_t)15 * J.stride_y) + lane);
				else if (!LUMA && lane < 8) ring_out[mbx % IR_RING][lane] = __ldcg((const uint32_t *)(C + ((lane - 4) >> 1) * cpl + (size_t)7 * J.stride_c) + (lane & 1));
			}
		} else {
			if (kind == MBK_IPCM) load_pcm<LUMA>(ws, J, r, lane);
			else {
				intra_luma(ws, r, lane);
				PT_MARK(3)  /* luma prediction */
				if (!LUMA) intra_chroma(ws, r, lane);
				PT_MARK(4)  /* chroma prediction */
			}
			store_mb<LUMA>(ws, J, Y, C, lane);
			if (to_ring) {
				if (lane < 4) ring_out[mbx % IR_RING][lane] = *(const uint32_t *)&YT(4 * lane, 15);
				else if (!LUMA && lane < 8) ring_out[mbx % IR_RING][lane] = *(const uint32_t *)&CT((lane - 4) >> 1, 4 * (lane & 1), 7);
			}
		}
		__syncwarp();
		PT_MARK(5)      /* stores */
		/* ---- error map byte: stored before the publication below that covers the macroblock ---- */
		if (MAPS && lane == 0) {
			uint8_t *map = map_of(J, J.dst_slot);
			unsigned e = r->err;
			if (kind == MBK_INTER) e = __ldcg(map + mby * W + mbx);      /* written by the inter kernel */
			else {
				const unsigned av = map_intra_neighbours(r);
				auto above = [&](int x) -> unsigned { return from_ring ? sm.ering[lrow - 1][x % IR_RING] : __ldcg(map + (mby - 1) * W + x); };
				if (av & 1) e = max(e, eleft);
				if (av & 2) e = max(e, above(mbx));
				if (av & 4) e = max(e, above(mbx + 1));
				if (av & 8) e = max(e, above(mbx - 1));
			}
			map[mby * W + mbx] = (uint8_t)e;
			if (to_ring) sm.ering[lrow][mbx % IR_RING] = (uint8_t)e;
			eleft = e;
		}
		/* ---- publish: shared-memory counter for the row below in this band; global counter for the next band, one chunk late ---- */
		if (lane == 0) {
			if (to_ring) { __threadfence_block(); *done_out = mbx + 1; }
			if (to_global && mbx > 0 && mbx % IR_CHUNK == 0) publish_row_progress(prog + mby, base, mbx);   /* covers macroblocks 0..mbx-1, stored in earlier iterations */
		}
		/* right-most column becomes the next macroblock's left neighbour (the other slot's tile) */
		{
			WarpSmem *wn = &sm.ws[w][(mbx + 1) % IR_SLOTS];
			if (lane < 16) wn->ytile[(lane + 1) * YT_STRIDE + 15] = YT(15, lane);
			else if (!LUMA && lane < 24) wn->ctile[0][(lane - 16 + 1) * CT_STRIDE + 7] = CT(0, 7, lane - 16);
			if (!LUMA && lane < 8) wn->ctile[1][(lane + 1) * CT_STRIDE + 7] = CT(1, 7, lane);
		}
		__syncwarp();
		if (lane == 0) { __threadfence_block(); *used = mbx + 1; }
		avail = __shfl_sync(0xffffffffu, avail, 0);
		PT_MARK(6)      /* publication, column hand-over */
	}
	PT_FLUSH(8)
	__syncwarp();
	if (lane == 0) {
		*taken_me = W + IR_RING;       /* nothing of the ring above is needed any more */
		if (to_global) publish_row_progress(prog + mby, base, W);
	}
}

/* MAPS: the picture has err_pic; LUMA: the picture is luma-only (recon.cu launches the instantiation that matches them,
 * so clean colour pictures run code without any map or luma-only test).  The luma-only instantiations state one block
 * per SM: without it ptxas fits them into 64 registers and spills (with it 104 / 106, no spill); 0 leaves the colour
 * ones as they were */
template <bool MAPS, bool LUMA>
__global__ void __launch_bounds__(IR_ROWS * 64, LUMA ? 1 : 0) e264_intra_rows_kernel(PicJob J) {
	TraceScope trace_(J, 2);
	reset_next_tickets(J);
	extern __shared__ __align__(16) unsigned char ir_smem_raw[];
	IntraRowsSmem &sm = *(IntraRowsSmem *)ir_smem_raw;
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, w = wid & (IR_ROWS - 1);
	const bool transform = wid >= IR_ROWS;
	const int bands = (J.h_mbs + IR_ROWS - 1) / IR_ROWS;
	unsigned parbits = 0;
	if (transform && lane == 0) mbar_setup(sm.bars[w], IR_SLOTS);
	/* bands in dispatch order: a band only waits for bands drawn before it */
	for (;;) {
		__syncthreads();
		if (threadIdx.x < IR_ROWS) { sm.done[threadIdx.x] = 0; sm.taken[threadIdx.x] = 0; sm.ready[threadIdx.x] = 0; sm.used[threadIdx.x] = 0; }
		if (threadIdx.x == 0) sm.band = (int)atomicAdd(J.tickets + TICKET_INTRA, 1u);
		__syncthreads();
		const int band = sm.band;
		if (band >= bands) break;
		if (transform) intra_row_transform<LUMA>(J, sm, band, w, lane, parbits);
		else intra_row_walk<MAPS, LUMA>(J, sm, band, w, lane);
	}
}


/* ---- intra macroblocks of P and B pictures ----
 * The parser lists them in raster order (E264Staging.intra_list); warps draw list entries by ticket, so a macroblock
 * only ever waits for entries drawn before its own.  Neighbours: A, D, B, C "reconstructed" flags — inter neighbours were
 * flagged by e264_inter4_kernel (kernel boundary), intra ones are flagged here after a fence.  The coefficient run is
 * fetched (cp.async.bulk) and inverse-transformed while the neighbours finish. */
/* Block size: the kernel's span is the longest chain of dependent intra macroblocks, not its amount of work, and the inter
 * kernel's blocks need a WHOLE SM: a few big blocks (INTRA_WARPS warps, several list entries per warp) leave most SMs to
 * them, where many 4-warp blocks put one small, latency-bound block on nearly every SM.  H100 (results/h100_geometry.txt),
 * 1080p replay of 32 streams: 16 warps 19.6 k frames/s, 8 warps 19.3 k, 4 warps 19.3 k. */
#ifndef INTRA_WARPS
#define INTRA_WARPS 16
#endif
struct __align__(16) IntraTkSmem {
	WarpSmem ws[INTRA_WARPS];
	int16_t coef[INTRA_WARPS][RES_COEF_MAX];
	unsigned long long bars[INTRA_WARPS];
};
/* The error map byte of an intra macroblock of a P/B picture, once the flags of its neighbours have been seen (lanes 0-3
 * acquired them, the __syncwarp() behind the waits orders the loads here).  Not inlined: only pictures with err_pic pay. */
__device__ __noinline__ void intra_error_byte(uint8_t *map, const E264MbRec *r, int mb, int W, int lane) {
	const unsigned av = map_intra_neighbours(r);
	int idx = -1;
	if (lane == 0 && (av & 1)) idx = mb - 1;
	else if (lane == 1 && (av & 2)) idx = mb - W;
	else if (lane == 2 && (av & 4)) idx = mb - W + 1;
	else if (lane == 3 && (av & 8)) idx = mb - W - 1;
	const unsigned e = __reduce_max_sync(0xffffffffu, idx >= 0 ? (unsigned)__ldcg(map + idx) : 0u);
	if (lane == 0) map[mb] = (uint8_t)max(e, (unsigned)r->err);
}
template <bool MAPS, bool LUMA>   /* as for e264_intra_rows_kernel */
__global__ void __launch_bounds__(INTRA_WARPS * 32) e264_intra_kernel(PicJob J) {
	TraceScope trace_(J, 2);
	reset_next_tickets(J);
	extern __shared__ __align__(16) unsigned char intra_tk_smem_raw[];
	IntraTkSmem &sm = *(IntraTkSmem *)intra_tk_smem_raw;
	const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
	WarpSmem *ws = &sm.ws[w];
	const int nmb = J.w_mbs * J.h_mbs, W = J.w_mbs, cpl = J.stride_c >> 1;
	unsigned parity = 0;
	if (lane == 0) mbar_setup(&sm.bars[w], 1);
	__syncwarp();
	for (;;) {
		unsigned t = 0;
		if (lane == 0) t = atomicAdd(J.tickets + TICKET_INTRA, 1u);
		t = __shfl_sync(0xffffffffu, t, 0);
		if (t >= (unsigned)J.n_intra) break;
		const int mb = (int)__ldg(J.intra_list + t);
		if (mb >= nmb) continue;
		const int mbx = mb % W, mby = mb / W;
		if (lane < 12) ws->rec4[lane] = __ldg((const uint4 *)(J.recs + mb) + lane);
		__syncwarp();
		const E264MbRec *r = (const E264MbRec *)ws->rec4;
		const int kind = r->kind;
		if (kind == MBK_INTER) continue;      /* (the list holds intra macroblocks only) */
		uint8_t *Y, *C; mb_planes(J, mbx, mby, Y, C);
		if (kind == MBK_IPCM) {
			load_pcm<LUMA>(ws, J, r, lane);
			store_mb<LUMA>(ws, J, Y, C, lane);
		} else {
			if (r->coded != 0) {
				coef_request(J, r, sm.coef[w], &sm.bars[w], lane);
				if (!mbar_wait(&sm.bars[w], parity)) { if (lane == 0) atomicExch(J.err, 3u); }
				parity ^= 1;
				residual_stage<LUMA>(ws, r, J.slices + r->slice_idx, sm.coef[w], lane);
			} else clear_residual(ws, lane);
			{	/* A, D, B, C: one lane each, the four round trips overlap */
				int idx = -1;
				if (lane == 0 && mbx > 0) idx = mb - 1;
				else if (lane == 1 && mby > 0 && mbx > 0) idx = mb - W - 1;
				else if (lane == 2 && mby > 0) idx = mb - W;
				else if (lane == 3 && mby > 0) idx = mbx < W - 1 ? mb - W + 1 : mb - W;
				if (idx >= 0) wait_flag_acquire(J.flags, idx, J.epoch, J.err);
			}
			__syncwarp();
			if (mby > 0) load_row_above<LUMA>(ws, Y - J.stride_y, C - J.stride_c, cpl, mbx > 0, mbx < W - 1, lane);
			if (mbx > 0) {
				if (lane < 16) YT(-1, lane) = __ldcg(Y + (size_t)lane * J.stride_y - 1);
				else if (!LUMA) { const int j = lane - 16, pl = j >> 3, row = j & 7; CT(pl, -1, row) = __ldcg(C + pl * cpl + (size_t)row * J.stride_c - 1); }
			}
			__syncwarp();
			intra_luma(ws, r, lane);
			if (!LUMA) intra_chroma(ws, r, lane);
			store_mb<LUMA>(ws, J, Y, C, lane);
		}
		__syncwarp();
		if (MAPS) intra_error_byte(map_of(J, J.dst_slot), r, mb, W, lane);   /* before the flag: the macroblocks that wait for it read the byte */
		if (lane == 0) { __threadfence(); *(volatile unsigned *)(J.flags + mb) = J.epoch; }
		__syncwarp();
	}
}
