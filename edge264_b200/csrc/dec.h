/* dec.h — host-side decoder state: parameter sets, DPB, slice context.
 * New code; it covers what the reference keeps in Edge264Decoder / Edge264Task / Edge264Context
 * (reference: edge264_internal.h:223-462) but organised around "parse to records, reconstruct
 * elsewhere". */
#ifndef E264B_DEC_H
#define E264B_DEC_H
#include <stdint.h>
#include <stddef.h>
#include <pthread.h>
#include "records.h"
#include "bits.h"
#include "cabac.h"
#include "../../include/edge264.h"

#define E264_MAX_SLOTS   32       /* device frame slots: two views of up to 15 references (the width of taint, ref_mask and slot_ids) */
#define E264_MONO_SLOTS  20       /* cap of a single-view sequence: 16 references + current + slack */
#define E264_MAX_SLICES  64       /* slices per picture (slice_idx is a byte; more are rejected) */
#define E264_MAX_PPS     16

typedef struct SPS {
	int valid;
	int profile_idc, level_idc, constraint_flags;
	int log2_max_frame_num, poc_type, log2_max_poc_lsb;
	int delta_pic_order_always_zero_flag, offset_for_non_ref_pic, offset_for_top_to_bottom_field;
	int num_ref_frames_in_poc_cycle; int32_t offset_for_ref_frame[256];
	int max_num_ref_frames, gaps_allowed;
	int width_mbs, height_mbs, direct_8x8_inference;
	int crop[4];                       /* left, right, top, bottom in luma samples */
	int max_num_reorder_frames, max_dec_frame_buffering;
	int scaling_present;
	uint8_t sl4x4[6][16], sl8x8[2][64];   /* resolved (fall-back rule A applied), raster order */
} SPS;

typedef struct PPS {
	int valid;
	int entropy_coding_mode, bottom_field_pic_order_present;
	int num_ref_idx_default[2];
	int weighted_pred_flag, weighted_bipred_idc;
	int pic_init_qp, chroma_qp_index_offset[2];
	int deblocking_filter_control_present, transform_8x8_mode;
	uint8_t sl4x4[6][16], sl8x8[2][64];   /* resolved against the SPS active when the PPS was parsed */
} PPS;

/* per-macroblock parsing context kept for the current picture only */
typedef struct MbInfo {
	uint16_t slice_id;        /* 0 = not decoded yet */
	uint8_t  is_intra, is_skip, is_direct, is_pcm, is_i16, t8x8;
	uint8_t  cbp;             /* luma 4 bits | chroma << 4 */
	uint8_t  chroma_pred_mode;
	uint8_t  cbf_dc;          /* bit0 luma DC (Intra16x16), bit1 Cb DC, bit2 Cr DC */
	uint8_t  cbf_cb, cbf_cr;  /* 4 AC bits each */
	uint16_t cbf_luma;        /* CABAC coded_block_flag per luma4x4BlkIdx */
	uint8_t  direct8;         /* per 8x8: predicted in direct mode (B) */
	uint8_t  tc[24];          /* CAVLC total_coeff: luma z-order 0..15, Cb 16..19, Cr 20..23 */
	int8_t   ipm[16];         /* Intra4x4/8x8PredMode per luma4x4BlkIdx, 2 when not I_NxN */
	uint8_t  mvd[2][16][2] __attribute__((aligned(2)));   /* |mvd| clipped to 255 per list/blk/comp (CABAC ctxIdxInc); filled pairwise as 16-bit words */
} MbInfo;

/* Neighbourhood of the macroblock being parsed, laid out so that motion-vector prediction and the mvd context are
 * plain index arithmetic: entry (x4, y4) of the 4x4-block grid, x4 in -1..4, y4 in -1..3, sits at (y4 + 1) * 8 + x4 + 1.
 * Row -1 and column -1 are copied from the neighbouring macroblocks' records when an inter macroblock starts (the
 * reference keeps the same information in its mvs/refIdx neighbour offsets, edge264_internal.h:128-143,
 * edge264_mvpred.c:44-71); the interior is written as partitions are parsed and flushed to the record at the end. */
typedef struct MvCache {
	uint32_t mv[2][40];       /* (uint16)x | y << 16; 0 where the list is not used or the block is unavailable */
	int8_t   ref[2][40];      /* reference index; -1 list not used / intra; -2 not available */
	uint16_t mvd[2][40];      /* |mvd_x| | |mvd_y| << 8, each clipped to 255 */
} MvCache;
#define MC_IDX(x4, y4) (((y4) + 1) * 8 + (x4) + 1)

typedef struct SliceHeader {
	int first_mb, slice_type, pps_id, frame_num, idr_pic_id, poc_lsb, delta_poc_bottom, delta_poc[2];
	int direct_spatial, num_ref[2];
	int cabac_init_idc, slice_qp, deblock_idc, filter_offset_a, filter_offset_b;
	/* ref_pic_list_modification */
	int n_mod[2]; struct { uint8_t op; uint32_t val; } mod[2][34];
	/* pred_weight_table */
	int luma_log2_wd, chroma_log2_wd;
	int16_t w[2][32][3], o[2][32][3];
	/* dec_ref_pic_marking */
	int no_output_of_prior_pics, long_term_reference_flag, adaptive_marking;
	int n_mmco; struct { uint8_t op; uint32_t a, b; } mmco[66];
} SliceHeader;

typedef struct Pic {
	int in_use;               /* slot holds a picture that is a reference or waits for output/consumption */
	int ref;                  /* 0 none, 1 short-term, 2 long-term */
	int needed_for_output;
	int frame_num, long_term_idx;
	int poc;                  /* PicOrderCnt = min(top, bottom): direct / implicit weights */
	int poc_top;              /* TopFieldOrderCnt: bumping and B list order (as the reference, headers.c:82,762) */
	int poc_dec, poc_top_dec; /* the values in force while the picture itself is decoded: memory_management_control_operation 5 rebases
	                           * poc/poc_top for output and later pictures only (8.2.1; reference headers.c:46-49, 673-680) */
	int32_t uid;              /* unique id of the picture = FrameId */
	int view;                 /* 0 base view, 1 second view of a stereo sequence (edge264_mvc.h) */
	int ref_frame;            /* the frame the reference decoder would hold the picture in (Edge264Decoder.ref_frame_view) */
	int nonexisting;
	int unfilled;             /* a skipped reference picture whose slot has not been filled yet (edge264_skip.h) */
	E264MbRec *recs;          /* pinned host records of this picture (kept: co-located info for B direct) */
	int32_t slot_uid[E264_MAX_SLOTS];   /* uid held by every slot when this picture was decoded */
	int host_buf;             /* host mirror receiving the pixels; dropped (-1) once submitted AND queued for output */
} Pic;

struct E264Backend;

typedef struct SliceCtx {
	/* entropy coding */
	int cabac;
	CabacDec cd;
	BitReader br;
#ifdef E264_ENCODER
	CabacEnc ce;
	BitWriter *bw;
	struct GenState *gen;
	int16_t gen_coefs[16 + 256 + 8 + 128];
	struct MbSyn *syn;
#endif
	/* geometry and slice parameters */
	int w_mbs, h_mbs;
	int slice_type, slice_id, slice_idx;
	int num_ref[2], direct_spatial, direct_8x8_inference, transform_8x8_mode;
	int qp, chroma_qp_offset[2], last_qp_delta_nz, deblock_idc, cabac_init_idc_col;
	int cur_poc;
	int8_t  ref_slot[2][32];
	int32_t ref_uid[2][32];
	int32_t ref_poc[2][32];
	uint8_t ref_long[2][32];
	/* temporal direct */
	const E264MbRec *col_recs; const int32_t *col_slot_uid; int col_valid;
	/* picture arrays */
	MbInfo *mbi; E264MbRec *recs; int16_t *coefs; uint32_t n_coefs, coef_cap;
	/* current macroblock */
	int mbx, mby, mbaddr;
	MbInfo *cur, *A, *B, *C, *D;
	E264MbRec *rec, *recA, *recB, *recC, *recD;
	int skip_run, prev_mb_skipped;
	int n_intra;
	int error;
	int missing_ref;          /* a reference-list entry of the slice has no picture (a substitute predicts in its place) */
	int any_err;              /* a delivered record got a nonzero err (slice_dec.c) */
	int luma_only;            /* chroma residuals are parsed, then dropped from the pool and the record (edge264_luma.h) */
	MvCache mc;
} SliceCtx;

/* One slice waiting to be parsed: its own copy of the RBSP and of the co-located picture's slot_uid table, and a slice
 * context prepared by the header parser.  dep = the picture whose records a B slice reads as co-located motion (must
 * be completely parsed first). */
struct PicBuild;
typedef struct SliceJob {
	struct SliceJob *next;
	uint8_t *rbsp;
	struct PicBuild *dep; uint64_t dep_seq;
	int col_slot;
	int32_t col_slot_uid[E264_MAX_SLOTS];
	SliceCtx sc;
} SliceJob;

/* One picture between its first slice header and its submission to the backend.  Without worker threads there is one
 * and the calling thread does its work; with workers (edge264_alloc n_threads != 0) several pictures are parsed at
 * the same time, like the reference's slice tasks (edge264_internal.h:223-261, worker_loop edge264_headers.c:450-603). */
typedef struct PicBuild {
	MbInfo *mbi;
	E264MbRec *recs; int16_t *coefs; uint32_t coef_cap, n_coefs;
	E264SliceRec *slices; int n_slices;
	uint32_t *intra_list; int staging;
	int mbs_done, n_intra, any_deblock; uint16_t slice_counter;
	int no_deblock;           /* the picture is output without the loop filter (edge264_loopfilter.h): its records are those of deblock idc 1 */
	int slot, host_buf, conceal_ref;
	int any_err;              /* some record has err != 0 (a slice error, a missing reference, concealment) */
	int32_t slot_ids[E264_MAX_SLOTS];   /* FrameId held by every frame slot when the picture started (Pic.slot_uid): the motion export's table */
	uint32_t ref_mask;        /* frame slots the picture's records may predict from */
	int in_use, closed, running, parsed;
	int close_complete;       /* a worker closes the picture once its slices cover every macroblock (edge264_latency.h) */
	int held;                 /* the calling thread is adding a slice: no worker may close the picture meanwhile */
	uint64_t seq;
	E264PicDesc pd;           /* filled when parsed: what goes to the backend when the picture's turn comes */
	SliceJob *head, *tail;
} PicBuild;
#define E264_MAX_BUILDS 6
#define E264_MAX_THREADS 4

/* host mirror of an output picture */
typedef struct HostBuf {
	uint8_t *p;           /* pinned (or user) memory, frame layout of the reference */
	void *mbs;            /* user mbs allocation when alloc_cb is used (unused by us) */
	uint8_t *map;         /* pinned host memory: the picture's error map (one byte per macroblock), valid when err_pic */
	int err_pic;          /* the picture was reconstructed with an error map (E264PicDesc.err_pic) */
	uint8_t *motion;      /* the picture's motion export (records.h E264_MOTION_*), memory of the samples' kind; NULL without export */
	void *motion_mbs;     /* the mbs allocation alloc_cb returned with it */
	int motion_dev;       /* motion is device memory */
	uint8_t *packed;      /* the picture's packed output (records.h e264_packed_layout), memory of the samples' kind; NULL without it */
	void *packed_mbs;     /* the mbs allocation alloc_cb returned with it */
	int packed_dev;       /* packed is device memory */
	E264PackedDesc pk;    /* what the picture in the buffer was packed as (cropping rectangle and resized size of its sequence) */
	uint8_t *picstats;    /* the picture's statistics (records.h E264_PICSTATS_*), memory of the samples' kind; NULL without them */
	void *picstats_mbs;   /* the mbs allocation alloc_cb returned with it */
	int picstats_dev;     /* picstats is device memory */
	int state;            /* 0 free, 1 attached to a decoded picture, 2 in the output queue, 3 handed out */
	int borrowed;
	int32_t frame_id;
	uint64_t ticket;      /* backend completion ticket of the picture written into it */
	int ref_frame;        /* Pic.ref_frame of the picture in it */
	int submitted;        /* reconstruction has been enqueued (ticket valid) */
} HostBuf;
#define E264_MAX_HOSTBUFS 64

struct Edge264Decoder {
	/* configuration */
	Edge264AllocCb alloc_cb; Edge264FreeCb free_cb; void *alloc_arg;
	const struct E264Backend *be; void *be_ctx;
	/* parameter sets */
	SPS sps; PPS pps[E264_MAX_PPS];
	SPS ssps;                          /* subset SPS of the second view, valid while mvc */
	int mvc;                           /* stereo: a subset SPS was accepted; off again at End of sequence and flush (edge264_mvc.h) */
	/* geometry of the active sequence */
	int configured, w_mbs, h_mbs, stride_y, stride_c, plane_y, plane_c, frame_bytes, n_slots;
	Edge264Frame out_fmt;
	/* DPB */
	Pic pics[E264_MAX_SLOTS];
	int cur;                           /* slot of the picture being decoded, -1 none */
	int cur_idr, cur_nal_ref_idc;
	/* Each view keeps its own DPB: the helpers below work on the pictures of d->view, the view of the picture being started
	 * or finished (the reference's same_views mask, edge264_headers.c:61-100) */
	int view;
	int base_slot;                     /* the last base view picture: the second view's inter-view reference, kept in its slot until the next one */
	int inter_view_flag;               /* of the last prefix NAL unit: the base view component that follows is an inter-view reference */
	int au_skip;                       /* the skip decision of the access unit's base view, which its second view follows */
	/* The reference decoder counts a picture just inserted in the DPB towards its view's max_num_reorder_frames only when
	 * the last picture of its frame buffer was of the same view (its view mask is taken before the picture joins it,
	 * edge264_headers.c:971, 1160, 1249).  Which frame buffer that is follows from its allocation rule (the lowest one
	 * holding no reference, no picture waiting for output, none queued or borrowed) and is tracked here so that second views
	 * leave at the same decode_NAL calls as there.  A single-view stream always counts its picture. */
	uint8_t ref_frame_view[32];
	int ghost_frames;                  /* non-existing frames the reference inserts before the current picture (number_frame_id) */
	int cur_skip;                      /* the current picture is skipped: its headers run, its slice data is dropped */
	int skip_mode;                     /* edge264_set_skip: applied to each picture at its first slice */
	int loop_filter_mode;              /* edge264_set_loop_filter: applied to each picture at its first slice */
	int output_latency;                /* edge264_set_output_latency: -1, or the cap on the reorder depth, applied to each picture at its first slice */
	int low_latency;                   /* output_latency >= 0 at the last picture's first slice: get_frame waits for closed pictures */
	int prev_ref_frame_num[2], prev_ref_poc[2];   /* per view: frame_num and POC of the previous reference picture (8.2.1) */
	int q_prev_ref_frame_num[2], q_cur_frame_num;   /* reference-style absolute frame numbers, only used to number FrameIds like it */
	int32_t next_uid;
	SliceHeader sh;                    /* header of the slice being parsed */
	SliceHeader first_sh;              /* header of the first slice of the current picture (marking) */
	/* current picture build-up */
	PicBuild *pb;                      /* the picture slices are being added to (NULL between pictures) */
	PicBuild builds[E264_MAX_BUILDS];
	int n_builds;
	/* worker threads (0 = the calling thread parses and submits each picture inside edge264_decode_NAL) */
	int n_threads, stop;
	pthread_t threads[E264_MAX_THREADS];
	pthread_mutex_t lock, be_lock;     /* lock: builds, queues, hb[].submitted; be_lock: backend calls from several threads */
	pthread_cond_t work_cv, done_cv;
	uint64_t next_seq, submit_seq;     /* pictures are submitted to the backend in decoding order */
	int submitting;                    /* a thread is inside the backend with picture submit_seq */
	int slot_users[E264_MAX_SLOTS];    /* builds still reading or writing the records of a frame slot */
	uint32_t taint;                    /* frame slots whose error map may be nonzero (E264PicDesc.taint), in submission order */
	PicBuild *slot_build[E264_MAX_SLOTS]; uint64_t slot_build_seq[E264_MAX_SLOTS];
	/* output */
	HostBuf hb[E264_MAX_HOSTBUFS];
	int outq[2][E264_MAX_HOSTBUFS]; int outq_n[2];   /* per view; a stereo frame pairs the heads of both */
	int pending_release[2];            /* host buffers handed out without borrow, released at next decode_NAL */
	int sync_output;                   /* E264_SYNC_OUTPUT=1: get_frame always waits for the device (the behaviour before round 2's last step; A/B switch) */
	int motion;                        /* edge264_enable_motion: every output picture carries its motion export */
	int slices_seen;                   /* a slice NAL unit has been decoded (edge264_enable_motion / _packed / _resized / _picstats are refused from then on) */
	int packed, packed_format, packed_scale;   /* edge264_enable_packed: every output picture carries its packed output */
	int packed_width, packed_height;   /* edge264_enable_resized (packed_scale -1): the requested size, one of them possibly 0 */
	int luma_only;                     /* edge264_enable_luma_only: every picture is reconstructed with luma only */
	int picstats;                      /* edge264_enable_picstats: every output picture carries its statistics */
	int block_output;                  /* the last decode_NAL asked the application to fetch frames (ENOBUFS, end of stream): get_frame waits for the device */
	/* scratch: RBSP of the last non-slice NAL unit */
	uint8_t *rbsp; size_t rbsp_cap;
};

/* backend = the thing that turns records into pixels.  The product library binds the CUDA
 * runtime (edge264_b200/csrc/recon.cu); the test-only oracle library binds oracle/port_recon.c. */
typedef struct E264Backend {
	const char *name;
	int  (*create)(void **ctx);
	void (*destroy)(void *ctx);
	/* (re)allocate n_slots frame slots for this geometry; drops all pictures */
	int  (*configure)(void *ctx, const E264PicDesc *geom, int n_slots);
	/* pinned host allocation helpers */
	void *(*host_alloc)(void *ctx, size_t bytes);
	void  (*host_free)(void *ctx, void *p);
	/* staging for the next picture: returns pinned host areas the parser fills directly */
	int  (*acquire_staging)(void *ctx, int slot, E264Staging *out);
	/* reconstruct one picture into `pd->dst_slot` and mirror it into host_out; returns a ticket */
	int  (*submit)(void *ctx, const E264PicDesc *pd, uint8_t *host_out, uint64_t *ticket);
	int  (*wait)(void *ctx, uint64_t ticket);
	/* fill a slot with a constant (non-existing frames of frame_num gaps); its error map becomes all 100 */
	int  (*fill_slot)(void *ctx, int slot, int y, int c);
	/* non-blocking form of wait: 0 = the picture is complete, EAGAIN = not yet, < 0 = device error */
	int  (*poll)(void *ctx, uint64_t ticket);
	/* error maps (Edge264Frame.mb_errors).  A backend that keeps them has all three; one with NULL here has none, and its
	 * pictures come out with mb_errors NULL.  submit_maps is submit that also copies the picture's error map into
	 * host_map when pd->err_pic; pinned_alloc / pinned_free give host memory whatever the output mirrors are. */
	int  (*submit_maps)(void *ctx, const E264PicDesc *pd, uint8_t *host_out, uint8_t *host_map, uint64_t *ticket);
	void *(*pinned_alloc)(void *ctx, size_t bytes);
	void  (*pinned_free)(void *ctx, void *p);
	/* motion export (include/edge264_motion.h); NULL: the backend has none.  submit_maps that also writes the picture's
	 * export into `motion` (E264_MOTION_BYTES per macroblock), with slot_ids[s] the FrameId of frame slot s
	 * (E264_MAX_SLOTS entries, -1 for an empty slot); *on_device tells whether `motion` is device memory. */
	int  (*submit_motion)(void *ctx, const E264PicDesc *pd, uint8_t *host_out, uint8_t *host_map, uint8_t *motion, const int32_t *slot_ids, int *on_device, uint64_t *ticket);
	/* packed output (include/edge264_packed.h); NULL: the backend has none.  submit with every optional output in one
	 * struct (records.h E264Outputs): the error map, the motion export and the packed output, each left out when NULL. */
	int  (*submit_outputs)(void *ctx, const E264PicDesc *pd, uint8_t *host_out, const E264Outputs *out, uint64_t *ticket);
} E264Backend;
const E264Backend *e264_default_backend(void);

/* slice_dec.c */
int e264_parse_slice_data(SliceCtx *s);
/* helpers shared with the generator (syntax_impl.h) */
#endif
