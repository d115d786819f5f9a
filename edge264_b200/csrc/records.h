/* records.h — the host→device record ABI of the reconstruction path.
 *
 * The CPU parser turns each macroblock into ONE fixed-size E264MbRec plus a variable run of int16
 * coefficients in the picture's coefficient pool; a picture also carries a small table of
 * E264SliceRec.  This replaces the reference's in-memory contract between its slice parser and its
 * pixel functions (reference: Edge264Macroblock edge264_internal.h:128-143, Edge264Task :223-261,
 * ctx->c[] :311) — the information is the same (SURVEY.md Appendix C), the layout is ours.
 *
 * Index conventions: every per-4x4 quantity (mv, coded bits, intra modes) is indexed by the spec's
 * luma4x4BlkIdx "z-order" b = 4*(8x8 index) + (4x4 index inside it); 8x8 quantities by raster
 * 8x8 index.  Coefficients inside a block are in RASTER order (c[y*N+x]) as int16 levels before
 * dequantisation.
 *
 * Coefficient run of one macroblock, at pool[coef_off], in this order (all pieces are multiples of
 * 8 int16 so every block stays 16-byte aligned):
 *   I_PCM:  384 bytes of raw samples (Y 256, Cb 64, Cr 64) = 192 int16 slots
 *   else:   [16 luma DC levels, raster 4x4 over the 16 blocks]     if coded bit 24 (Intra16x16 only)
 *           for each coded luma 4x4 block in z-order: 16 levels    (transform 4x4)
 *           or for each coded 8x8 block: 64 levels                 (transform 8x8; its 4 bits are set together)
 *           [4 Cb DC + 4 Cr DC levels, raster 2x2]                 if coded bit 25 or 26
 *           for each coded chroma AC block (Cb0..3 then Cr0..3): 16 levels (slot 0 unused, zero)
 *
 * The record contract: what the parser guarantees for every picture it submits, damaged input included, and what the
 * kernels rely on (a record outside it may make a kernel read samples nobody wrote, or copy outside the coefficient
 * pool).  oracle/record_check.c checks this list (E264_CHECK_RECORDS=1 on the CPU restatement backend) but for err, which
 * the error-map test backend checks.
 *   Picture   dst_slot < n_slots; 1 <= n_slices <= 64; intra_list holds the addresses of the non-inter macroblocks in
 *             raster order and n_intra counts them; any_deblock is set when a macroblock has MBF_DEBLOCK.
 *   Slices    filter_offset_a/b even in -12..12; deblock_idc 0..2; slice_type 0..2; wp_mode 0..2; log2_wd 0..7;
 *             weights -128..128, offsets -128..127, implicit_w1 -64..128; scaling entries 1..255.
 *   Kind      kind 0..4, flags inside MBF_*, slice_idx < n_slices, coded inside CODED_*.  MBF_T8x8 is set on every
 *             MBK_I8x8 and never on MBK_I4x4, MBK_I16x16 or MBK_IPCM; with MBF_T8x8 the luma bits come in groups of 4.
 *             CODED_Y_DC appears only on MBK_I16x16; MBK_IPCM has no coded bits.
 *   QPs       qp[0] 0..51 (0 for MBK_IPCM); qp[1], qp[2] are values of Table 8-15 (0..39).
 *   Levels    coef_off is a multiple of 8 and the run (192 slots for MBK_IPCM) ends inside n_coefs.
 *   Intra     a neighbour that a mode byte marks available (bit clear) lies inside the picture and in the same slice
 *             (slice_idx); C is always unavailable for the 4x4 blocks z = 3, 7, 11, 13, 15 and the 8x8 block 3.
 *             The parser sets the bits of 6.4.11.4 exactly; a record may mark more neighbours unavailable than that
 *             (the concealment records mark all of them).  Every mode is legal for its bits (e264_intra_mode_legal).
 *   Deblock   MBF_EDGE_L / MBF_EDGE_T only with MBF_DEBLOCK, never on the picture's left column / top row; MBF_DEBLOCK
 *             only in slices with deblock_idc != 1.  With deblock_idc 0 both edges are set wherever a neighbour exists,
 *             with deblock_idc 2 an edge is set only towards a macroblock of the same slice.
 *   Error     err <= 100 (checked with the error maps, tests/native/port_maps_backend.c).
 *   Inter     every 8x8 block of an MBK_INTER uses at least one list; a used list has ref_idx 0..15 and a ref_pic in
 *             [0, n_slots) other than dst_slot; an unused list, and every list of an intra macroblock, has -1 in both.
 *             Motion vectors may take any int16 value.
 */
#ifndef E264B_RECORDS_H
#define E264B_RECORDS_H
#include <stddef.h>
#include <stdint.h>

/* widest picture the parser accepts, in macroblocks: the device's row-progress words count a row's macroblocks below
 * PROG_STRIDE (recon_kernels.cuh) */
#define E264_MAX_WIDTH_MBS 1023

enum { MBK_I4x4 = 0, MBK_I8x8 = 1, MBK_I16x16 = 2, MBK_IPCM = 3, MBK_INTER = 4 };

/* E264MbRec.flags */
#define MBF_T8x8     0x01   /* transform_size_8x8_flag */
#define MBF_EDGE_L   0x02   /* deblock the left macroblock edge  (reference filter_edges bit0, slice.c:1692,1724) */
#define MBF_EDGE_T   0x04   /* deblock the top macroblock edge   (bit1, slice.c:1762) */
#define MBF_DEBLOCK  0x08   /* this macroblock is deblocked at all (disable_deblocking_filter_idc != 1) */
#define MBF_SKIP     0x10   /* P_Skip / B_Skip (informational) */

/* bits of E264MbRec.coded */
#define CODED_LUMA(b)   (1u << (b))          /* b = luma4x4BlkIdx 0..15 */
#define CODED_CB_AC(i)  (1u << (16 + (i)))
#define CODED_CR_AC(i)  (1u << (20 + (i)))
#define CODED_Y_DC      (1u << 24)
#define CODED_CB_DC     (1u << 25)
#define CODED_CR_DC     (1u << 26)

/* intra mode bytes: low nibble = prediction mode of the standard (Intra4x4/8x8: 0..8, Intra16x16
 * and chroma: 0..3), high nibble = unavailability of the neighbours A(left)=1, B(top)=2,
 * C(top-right)=4, D(top-left)=8 — the device applies the substitution rules of 8.3.1.2 / 8.3.2.2
 * (the reference resolves the same information into its own 14/32/7/7 mode enums on the host:
 * slice.c:573-594, 720-725, 874-879). */
#define IMODE(mode, unavail) ((uint8_t)((mode) | ((unavail) << 4)))

typedef struct E264MbRec {
	uint8_t  kind;          /* MBK_* */
	uint8_t  flags;         /* MBF_* */
	uint8_t  qp[3];         /* QP_Y, QP'c for Cb, Cr of THIS macroblock */
	uint8_t  chroma_mode;   /* IMODE(intra_chroma_pred_mode, unavail A|B|D) */
	uint8_t  i16_mode;      /* IMODE(Intra16x16PredMode, unavail A|B|D) */
	uint8_t  slice_idx;     /* index into the picture's E264SliceRec table */
	uint32_t coded;         /* CODED_* */
	uint32_t coef_off;      /* int16 index into the picture's coefficient pool */
	uint8_t  modes[16];     /* IMODE per luma4x4BlkIdx (Intra4x4) or in [0..3] per 8x8 (Intra8x8) */
	int8_t   ref_idx[2][4]; /* per list, per 8x8: reference index, -1 = list unused */
	int8_t   ref_pic[2][4]; /* per list, per 8x8: frame slot of the reference picture, -1 = unused */
	uint8_t  err;           /* the macroblock's own error, 0..100 (0 = delivered intact; see E264PicDesc.err_pic) */
	uint8_t  reserved[15];
	int16_t  mv[2][16][2];  /* per list, per luma4x4BlkIdx: quarter-pel (x, y) */
} E264MbRec;                /* 192 bytes */

enum { WP_DEFAULT = 0, WP_EXPLICIT = 1, WP_IMPLICIT = 2 };

typedef struct E264SliceRec {
	int8_t   filter_offset_a;   /* FilterOffsetA = slice_alpha_c0_offset_div2 * 2 */
	int8_t   filter_offset_b;
	uint8_t  deblock_idc;       /* disable_deblocking_filter_idc */
	uint8_t  slice_type;        /* 0 P, 1 B, 2 I */
	uint8_t  wp_mode;           /* WP_* actually in force for this slice */
	uint8_t  luma_log2_wd;
	uint8_t  chroma_log2_wd;
	uint8_t  reserved;
	int16_t  wp_w[2][16][3];    /* explicit weights  [list][refIdx][Y,Cb,Cr] */
	int16_t  wp_o[2][16][3];    /* explicit offsets */
	int16_t  implicit_w1[16][16]; /* implicit bi-pred weight of the list-1 sample for (refIdxL0, refIdxL1), -64..128; w0 = 64 - w1 */
	uint8_t  scaling4x4[6][16]; /* merged scaling lists Y-intra,Cb-intra,Cr-intra,Y-inter,Cb-inter,Cr-inter; raster */
	uint8_t  scaling8x8[2][64]; /* Y-intra, Y-inter; raster */
} E264SliceRec;                 /* 8 + 192 + 192 + 512 + 96 + 128 = 1128 bytes */

/* One picture worth of work for the device (host view; device pointers are filled by the runtime). */
typedef struct E264PicDesc {
	int32_t width_mbs, height_mbs;
	int32_t stride_y, stride_c;   /* bytes; chroma rows alternate Cb,Cr inside one stride_c (reference headers.c:2027-2046) */
	int32_t plane_y;              /* byte offset of the chroma plane inside a frame buffer */
	int32_t frame_bytes;          /* size of one frame slot */
	int32_t dst_slot;             /* frame slot being reconstructed */
	int32_t n_slices;
	int32_t n_coefs;              /* int16 entries used in the coefficient pool */
	int32_t any_deblock;          /* at least one macroblock has MBF_DEBLOCK */
	int32_t n_intra;              /* number of intra macroblocks = entries of the staging's intra_list */
	int32_t staging;              /* handle of the staging area the picture was written into (E264Staging.handle) */
	uint8_t err_pic;              /* error map wanted: some record has err != 0 or a slot in taint is referenced; with 0 the
	                               * kernels touch no map and the slot's map counts as all zeros afterwards */
	uint8_t luma_only;            /* reconstruct and deblock the Y plane only, then set the slot's chroma plane to 128
	                               * (include/edge264_luma.h); the chroma levels and coded bits of the records are ignored.
	                               * The parser's records of such pictures reconstruct chroma 128 anyway (decoder.c
	                               * edge264_enable_luma_only), so a backend that ignores this field gives the same frame */
	uint8_t reserved[2];          /* (err_pic and luma_only share the word err_pic had: the struct stays 56 bytes, the size
	                               * the picture dumps of the deblocking tests are read with) */
	uint32_t taint;              /* bit s: frame slot s holds a picture whose map may be nonzero (fill_slot, err_pic) */
} E264PicDesc;

/* The motion export of one picture (include/edge264_motion.h): one buffer of E264_MOTION_BYTES bytes per macroblock, the
 * four arrays at these offsets, in bytes per macroblock of the picture (nmb = width_mbs * height_mbs):
 *   mv            E264_MOTION_MV * nmb    int16 [2][4 height_mbs][4 width_mbs][2]
 *   ref_frame_id  E264_MOTION_REF * nmb   int32 [2][2 height_mbs][2 width_mbs]
 *   mb_type       E264_MOTION_TYPE * nmb  uint8 [height_mbs][width_mbs]
 *   mb_qp         E264_MOTION_QP * nmb    uint8 [height_mbs][width_mbs] */
enum { E264_MOTION_MV = 0, E264_MOTION_REF = 128, E264_MOTION_TYPE = 160, E264_MOTION_QP = 161, E264_MOTION_BYTES = 162 };

/* The picture statistics of one picture (include/edge264_picstats.h): one buffer of E264_PICSTATS_BYTES(nmb) bytes,
 *   hist    at E264_PICSTATS_HIST                uint32 [3][256]
 *   sum     at E264_PICSTATS_SUM                 uint32 [3][height_mbs][width_mbs]
 *   sum_sq  at E264_PICSTATS_SUM + 12 * nmb      uint32 [3][height_mbs][width_mbs] */
enum { E264_PICSTATS_HIST = 0, E264_PICSTATS_SUM = 3072, E264_PICSTATS_MB_BYTES = 24 };
#define E264_PICSTATS_SUM_SQ(nmb) (E264_PICSTATS_SUM + 12 * (size_t)(nmb))
#define E264_PICSTATS_BYTES(nmb) (E264_PICSTATS_SUM + E264_PICSTATS_MB_BYTES * (size_t)(nmb))

/* The packed output of one picture (include/edge264_packed.h): the cropped picture as I420 or NV12, box-downscaled by
 * 1 << log2_scale, or resized to target_width x target_height, in one buffer.  E264PackedDesc says what to pack,
 * e264_packed_layout where every plane goes: sizes are ceil(cropped size / scale), or the target (chroma: half of it), a
 * row stride is the row's bytes rounded up to 64, a plane starts on a multiple of 256. */
enum { E264_PACKED_I420 = 0, E264_PACKED_NV12 = 1 };
typedef struct E264PackedDesc {
	int32_t format, log2_scale;         /* E264_PACKED_*, 0..3, or -1 for the resized output */
	int32_t left, top, width, height;   /* the cropping rectangle inside the coded picture, luma samples (all even: 4:2:0 frames) */
	int32_t target_width, target_height;   /* resized output: the luma size, even, 2..16384; 0, 0 in the power-of-two mode */
} E264PackedDesc;
typedef struct E264PackedLayout {
	int32_t width, height, width_C, height_C;   /* samples per plane after cropping and scaling */
	int32_t stride[3], offset[3];               /* I420: Y, Cb, Cr; NV12: Y, interleaved CbCr, unused (0) */
	int32_t bytes;                              /* size of the buffer */
} E264PackedLayout;
static inline E264PackedLayout e264_packed_layout(const E264PackedDesc *p) {
	E264PackedLayout l;
	if (p->target_width) {
		l.width = p->target_width; l.height = p->target_height; l.width_C = l.width >> 1; l.height_C = l.height >> 1;
	} else {
		const int n = 1 << p->log2_scale;
		l.width = (p->width + n - 1) >> p->log2_scale; l.height = (p->height + n - 1) >> p->log2_scale;
		l.width_C = ((p->width >> 1) + n - 1) >> p->log2_scale; l.height_C = ((p->height >> 1) + n - 1) >> p->log2_scale;
	}
	l.stride[0] = (l.width + 63) & ~63;
	l.stride[1] = ((p->format == E264_PACKED_NV12 ? 2 * l.width_C : l.width_C) + 63) & ~63;
	l.stride[2] = p->format == E264_PACKED_NV12 ? 0 : l.stride[1];
	l.offset[0] = 0;
	l.offset[1] = (l.stride[0] * l.height + 255) & ~255;
	l.offset[2] = p->format == E264_PACKED_NV12 ? 0 : (l.offset[1] + l.stride[1] * l.height_C + 255) & ~255;
	l.bytes = (p->format == E264_PACKED_NV12 ? l.offset[1] + l.stride[1] * l.height_C : l.offset[2] + l.stride[2] * l.height_C);
	l.bytes = (l.bytes + 255) & ~255;
	return l;
}

/* What a submit may produce besides the samples; a NULL pointer leaves that output out (no launch, no copy, no
 * allocation for it).  map: the error map, copied when pd->err_pic.  motion: the motion export, slot_ids[s] the FrameId
 * of frame slot s for s < n_ids, -1 elsewhere.  packed: the packed output described by pk.  picstats: the picture
 * statistics, the histograms over the cropping rectangle ps_left, ps_top, ps_width x ps_height (luma samples inside the
 * coded picture, all even).  The *_on_device words (may be NULL) receive whether that destination is device memory. */
typedef struct E264Outputs {
	uint8_t *map;
	uint8_t *motion; const int32_t *slot_ids; int32_t n_ids; int *motion_on_device;
	uint8_t *packed; E264PackedDesc pk; int *packed_on_device;
	uint8_t *picstats; int32_t ps_left, ps_top, ps_width, ps_height; int *picstats_on_device;
} E264Outputs;

/* Host-visible staging of one picture, handed out by the backend (pinned memory for the CUDA backend): the parser
 * writes records, levels and slice records straight into it; intra_list receives the addresses of the picture's intra
 * macroblocks in raster order (the device schedules them from it). */
typedef struct E264Staging {
	int32_t handle;
	uint32_t coef_capacity;       /* int16 entries in coefs */
	struct E264MbRec *recs;
	int16_t *coefs;
	struct E264SliceRec *slices;
	uint32_t *intra_list;
} E264Staging;

static inline int e264_blk_x(int b) { return ((b & 1) | ((b >> 1) & 2)); }          /* z-order -> 4x4 column */
static inline int e264_blk_y(int b) { return (((b >> 1) & 1) | ((b >> 2) & 2)); }   /* z-order -> 4x4 row    */
static inline int e264_blk_z(int x, int y) { return (x & 1) | ((y & 1) << 1) | ((x & 2) << 1) | ((y & 2) << 2); }

/* whether a prediction mode only reads neighbours its unavailability bits (A=1, B=2, D=8) allow (8.3.1.2, 8.3.2.2,
 * 8.3.3, 8.3.4); C is substituted when unavailable.  kind: MBK_I4x4 / MBK_I8x8 (mode 0..8), MBK_I16x16 (0..3), or
 * -1 for the chroma mode (0..3).  DC is legal for every availability. */
static inline int e264_intra_mode_legal(int kind, int mode, int un) {
	if (kind == MBK_I4x4 || kind == MBK_I8x8) {
		switch (mode) {
		case 0: case 3: case 7: return !(un & 2);
		case 1: case 8: return !(un & 1);
		case 2: return 1;
		case 4: case 5: case 6: return !(un & 11);
		default: return 0;
		}
	}
	if (kind == MBK_I16x16) return mode == 0 ? !(un & 2) : mode == 1 ? !(un & 1) : mode == 2 ? 1 : mode == 3 ? !(un & 11) : 0;
	return mode == 0 ? 1 : mode == 1 ? !(un & 1) : mode == 2 ? !(un & 2) : mode == 3 ? !(un & 11) : 0;
}

#endif
