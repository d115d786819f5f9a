/*
 * e264b_recon.h — C ABI of the H100 (sm_90a) reconstruction runtime (the "thin shim" under the edge264 API).
 *
 * The reference has no separable interface here: its slice parser calls the pixel functions
 * in-process through static prototypes (reference edge264_internal.h:1349-1374: decode_intra4x4/8x8/
 * 16x16/Chroma, decode_inter, add_idct4x4/add_dc4x4/add_idct8x8, transform_dc4x4/dc2x2, deblock_mb).
 * These entry points replace that contract for a device backend: the host parser fills records
 * (edge264_b200/csrc/records.h) in pinned staging and submits whole pictures.  Plain pointers and
 * sizes only; every function returns 0 on success, -1 on a CUDA failure (message on stderr).
 *
 *   reference call sites replaced                         entry point
 *   per-MB decode_intra / decode_inter / add_idct calls   e264b_submit (one picture of records)
 *   (edge264_slice.c:466-664,881; edge264_mvpred.c:73-513)
 *   deblock_mb loop (edge264_slice.c:1816, headers.c:510,551)   e264b_submit (second kernel)
 *   alloc_frame / samples_buffers (edge264_headers.c:113-141)   e264b_configure, e264b_host_alloc
 *   next_deblock_addr == INT_MAX "frame complete" (edge264.c:373)   e264b_wait(ticket)
 */
#ifndef E264B_RECON_H
#define E264B_RECON_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

struct E264MbRec; struct E264SliceRec; struct E264PicDesc; struct E264Staging; struct E264Outputs; struct Edge264Decoder;
typedef struct E264bDevice E264bDevice;

int   e264b_create(E264bDevice **out);              /* device = $E264B_DEVICE (default 0); fails without a GPU */
void  e264b_destroy(E264bDevice *dev);
int   e264b_configure(E264bDevice *dev, const struct E264PicDesc *geometry, int n_slots);
void *e264b_host_alloc(E264bDevice *dev, size_t bytes);       /* pinned host memory */
void  e264b_host_free(E264bDevice *dev, void *p);
int   e264b_acquire_staging(E264bDevice *dev, int slot, struct E264Staging *out);   /* pinned areas the parser fills; out->handle goes back in E264PicDesc.staging */
void *e264b_pinned_alloc(E264bDevice *dev, size_t bytes);     /* pinned host memory, whatever E264B_OUTPUT says (error maps) */
void  e264b_pinned_free(E264bDevice *dev, void *p);
int   e264b_submit(E264bDevice *dev, const struct E264PicDesc *pic, uint8_t *host_out, uint64_t *ticket);
/* e264b_submit that also copies the picture's error map (one byte per macroblock) into host_map when pic->err_pic is set */
int   e264b_submit_maps(E264bDevice *dev, const struct E264PicDesc *pic, uint8_t *host_out, uint8_t *host_map, uint64_t *ticket);
/* e264b_submit_maps that also writes the picture's motion export (include/edge264_motion.h; layout E264_MOTION_* of
 * edge264_b200/csrc/records.h, 162 bytes per macroblock) into `motion`, host or device memory: slot_ids[s] is the FrameId
 * of frame slot s for s < n_ids (at most 32), -1 elsewhere; *on_device (if not NULL) tells whether `motion` is device
 * memory.  With motion NULL it is e264b_submit_maps: no launch, no copy. */
int   e264b_submit_motion(E264bDevice *dev, const struct E264PicDesc *pic, uint8_t *host_out, uint8_t *host_map, uint8_t *motion,
                          const int32_t *slot_ids, int n_ids, int *on_device, uint64_t *ticket);
/* The one submit the three above are thin callers of: `out` (struct E264Outputs of edge264_b200/csrc/records.h) names the
 * optional outputs, each left out when its pointer is NULL: the error map, the motion export, the packed output
 * (include/edge264_packed.h: the cropped picture as I420 or NV12, optionally box-downscaled, written by e264_pack_kernel,
 * or resized to out->pk's target size by exact area averaging, written by e264_resize_kernel; with the layout of
 * e264_packed_layout; one launch and one copy of that many bytes per picture), and the picture statistics
 * (include/edge264_picstats.h: histograms over out's cropping rectangle, per-macroblock sums and sums of squares, written
 * by e264_picstats_kernel with the layout E264_PICSTATS_*; one memset, one launch and one copy of
 * E264_PICSTATS_BYTES(nmb) bytes per picture). */
int   e264b_submit_outputs(E264bDevice *dev, const struct E264PicDesc *pic, uint8_t *host_out, const struct E264Outputs *out, uint64_t *ticket);
int   e264b_wait(E264bDevice *dev, uint64_t ticket);
int   e264b_poll(E264bDevice *dev, uint64_t ticket);          /* 0 complete, EAGAIN still on the device, < 0 device error */
int   e264b_fill_slot(E264bDevice *dev, int slot, int luma, int chroma);   /* and the slot's error map to all 100 */
int   e264b_slot_map(E264bDevice *dev, int slot, uint8_t *out);               /* a slot's error map (synchronous) */
int   e264b_error_flag(E264bDevice *dev);            /* 1 if a dependency wait timed out on the device */
void  e264b_stats(E264bDevice *dev, uint64_t *kernel_launches, uint64_t *h2d_bytes, uint64_t *d2h_bytes);

/* measurement support (bench.py): with $E264B_KEEP=1 every submitted picture's device-side records
 * are retained so the kernels can be re-run with inputs resident in HBM */
int      e264b_kept_count(E264bDevice *dev);
double   e264b_kept_algorithmic_bytes(E264bDevice *dev, double *recon_bytes, double *deblock_bytes, uint64_t *macroblocks);
typedef struct E264bReplayStats {
	float    ms_total;             /* device time from the common start to the last stream's end */
	int      threads;              /* host threads that issued the launches; 0: one CUDA graph per stream and repetition */
	uint64_t launches;             /* kernels executed in the timed region */
	double   kernel_ms[5];         /* per kernel kind (1 inter, 2 intra, 3 deblock; 0 and 4 unused): sum over launches of last-block-end minus first-block-start */
	uint64_t kernel_launches[5];
	int      inflight;             /* graph replay: streams with pictures on the GPU at a time */
	int      reserved;
} E264bReplayStats;
int      e264b_replay(E264bDevice **devs, int n, int reps, int threads, E264bReplayStats *stats);
uint64_t e264b_slot_hash(E264bDevice *dev, int slot);
int      e264b_slot_count(E264bDevice *dev);                  /* frame slots of the geometry last configured */
long long e264b_picture_bytes(E264bDevice *dev);              /* width x height x 3/2 */
int      e264b_replay_frames(E264bDevice *dev, uint8_t *out);  /* every kept picture once more, in decode order, into out */
/* known-answer support (tests): one block through the device's intra predictors (fn 0-3) or luma interpolation (fn 4) */
int      e264b_kat(int fn, int mode, const uint8_t *in, int in_bytes, uint8_t *out, int w, int h);
/* the intra predictors (fn 0-3) over n draws in one launch: modes[n], borders 66 bytes and out 256 bytes per draw (recon.cu) */
int      e264b_kat_batch(int fn, const uint8_t *modes, const uint8_t *borders, int n, uint8_t *out);
/* the kernels' residual_stage over n records (a warp each, luma-only instantiation when luma_only): levels at
 * pool[recs[i].coef_off], slices[recs[i].slice_idx]; out receives 384 int16 per record, Y 16x16 then Cb, Cr 8x8 (recon.cu) */
int      e264b_kat_residual(const struct E264MbRec *recs, int n, const struct E264SliceRec *slices, int n_slices, const int16_t *pool, int n_coefs, int luma_only, int16_t *out);
/* the inter kernel's window loads and interpolation over n draws (x, y, xFrac, yFrac) of a w x h plane: a 4x4 luma block
 * (16 bytes of out each) or, with chroma set, a 2x2 chroma block (4 bytes each) (recon.cu) */
int      e264b_kat_inter(int chroma, const uint8_t *plane, int stride, int w, int h, int bytes, const int32_t *draws, int n, uint8_t *out);
E264bDevice *e264b_of_decoder(struct Edge264Decoder *dec);

#ifdef __cplusplus
}
#endif
#endif
