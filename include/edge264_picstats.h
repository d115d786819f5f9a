/*
 * edge264_picstats.h — picture statistics: each output frame's histograms, and per-macroblock sums and sums of squares.
 *
 * An extension of libedge264_b200.so that the reference's edge264.h does not have (that header and Edge264Frame stay as
 * the reference declares them).  Tools that analyse video rather than display it (scene-cut and blank-frame detection,
 * perceptual hashing, background subtraction, OCR, PSNR-Y) first ask simple questions of each frame: its histogram, how
 * bright and how textured each region is.  A kernel of the decoder (e264_picstats_kernel) answers them when the picture
 * is reconstructed, from the picture already on the GPU, so that no application has to read every sample again.
 * "picstats" is not the runtime's e264b_stats (launch and byte counters).
 *
 * Definition.  Y, Cb and Cr are the coded planes of the frame: reached from Edge264Frame.samples[] by moving back over
 * frame_crop_offsets (chroma by half the luma offsets), Cr rows alternating with Cb rows as Edge264Frame lays them out.
 * W = width_mbs and H = height_mbs are the coded picture size in macroblocks, the grid of Edge264Frame.mb_errors and of
 * edge264_motion.h.
 *
 *   hist    uint32 [3][256]   hist[p][v]: the number of samples equal to v in the CROPPED plane p (Y, Cb, Cr):
 *                             width_Y x height_Y samples for Y, width_C x height_C for each of Cb and Cr.  Cropped-away
 *                             and padding samples are not counted.
 *   sum     uint32 [3][H][W]  the sum of the samples of each CODED macroblock: its 16x16 Y samples, 8x8 Cb, 8x8 Cr
 *   sum_sq  uint32 [3][H][W]  the sum of the squares of the same samples
 *
 * The per-macroblock arrays cover the coded grid, so they line up with mb_errors and the motion export; the histogram
 * describes the picture the viewer sees (the 8 rows 1080p streams crop away would bias a blank-frame test).  Bounds:
 * sum <= 65 280, sum_sq <= 16 646 400, a bin <= 16384 * 16384: all fit in uint32.  Two invariants hold on every frame:
 *   - for each plane p, the bins of hist[p] add up to that plane's cropped sample count;
 *   - without cropping, the sum over v of v * hist[0][v] equals the sum of sum[0].
 * The statistics are a function of the frame's own planes alone: the same on every backend, thread count and output
 * order, never those of the packed or resized output (edge264_packed.h).  With luma-only decoding (edge264_luma.h) the
 * chroma statistics are those of a plane of 128.
 *
 * Layout: one buffer per output frame of 3072 + 24 W H bytes: hist at offset 0, sum at 3072, sum_sq at 3072 + 12 W H.
 */
#ifndef EDGE264_B200_PICSTATS_H
#define EDGE264_B200_PICSTATS_H

#include "edge264.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct Edge264PicStats {
	const uint32_t *hist;           /* [3][256]  */
	const uint32_t *sum;            /* [3][H][W] */
	const uint32_t *sum_sq;         /* [3][H][W] */
	int32_t width_mbs, height_mbs;
	int32_t on_device;              /* the arrays are device memory (like the samples: E264B_OUTPUT=device, or an alloc_cb that
	                                 * returns device memory), else host memory */
} Edge264PicStats;

/* Compute the statistics of every picture this decoder outputs.  Call it after edge264_alloc and before the first slice:
 * it returns 0, EBUSY once a slice has been decoded, EINVAL for a NULL decoder, ENOTSUP when the library's backend has no
 * statistics.  With an alloc_cb, the decoder asks it for one more buffer per output frame, after the packed one
 * (samples_size = 3072 + 24 bytes per macroblock, mbs_size 0) and returns it through free_cb.  It combines with n_threads,
 * E264B_OUTPUT=device, edge264_set_skip, edge264_enable_luma_only, edge264_enable_motion, edge264_enable_packed and
 * edge264_enable_resized. */
int edge264_enable_picstats(Edge264Decoder *dec);

/* The statistics of a frame just returned by edge264_get_frame.  They stay valid exactly as long as the frame's samples:
 * until the next edge264_decode_NAL, or until edge264_return_frame when the frame was borrowed.  Returns 0, ENOENT when
 * the statistics are not enabled, EINVAL when the frame is not one the application currently holds. */
int edge264_get_picstats(Edge264Decoder *dec, const Edge264Frame *frame, Edge264PicStats *out);

#ifdef __cplusplus
}
#endif
#endif
