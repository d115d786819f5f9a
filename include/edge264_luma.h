/*
 * edge264_luma.h — luma-only decoding: a decoder mode whose kernels reconstruct and deblock only the Y plane.
 *
 * An extension of libedge264_b200.so that the reference's edge264.h does not have (that header and Edge264Frame stay as
 * the reference declares them).  Consumers that analyse video rather than display it often read luma alone: scene-cut
 * and blank-frame detection, perceptual hashing, background subtraction, feature tracking, OCR, PSNR-Y / SSIM-Y.  In
 * 4:2:0 8-bit decoding no luma sample depends on chroma (intra and inter luma prediction read luma, boundary strengths
 * read luma coded bits, the luma filters read luma), so the chroma work can be left out and the Y plane stays exact.
 * The chroma syntax elements are still parsed (the entropy decoder has to, to reach the next macroblock); their levels
 * are dropped before they reach the GPU.
 *
 * Guarantees, against a full decode of the same stream with the same settings:
 *   - Every output frame has the same FrameId, order, sizes, strides, cropping and return_arg, and every
 *     edge264_decode_NAL return code is the same.
 *   - samples[0]: every sample inside width_Y x height_Y is equal.
 *   - The chroma plane: every Cb and Cr sample inside width_C x height_C is 128.  The layout is unchanged: samples[1]
 *     and samples[2] point into one plane whose rows alternate Cb and Cr.
 *   - mb_errors and the motion export (edge264_motion.h) are equal.
 *   - The packed and resized outputs (edge264_packed.h) follow their definitions over these planes: their Y plane is
 *     equal, their chroma planes are 128 (box or area averaging of a constant is that constant).
 *   - The mode combines with n_threads, alloc_cb (host or device memory), E264B_OUTPUT=device, edge264_set_skip,
 *     edge264_enable_motion, edge264_enable_packed and edge264_enable_resized.
 *   - Without the call the decoder does exactly what it does without this header.
 * 4:0:0 (monochrome) streams are not supported by this mode either: they still answer ENOTSUP.
 */
#ifndef EDGE264_B200_LUMA_H
#define EDGE264_B200_LUMA_H

#include "edge264.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Decode every picture of this decoder with luma only (see the guarantees above).  Call it after edge264_alloc and
 * before the first slice.  Returns 0, EBUSY once a slice has been decoded, EINVAL for a NULL decoder. */
int edge264_enable_luma_only(Edge264Decoder *dec);

#ifdef __cplusplus
}
#endif
#endif
