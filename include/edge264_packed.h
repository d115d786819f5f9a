/*
 * edge264_packed.h — packed output: each output frame cropped, as I420 or NV12, optionally box-downscaled by 2, 4 or 8.
 *
 * An extension of libedge264_b200.so that the reference's edge264.h does not have (that header and Edge264Frame stay as
 * the reference declares them).  Edge264Frame is the reference's layout: padded planes, Cb and Cr rows alternating in one
 * chroma plane, the cropping rectangle as pointer offsets.  This is the same picture in the layout GPU consumers take
 * (encoders, image libraries, tensors), written by a kernel of the decoder (e264_pack_kernel) when the picture is
 * reconstructed, so that no application has to repack, and a reduced picture never costs a full-size copy.
 *
 * Definition.  Let Y, Cb, Cr be the cropped planes exactly as Edge264Frame.samples[], width_Y / height_Y and
 * width_C / height_C describe them, k = log2_scale, n = 1 << k.  For each plane P of w x h samples the output plane has
 * ceil(w / n) x ceil(h / n) samples,
 *
 *   out[y][x] = (sum over dy, dx in 0..n-1 of P[min(y n + dy, h - 1)][min(x n + dx, w - 1)] + (n n >> 1)) >> (2 k)
 *
 * — one exact box sum with one rounding (not a cascade of 2x2 averages), the last row and column replicated inside the
 * cropped picture; cropped-away and padding samples are never read.  k = 0 is a copy.
 *
 * Cropped luma sizes are even (4:2:0 frames), therefore width_C == ceil(width / 2) and height_C == ceil(height / 2) for
 * every k: NV12 consumers may rely on it.
 *
 * Layout: one buffer.  stride[i] is the plane's row bytes (NV12's CbCr row: 2 * width_C) rounded up to a multiple of
 * 64; every plane starts on a multiple of 256 bytes from planes[0].  Padding bytes are unspecified.
 */
#ifndef EDGE264_B200_PACKED_H
#define EDGE264_B200_PACKED_H

#include "edge264.h"

#ifdef __cplusplus
extern "C" {
#endif

enum { EDGE264_PACKED_I420 = 0, EDGE264_PACKED_NV12 = 1 };

typedef struct Edge264Packed {
	const uint8_t *planes[3];   /* I420: Y, Cb, Cr.  NV12: Y, interleaved CbCr, NULL */
	int32_t stride[3];          /* bytes between rows of each plane (0 for the absent one) */
	int32_t width, height;      /* luma samples, after cropping and scaling */
	int32_t width_C, height_C;  /* chroma samples per component */
	int32_t format, log2_scale;
	int32_t on_device;          /* the planes are device memory (like the samples: E264B_OUTPUT=device, or an alloc_cb that
	                             * returns device memory), else host memory */
} Edge264Packed;

/* Pack every picture this decoder outputs as `format` (EDGE264_PACKED_*), downscaled by 1 << log2_scale (0..3).  Call it
 * after edge264_alloc and before the first slice: it returns 0, EBUSY once a slice has been decoded, EINVAL for a NULL
 * decoder, an unknown format or a scale outside 0..3, ENOTSUP when the library's backend has no packed output.  With an
 * alloc_cb, the decoder asks it for one more buffer per output frame (samples_size = the packed size, mbs_size 0) and
 * returns it through free_cb.  It may be combined with edge264_enable_motion. */
int edge264_enable_packed(Edge264Decoder *dec, int format, int log2_scale);

/* The packed picture of a frame just returned by edge264_get_frame, with the dimensions of that frame.  It stays valid
 * exactly as long as the frame's samples: until the next edge264_decode_NAL, or until edge264_return_frame when the frame
 * was borrowed.  Returns 0, ENOENT when packed output is not enabled, EINVAL when the frame is not one the application
 * currently holds. */
int edge264_get_packed(Edge264Decoder *dec, const Edge264Frame *frame, Edge264Packed *out);

#ifdef __cplusplus
}
#endif
#endif
