/*
 * edge264_packed.h — packed output: each output frame cropped, as I420 or NV12, optionally box-downscaled by 2, 4 or 8,
 * or resized to any size by exact area averaging.
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
 * Resized output (edge264_enable_resized): the same planes resampled to a target size by exact area averaging.  For
 * each plane P of s_w x s_h cropped samples (chroma: half the luma size, as above) and its target of t_w x t_h samples
 * (chroma: half the luma target), output sample (x, y) covers [x s_w, (x + 1) s_w) x [y s_h, (y + 1) s_h) and source
 * sample (i, j) covers [i t_w, (i + 1) t_w) x [j t_h, (j + 1) t_h), in units of 1 / (t_w t_h) of a source sample.  With
 * the overlaps
 *
 *   a(x, i) = max(0, min((x + 1) s_w, (i + 1) t_w) - max(x s_w, i t_w)),   b(y, j) the same with s_h, t_h,
 *   N = sum over j, i of b(y, j) a(x, i) P[j][i],   D = s_w s_h,
 *   out[y][x] = floor((2 N + D) / (2 D))
 *
 * — one exact sum, rounded once, half up (N reaches about 2^36).  Only the source samples whose area overlaps the output
 * sample are read; in each row of that span only the first and the last can have a partial weight, every other weight is
 * t_w (vertically t_h).  t = s is a copy; when s = 2^k t on both axes the result is the packed output of log2_scale k,
 * byte for byte.  Enlarging is defined (each sample the overlap-weighted mean of at most 2 x 2 sources), so that a
 * fixed target holds when a stream shrinks below it; it is not a quality upscaler.  Edge264Packed then reports the
 * target as width x height, half of it as width_C x height_C, and log2_scale -1.
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
	int32_t format, log2_scale;  /* log2_scale -1: the resized output */
	int32_t on_device;          /* the planes are device memory (like the samples: E264B_OUTPUT=device, or an alloc_cb that
	                             * returns device memory), else host memory */
} Edge264Packed;

/* Pack every picture this decoder outputs as `format` (EDGE264_PACKED_*), downscaled by 1 << log2_scale (0..3).  Call it
 * after edge264_alloc and before the first slice: it returns 0, EBUSY once a slice has been decoded, EINVAL for a NULL
 * decoder, an unknown format or a scale outside 0..3, ENOTSUP when the library's backend has no packed output.  With an
 * alloc_cb, the decoder asks it for one more buffer per output frame (samples_size = the packed size, mbs_size 0) and
 * returns it through free_cb.  It may be combined with edge264_enable_motion. */
int edge264_enable_packed(Edge264Decoder *dec, int format, int log2_scale);

/* Pack every output picture as `format`, resampled to width x height luma samples by exact area averaging (the resized
 * output above).  The contract is edge264_enable_packed's: call it after edge264_alloc and before the first slice; it
 * returns 0, EBUSY once a slice has been decoded, EINVAL for a NULL decoder, an unknown format, an odd or negative size,
 * a size above 16384 or both sizes 0, ENOTSUP when the library's backend has no packed output.  A decoder has one packed
 * output: this call and edge264_enable_packed each replace the setting of the other.  One of width / height may be 0:
 * it is then derived for each sequence from the cropped picture s_w x s_h as the nearest even size that keeps the aspect
 * ratio, t_w = min(16384, max(2, 2 floor((s_w t_h + s_h) / (2 s_h)))) (and symmetrically t_h).  With both given, every
 * frame of every sequence has that shape, also after a size change.  The frames come out through edge264_get_packed;
 * the buffer's memory kind, lifetime and alloc_cb calls are those of edge264_enable_packed. */
int edge264_enable_resized(Edge264Decoder *dec, int format, int width, int height);

/* The packed picture of a frame just returned by edge264_get_frame, with the dimensions of that frame.  It stays valid
 * exactly as long as the frame's samples: until the next edge264_decode_NAL, or until edge264_return_frame when the frame
 * was borrowed.  Returns 0, ENOENT when packed output is not enabled, EINVAL when the frame is not one the application
 * currently holds. */
int edge264_get_packed(Edge264Decoder *dec, const Edge264Frame *frame, Edge264Packed *out);

#ifdef __cplusplus
}
#endif
#endif
