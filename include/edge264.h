/*
 * edge264.h — C ABI of the H100-native H.264 reconstruction backend.
 *
 * This header declares the SAME seven entry points and the SAME Edge264Frame
 * layout (96 bytes on LP64) as the reference decoder's public header
 * (reference: edge264.h:38-70), so that an application built against the
 * reference links against libedge264_b200.so unchanged.  Only the declarations
 * are shared with the reference; everything behind them is new code:
 * the CPU parses the bitstream into per-macroblock records and sm_90a CUDA
 * kernels reconstruct the pixels (see DESIGN.md).
 *
 *   reference interface                       replaced by (this library)
 *   edge264_find_start_code  edge264.c:87     src: edge264_b200/csrc/decoder.c
 *   edge264_alloc            edge264.c:142    idem (n_threads is accepted, ignored: GPU backend)
 *   edge264_flush            edge264.c:261    idem
 *   edge264_free             edge264.c:273    idem
 *   edge264_decode_NAL       edge264.c:296    idem (same errno return codes)
 *   edge264_get_frame        edge264.c:365    idem (frame pixels are a pinned host mirror)
 *   edge264_return_frame     edge264.c:411    idem
 */
#ifndef EDGE264_B200_PUBLIC_H
#define EDGE264_B200_PUBLIC_H

#include <errno.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct Edge264Decoder Edge264Decoder;

/* callbacks (reference edge264.h:40-43) */
typedef int  (*Edge264LogCb)(const char *str, void *log_arg);
typedef void (*Edge264UnrefCb)(int ret, void *unref_arg);
typedef void (*Edge264AllocCb)(void **samples, unsigned samples_size, void **mbs, unsigned mbs_size,
                               int errno_on_fail, void *alloc_arg);
typedef void (*Edge264FreeCb)(void *samples, void *mbs, void *alloc_arg);

/* One output picture (reference edge264.h:45-62).  Field order and widths are ABI. */
typedef struct Edge264Frame {
	const uint8_t *samples[3];      /* Y, Cb, Cr; already offset by the cropping rectangle   */
	const uint8_t *samples_mvc[3];  /* second view of a stereo frame (edge264_mvc.h), else NULL */
	const uint8_t *mb_errors;       /* NULL when no macroblock can be wrong, else 0..100 per macroblock of the coded
	                                 * picture, row y at mb_errors + y * stride_mb (= width in macroblocks); pinned
	                                 * host memory, valid as long as the samples */
	int8_t  bit_depth_Y;
	int8_t  bit_depth_C;
	int16_t width_Y;
	int16_t width_C;
	int16_t height_Y;
	int16_t height_C;
	int16_t stride_Y;               /* bytes between luma rows                                */
	int16_t stride_C;               /* bytes between two Cb rows (a Cr row sits in between)   */
	int16_t stride_mb;
	int32_t FrameId;
	int32_t FrameId_mvc;            /* FrameId of the second view, when samples_mvc is set    */
	int16_t frame_crop_offsets[4];  /* {top,right,bottom,left} in luma samples                */
	void   *return_arg;             /* pass to edge264_return_frame when borrowed             */
} Edge264Frame;

const uint8_t  *edge264_find_start_code(const uint8_t *buf, const uint8_t *end, int four_byte);
Edge264Decoder *edge264_alloc(int n_threads, Edge264LogCb log_cb, void *log_arg, int log_mbs,
                              Edge264AllocCb alloc_cb, Edge264FreeCb free_cb, void *alloc_arg);
void edge264_flush(Edge264Decoder *dec);
void edge264_free(Edge264Decoder **pdec);
int  edge264_decode_NAL(Edge264Decoder *dec, const uint8_t *buf, const uint8_t *end,
                        Edge264UnrefCb unref_cb, void *unref_arg);
int  edge264_get_frame(Edge264Decoder *dec, Edge264Frame *out, int borrow);
void edge264_return_frame(Edge264Decoder *dec, void *return_arg);

#ifdef __cplusplus
}
#endif
#endif
