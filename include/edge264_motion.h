/*
 * edge264_motion.h — motion export: each output frame's motion field, reference FrameIds, macroblock types and QPs.
 *
 * An extension of libedge264_b200.so that the reference's edge264.h does not have (that header and Edge264Frame stay as
 * the reference declares them).  The values are those reconstruction used, derived on the GPU from the decoder's
 * per-macroblock records, for the coded picture (not cropped), like Edge264Frame.mb_errors:
 *
 *   mv            int16 [2][4 H][4 W][2]  per list and 4x4 block, raster order: (x, y) in quarter samples;
 *                                         (0, 0) where the list is not used
 *   ref_frame_id  int32 [2][2 H][2 W]     per list and 8x8 block: FrameId of the picture the block predicts from;
 *                                         -1 where the list is not used or the macroblock is intra
 *   mb_type       uint8 [H][W]            EDGE264_MB_*
 *   mb_qp         uint8 [H][W]            QP_Y (0 for I_PCM)
 *
 * with W = width_mbs, H = height_mbs.  Where a damaged stream made the decoder substitute a reference picture, ref_frame_id
 * names the picture actually used; concealed macroblocks report the record they were reconstructed from (a P_Skip copy
 * of the most recent reference, or Intra16x16 DC) and Edge264Frame.mb_errors marks them 100.
 */
#ifndef EDGE264_B200_MOTION_H
#define EDGE264_B200_MOTION_H

#include "edge264.h"

#ifdef __cplusplus
extern "C" {
#endif

enum { EDGE264_MB_I4x4 = 0, EDGE264_MB_I8x8 = 1, EDGE264_MB_I16x16 = 2, EDGE264_MB_IPCM = 3, EDGE264_MB_INTER = 4, EDGE264_MB_SKIP = 5 };

typedef struct Edge264Motion {
	const int16_t *mv;
	const int32_t *ref_frame_id;
	const uint8_t *mb_type;
	const uint8_t *mb_qp;
	int32_t width_mbs, height_mbs;
	int32_t on_device;              /* the arrays are device memory (like the samples: E264B_OUTPUT=device, or an alloc_cb that
	                                 * returns device memory), else host memory */
} Edge264Motion;

/* Export the motion of every picture this decoder outputs.  Call it after edge264_alloc and before the first slice: it
 * returns 0, EBUSY once a slice has been decoded, ENOTSUP when the library's backend has no export.  With an alloc_cb,
 * the decoder asks it for one more buffer per output frame (samples_size = 162 bytes per macroblock, mbs_size 0) and
 * returns it through free_cb. */
int edge264_enable_motion(Edge264Decoder *dec);

/* The export of a frame just returned by edge264_get_frame.  It stays valid exactly as long as the frame's samples: until
 * the next edge264_decode_NAL, or until edge264_return_frame when the frame was borrowed.  Returns 0, ENOENT when the
 * export is not enabled, EINVAL when the frame is not one the application currently holds. */
int edge264_get_motion(Edge264Decoder *dec, const Edge264Frame *frame, Edge264Motion *out);

#ifdef __cplusplus
}
#endif
#endif
