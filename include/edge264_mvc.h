/*
 * edge264_mvc.h — stereo (MVC) streams: both views reconstructed on the GPU, paired in one output frame.
 *
 * libedge264_b200.so decodes the Stereo High and Multiview High profiles with exactly two views, following the
 * reference's model of MVC:
 *   - Stereo decoding turns on when a subset sequence parameter set (NAL unit 15) is accepted, and off only at an End of
 *     sequence NAL unit (or edge264_flush).  A subset SPS with num_views != 2, of profile 134 (MFC High), whose frame
 *     format differs from its base view's SPS, or whose views do not fit in 32 frame slots (max_num_ref_frames > 15)
 *     answers ENOTSUP; the stream is then decoded as its base view alone.
 *   - Prefix NAL units (14) carry the base view's inter_view_flag; slices of the second view (NAL unit 20) are decoded
 *     with the subset SPS, their own frame_num, POC, reference marking, sliding window and frame_num gaps.
 *   - The second view predicts from its own view and from the base view of the same access unit, which is appended to
 *     its reference lists (modification_of_pic_nums_idc 4 and 5 name it).
 *   - Every view component takes a FrameId, in decoding order.
 *
 * Output (edge264_get_frame): a stereo frame is the pair (base view, second view) of one access unit, returned once both
 * are ready.  samples, FrameId and mb_errors describe the base view; samples_mvc and FrameId_mvc the second view.
 * return_arg covers both pictures, and edge264_return_frame releases both.  After an End of sequence, frames are single
 * view again (samples_mvc NULL).
 *
 * Modes: edge264_enable_luma_only applies to both views.  edge264_set_loop_filter decides per view component, a base view
 * with inter_view_flag 1 counting as a reference for EDGE264_LOOP_FILTER_REF.  edge264_set_skip decides per access unit,
 * at its base view, with the same count for EDGE264_SKIP_NONREF; the second view of a skipped access unit is skipped too.
 */
#ifndef EDGE264_B200_MVC_H
#define EDGE264_B200_MVC_H

#include "edge264.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The second view of `frame` (a frame returned by edge264_get_frame and still held) as a frame of its own: samples and
 * FrameId are the pair's samples_mvc and FrameId_mvc, mb_errors is the second view's error map, samples_mvc is NULL.
 * `out` can be passed to edge264_get_motion, edge264_get_packed and edge264_get_picstats while the pair is held; it is
 * released with the pair.  Returns 0, ENOENT for a single-view frame, or EINVAL for a NULL argument or a frame the
 * application does not hold. */
int edge264_get_second_view(Edge264Decoder *dec, const Edge264Frame *frame, Edge264Frame *out);

#ifdef __cplusplus
}
#endif
#endif
