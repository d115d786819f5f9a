/*
 * edge264_loopfilter.h — skip the loop filter: a decoder mode that outputs non-reference (or all) pictures without
 * deblocking, and launches no deblocking for them.
 *
 * An extension of libedge264_b200.so that the reference's edge264.h does not have (that header and Edge264Frame stay as
 * the reference declares them).  The in-loop deblocking filter (8.7) is the costliest device work of a picture;
 * thumbnailers, detectors and indexers that do not need it can leave it out, like FFmpeg's skip_loop_filter.
 *
 * Which pictures are output unfiltered:
 *   EDGE264_LOOP_FILTER_ALL   none: every picture is filtered as the stream says (the default)
 *   EDGE264_LOOP_FILTER_REF   every picture with nal_ref_idc == 0; only reference pictures are filtered
 *   EDGE264_LOOP_FILTER_NONE  every picture
 *
 * Definition: a picture whose filter is skipped is output exactly as if every one of its slices had
 * disable_deblocking_filter_idc == 1, that is as the picture constructed before 8.7.  Nothing else about it changes:
 * its slice headers are parsed and checked as before (a bad filter offset is still an error), and the return codes,
 * FrameIds, output order, mb_errors and the motion export are those of a full decode.
 *
 * Guarantees:
 *   - EDGE264_LOOP_FILTER_REF causes no drift.  Every reference picture, and so every output frame of a reference
 *     picture, is byte-equal to the full decode's; every prediction reads what it reads in a full decode.  The frame of
 *     a non-reference picture is the full decode's picture before deblocking.
 *   - EDGE264_LOOP_FILTER_NONE drifts: later pictures predict from unfiltered references, so their frames differ from
 *     the full decode's by more than the filter.  It is meant for thumbnails and previews.
 *   - The packed, resized and picture-statistics outputs (edge264_packed.h, edge264_picstats.h) describe the frame as
 *     output, here the unfiltered one.
 *   - The mode combines with n_threads, alloc_cb (host or device memory), E264B_OUTPUT=device, edge264_set_skip,
 *     edge264_enable_luma_only and every optional output.  With EDGE264_LOOP_FILTER_ALL the decoder does exactly what it
 *     does without this call.
 */
#ifndef EDGE264_B200_LOOPFILTER_H
#define EDGE264_B200_LOOPFILTER_H

#include "edge264.h"

#ifdef __cplusplus
extern "C" {
#endif

enum { EDGE264_LOOP_FILTER_ALL = 0, EDGE264_LOOP_FILTER_REF = 1, EDGE264_LOOP_FILTER_NONE = 2 };

/* Select which pictures are output without the loop filter (EDGE264_LOOP_FILTER_*).  It may be called at any time: the
 * mode applies from the next picture whose first slice arrives after the call, and a picture already started keeps the
 * decision taken at its first slice.  Returns 0, or EINVAL for a NULL decoder or an unknown mode. */
int edge264_set_loop_filter(Edge264Decoder *dec, int mode);

#ifdef __cplusplus
}
#endif
#endif
