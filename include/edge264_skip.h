/*
 * edge264_skip.h — skip unwanted pictures: a decoder mode that neither parses nor reconstructs non-reference or non-key
 * pictures.
 *
 * An extension of libedge264_b200.so that the reference's edge264.h does not have (that header and Edge264Frame stay as
 * the reference declares them).  Thumbnailers, scene indexers, seek previews and loaders that take one frame in N do not
 * need every picture; a skipped picture costs its slice headers and nothing else.
 *
 * Which pictures are skipped:
 *   EDGE264_SKIP_NONE    nothing (the default)
 *   EDGE264_SKIP_NONREF  every picture with nal_ref_idc == 0
 *   EDGE264_SKIP_NONKEY  every picture that is not IDR and whose first slice is not an I slice (slice_type % 5 != 2)
 *
 * Guarantees:
 *   - Every slice header of a skipped picture is parsed: new-picture detection, header errors and their return codes,
 *     picture order counts, frame_num, FrameId numbering (a skipped picture uses its FrameId), reference marking, frame_num
 *     gaps and output bumping go on exactly as in a full decode.  The decoded picture buffer evolves as in a full decode;
 *     only pixel work is left out.
 *   - The slice data of a skipped picture is never parsed; it takes no output buffer, nothing of it is sent to the GPU and
 *     it is never output.  edge264_decode_NAL returns 0 for its slices unless a header fails.  Its first slice may answer
 *     ENOBUFS when the output queue is full, like the first slice of any other picture.
 *   - The frames output are those of a full decode with the skipped pictures removed: the same FrameIds, the same samples,
 *     the same order, as long as no decoded picture predicts from a skipped one.
 *   - A skipped reference picture (EDGE264_SKIP_NONKEY) stays in the decoded picture buffer as a non-existing frame, like
 *     the frames of a frame_num gap, with the picture order count and frame_num of its header.  The first time the
 *     reference list of a decoded picture names it, its samples are filled with a constant and every macroblock of its
 *     error map with 100, before that picture is reconstructed.  A decoded picture that predicts from it is therefore
 *     defined, and Edge264Frame.mb_errors marks the macroblocks concerned.  Direct prediction sees it as non-existing.
 *     This happens with pictures whose first slice is I and later slices are not, and after a change of mode; the I
 *     pictures of a plain stream never predict from a skipped picture.
 *   - mb_errors, the motion export and the packed output are unchanged for decoded pictures.  With EDGE264_SKIP_NONE
 *     the decoder does exactly what it does without this call.
 */
#ifndef EDGE264_B200_SKIP_H
#define EDGE264_B200_SKIP_H

#include "edge264.h"

#ifdef __cplusplus
extern "C" {
#endif

enum { EDGE264_SKIP_NONE = 0, EDGE264_SKIP_NONREF = 1, EDGE264_SKIP_NONKEY = 2 };

/* Select which pictures to skip (EDGE264_SKIP_*).  It may be called at any time: the mode applies from the next picture
 * whose first slice arrives after the call, and a picture already started keeps the decision taken at its first slice.
 * Switching to a mode that decodes more pictures is allowed anywhere; switching at an IDR picture gives, from that picture
 * on, the frames of a full decode.  Returns 0, or EINVAL for a NULL decoder or an unknown mode. */
int edge264_set_skip(Edge264Decoder *dec, int mode);

#ifdef __cplusplus
}
#endif
#endif
