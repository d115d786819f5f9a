/*
 * edge264_latency.h — low-latency output: a decoder mode that caps the output reorder depth and hands each frame out as
 * soon as the device has finished it.
 *
 * An extension of libedge264_b200.so that the reference's edge264.h does not have (that header and Edge264Frame stay as
 * the reference declares them).  By default a picture leaves the decoder by C.4.5.3 bumping with the stream's
 * max_num_reorder_frames, which a sequence parameter set without VUI bitstream_restriction infers from the level (up to
 * 16 frames, half a second at 30 fps, for the IPPP streams of many cameras), and edge264_get_frame answers ENOMSG while a
 * due picture is still on the device.  Live decoders (cameras, RTSP/WebRTC ingest, cloud gaming, conferencing) want each
 * frame as soon as it can be had, like FFmpeg's low_delay flag.
 *
 * Definition: decoding a stream with max_reorder = N is decoding its twin: the same bits, except that every SPS and
 * subset SPS carries VUI bitstream_restriction with max_num_reorder_frames = min(N, the value in force) and
 * max_dec_frame_buffering unchanged.  The decoded picture buffer evolves exactly as in the default decode: samples,
 * FrameIds, mb_errors, the motion export and the packed, resized and statistics outputs are unchanged; only the moment a
 * frame is handed out changes.  With a depth smaller than the stream needs, frames can leave out of POC order, as they
 * leave the twin.  The depth applies to each view; a stereo pair leaves once both views are due, as without the mode.
 *
 * While the mode is on (max_reorder >= 0), edge264_get_frame waits for a due frame whose picture is closed, first for the
 * worker threads still parsing it, then for the device, instead of answering ENOMSG.  A picture is closed once its slices
 * cover every macroblock (with worker threads, by the worker that parses the last of them), or by the next picture's first
 * slice, a flush or the end of the stream (a picture missing macroblocks is concealed as before).  A due picture still
 * open is never waited for: its next slices have not been passed in yet.  So ENOMSG means that no frame is due, or that the
 * due frame is still receiving slices.  Without worker threads, the frames each edge264_get_frame loop returns after an
 * edge264_decode_NAL are those the reference decoder returns on the twin stream after the same NAL unit.  With worker
 * threads, a picture's last slice may still be unparsed when the loop runs; its frame comes out no later than the loop
 * after the next picture's first NAL unit.  Pictures still reach the device strictly in decoding order.
 *
 * The mode combines with n_threads, alloc_cb, E264B_OUTPUT=device, edge264_set_skip, edge264_enable_luma_only,
 * edge264_set_loop_filter, stereo streams and every optional output.  With max_reorder = -1 the decoder does exactly what
 * it does without this call.
 */
#ifndef EDGE264_B200_LATENCY_H
#define EDGE264_B200_LATENCY_H

#include "edge264.h"

#ifdef __cplusplus
extern "C" {
#endif

/* max_reorder: -1 (the default) = the stream's own max_num_reorder_frames; 0..16 = at most that many.  It may be called at
 * any time: the setting applies from the next picture whose first slice arrives after the call, and a picture already
 * started keeps the depth read at its first slice.  Returns 0, or EINVAL for a NULL decoder or a value outside -1..16. */
int edge264_set_output_latency(Edge264Decoder *dec, int max_reorder);

#ifdef __cplusplus
}
#endif
#endif
