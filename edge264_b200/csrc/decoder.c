/* decoder.c — the edge264 C API over the record-producing parser and a reconstruction backend.
 *
 * Host-side counterpart of the reference's edge264.c + edge264_headers.c (reference: API
 * edge264.c:87-415; SPS/PPS/slice header/POC/ref lists/MMCO/bumping edge264_headers.c:61-141,
 * 611-1290, 1343-2059).  Everything is re-implemented from ITU-T H.264 with the reference's
 * observable behaviour (return codes, output order, frame layout, FrameId numbering) as the
 * contract; no pixel is touched here: pictures are handed to the backend as records.
 */
#define _GNU_SOURCE
#include <errno.h>
#include <limits.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>
#include "dec.h"
#include "h264_tables.h"
#include "../../include/edge264_motion.h"
#include "../../include/edge264_packed.h"
#include "../../include/edge264_picstats.h"
#include "../../include/edge264_skip.h"
#include "../../include/edge264_luma.h"
#include "../../include/edge264_loopfilter.h"
#include "../../include/edge264_mvc.h"
#include "../../include/edge264_latency.h"

/* optional host-side time accounting (E264_HOST_PROFILE=1): where decode_NAL/get_frame spend their time */
#include <time.h>
static int prof_on = -1;
static double prof_t[6]; static long prof_n[6];
static const char *const prof_names[6] = {"parse_slice_data", "acquire_staging", "submit", "wait", "clear_mbinfo", "headers+dpb"};
static inline double prof_now(void) { struct timespec t; clock_gettime(CLOCK_MONOTONIC, &t); return t.tv_sec + 1e-9 * t.tv_nsec; }
#define PROF_BEGIN double prof_t0_ = prof_on > 0 ? prof_now() : 0
#define PROF_END(i) do { if (prof_on > 0) { prof_t[i] += prof_now() - prof_t0_; prof_n[i]++; } } while (0)

/* ------------------------------------------------------------------------------------------ */
/* start codes (reference edge264.c:87-119: returns a pointer to the 00 00 01 / 00 00 00 01)     */
/* ------------------------------------------------------------------------------------------ */
const uint8_t *edge264_find_start_code(const uint8_t *buf, const uint8_t *end, int four_byte) {
	four_byte = four_byte != 0;
	const uint8_t *p = buf + four_byte;   /* the reference searches a 001 from buf+four_byte and backs up */
	if (p >= end) return end;
	for (;;) {
		/* find next 0x01 at or after p+2 (position of the '1' of a 001 that starts at >= p) */
		const uint8_t *s = p + 2;
		if (s >= end) return end;
		const uint8_t *one = (const uint8_t *)memchr(s, 1, (size_t)(end - s));
		if (!one) return end;
		if (one[-1] == 0 && one[-2] == 0) {
			const uint8_t *res = one - 2 - four_byte;
			if (*res == 0) return res < end ? res : end;
		}
		p = one - 1;   /* continue after this 0x01: next candidate '1' position is > one */
		if (p + 2 <= one) p = one - 1;
	}
}

/* ------------------------------------------------------------------------------------------ */
/* parameter sets                                                                               */
/* ------------------------------------------------------------------------------------------ */
static const uint32_t max_dpb_mbs_by_level[64] = {   /* Table A-1 MaxDpbMbs, indexed by level_idc */
	396, 396, 396, 396, 396, 396, 396, 396, 396, 396, 396, 900, 2376, 2376, 2376, 2376, 2376, 2376, 2376, 2376, 2376,
	4752, 8100, 8100, 8100, 8100, 8100, 8100, 8100, 8100, 8100, 18000, 20480, 32768, 32768, 32768, 32768, 32768, 32768,
	32768, 32768, 32768, 34816, 110400, 110400, 110400, 110400, 110400, 110400, 110400, 110400, 184320, 184320,
	696320, 696320, 696320, 696320, 696320, 696320, 696320, 696320, 696320, 696320, 0xffffffffu};

/* scaling_list(): returns 0 = explicit list written to dst (raster), 1 = useDefaultScalingMatrixFlag */
static int parse_scaling_list(BitReader *b, uint8_t *dst, int n, const uint8_t *scan) {
	int last = 8, next = 8;
	for (int j = 0; j < n; j++) {
		if (next != 0) {
			int delta = br_se(b);
			next = (last + delta + 256) & 255;
			if (j == 0 && next == 0) return 1;
		}
		dst[scan[j]] = (uint8_t)(next == 0 ? last : next);
		last = dst[scan[j]];
	}
	return 0;
}

/* The reference keeps not-transmitted PPS lists as zeros and substitutes the SPS lists at slice time
 * (reference headers.c:903-915, 1343-1413); we reproduce exactly that observable behaviour:
 *  lists: 6 of 4x4 then 2 of 8x8; `w4`/`w8` hold the fall-back values on entry. */
static void parse_scaling_lists(BitReader *b, uint8_t w4[6][16], uint8_t w8[2][64], int with8x8) {
	uint8_t fb[16]; memcpy(fb, w4[0], 16);
	const uint8_t *def = h264_default4x4_intra;
	for (int i = 0; i < 6; i++) {
		if (i == 3) { memcpy(fb, w4[3], 16); def = h264_default4x4_inter; }
		if (!br_u1(b)) memcpy(w4[i], fb, 16);
		else {
			if (parse_scaling_list(b, w4[i], 16, h264_zigzag4x4)) memcpy(w4[i], def, 16);
			memcpy(fb, w4[i], 16);
		}
	}
	if (!with8x8) return;
	for (int i = 0; i < 2; i++) {
		if (!br_u1(b)) continue;
		if (parse_scaling_list(b, w8[i], 64, h264_zigzag8x8)) memcpy(w8[i], i ? h264_default8x8_inter : h264_default8x8_intra, 64);
	}
}

static void skip_hrd(BitReader *b) {
	int cpb_cnt = br_ue_i(b, 32) + 1;
	br_u(b, 8);
	for (int i = 0; i < cpb_cnt && i < 32; i++) { br_ue(b); br_ue(b); br_u1(b); }
	br_u(b, 20);
}

/* mvc_vui_parameters_extension (H.14.1): walked over, like the reference (headers.c:1699-1736) */
static void skip_mvc_vui(BitReader *b) {
	for (int i = br_ue_i(b, 1023); i-- >= 0 && !b->overrun;) {
		br_u(b, 3);
		for (int j = br_ue_i(b, 1023); j >= 0 && !b->overrun; j--) br_ue(b);
		if (br_u1(b)) { br_u(b, 32); br_u(b, 32); br_u1(b); }
		int nal_hrd = br_u1(b); if (nal_hrd) skip_hrd(b);
		int vcl_hrd = br_u1(b); if (vcl_hrd) skip_hrd(b);
		if (nal_hrd || vcl_hrd) br_u1(b);
		br_u1(b);
	}
}

/* seq_parameter_set_mvc_extension (H.7.3.2.1.4): exactly two views; the inter-view references it lists are ignored, the
 * second view always predicts from its base (reference headers.c:1743-1790).  0 or ENOTSUP. */
static int parse_sps_mvc_extension(BitReader *b, int profile_idc) {
	int num_views = br_ue_i(b, 1023) + 1;
	for (int i = 0; i < num_views && !b->overrun; i++) br_ue(b);
	if (num_views != 2) return ENOTSUP;
	for (int k = 0; k < 4; k++) if (br_ue_i(b, 2)) br_ue(b);   /* anchor l0/l1, then non-anchor l0/l1 references of view 1 */
	for (int i = br_ue_i(b, 63); i >= 0 && !b->overrun; i--) {   /* level values and their operation points */
		br_u(b, 8);
		for (int j = br_ue_i(b, 1023); j >= 0 && !b->overrun; j--) {
			br_u(b, 3);
			for (int k = br_ue_i(b, 1023); k >= 0 && !b->overrun; k--) br_ue(b);
			br_ue(b);
		}
	}
	return profile_idc == 134 ? ENOTSUP : 0;   /* MFC High */
}

/* subset: a subset sequence parameter set (NAL unit 15), whose MVC extension follows the SPS data */
static int parse_sps(Edge264Decoder *d, BitReader *b, SPS *out, int subset) {
	SPS s; memset(&s, 0, sizeof(s));
	int ret = 0;
	memset(s.sl4x4, 16, sizeof(s.sl4x4)); memset(s.sl8x8, 16, sizeof(s.sl8x8));
	s.profile_idc = br_u(b, 8); s.constraint_flags = br_u(b, 8); s.level_idc = br_u(b, 8);
	br_ue(b);   /* seq_parameter_set_id: ignored like the reference (headers.c:1851) */
	s.log2_max_poc_lsb = 16;
	if (s.profile_idc != 66 && s.profile_idc != 77 && s.profile_idc != 88) {
		int chroma_format_idc = br_ue_i(b, 4);
		if (chroma_format_idc != 1) { ret = ENOTSUP; if (chroma_format_idc == 3) br_u1(b); }
		if (br_ue(b) != 0) ret = ENOTSUP;   /* bit_depth_luma_minus8 */
		if (br_ue(b) != 0) ret = ENOTSUP;
		if (br_u1(b)) ret = ENOTSUP;        /* qpprime_y_zero_transform_bypass_flag */
		if (br_u1(b)) {                     /* seq_scaling_matrix_present_flag */
			s.scaling_present = 1;
			memcpy(s.sl4x4[0], h264_default4x4_intra, 16); memcpy(s.sl4x4[3], h264_default4x4_inter, 16);
			memcpy(s.sl8x8[0], h264_default8x8_intra, 64); memcpy(s.sl8x8[1], h264_default8x8_inter, 64);
			if (chroma_format_idc == 3) return ENOTSUP;
			parse_scaling_lists(b, s.sl4x4, s.sl8x8, 1);
		}
	}
	s.log2_max_frame_num = br_ue_i(b, 13) + 4;
	s.poc_type = br_ue_i(b, 3);
	if (s.log2_max_frame_num > 16 || s.poc_type > 2) return EBADMSG;
	if (s.poc_type == 0) { s.log2_max_poc_lsb = br_ue_i(b, 13) + 4; if (s.log2_max_poc_lsb > 16) return EBADMSG; }
	else if (s.poc_type == 1) {
		s.delta_pic_order_always_zero_flag = br_u1(b);
		s.offset_for_non_ref_pic = br_se(b);
		s.offset_for_top_to_bottom_field = br_se(b);
		s.num_ref_frames_in_poc_cycle = br_ue_i(b, 256);
		if (s.num_ref_frames_in_poc_cycle > 255) return EBADMSG;
		for (int i = 0; i < s.num_ref_frames_in_poc_cycle; i++) s.offset_for_ref_frame[i] = br_se(b);
	}
	int max_num_ref_frames = br_ue_i(b, 17);
	s.gaps_allowed = br_u1(b);
	s.width_mbs = br_ue_i(b, 4096) + 1;
	s.height_mbs = br_ue_i(b, 4096) + 1;
	if (s.width_mbs > E264_MAX_WIDTH_MBS || s.height_mbs > 1055 || max_num_ref_frames > 16) return EBADMSG;
	int frame_mbs_only = br_u1(b);
	if (!frame_mbs_only) { ret = ENOTSUP; br_u1(b); }
	s.direct_8x8_inference = br_u1(b);
	unsigned lvl = s.level_idc < 63 ? s.level_idc : 63;
	int max_dpb_frames = (int)(max_dpb_mbs_by_level[lvl] / (unsigned)(s.width_mbs * s.height_mbs));
	if (max_dpb_frames > 16) max_dpb_frames = 16;
	s.max_num_ref_frames = max_num_ref_frames < max_dpb_frames ? max_num_ref_frames : max_dpb_frames;
	int intra_profile = (s.profile_idc == 44 || s.profile_idc == 86 || s.profile_idc == 100 || s.profile_idc == 110 ||
	                     s.profile_idc == 122 || s.profile_idc == 244) && (s.constraint_flags & (1 << 4));
	if (intra_profile) { s.max_num_reorder_frames = 0; s.max_dec_frame_buffering = s.max_num_ref_frames; }
	else s.max_num_reorder_frames = s.max_dec_frame_buffering = max_dpb_frames;
	if (br_u1(b)) {   /* frame_cropping_flag; 4:2:0 frame: units of 2 luma samples */
		/* out-of-range offsets are clamped, not rejected, like the reference's bounded get_ue16 (headers.c:1975-1983) */
		int limx = s.width_mbs * 8 - 1, limy = s.height_mbs * 8 - 1;
		int v = br_ue_i(b, 1 << 20); s.crop[0] = (v < 0 || v > limx ? limx : v) * 2;
		v = br_ue_i(b, 1 << 20); s.crop[1] = (v < 0 || v > limx - s.crop[0] / 2 ? limx - s.crop[0] / 2 : v) * 2;
		v = br_ue_i(b, 1 << 20); s.crop[2] = (v < 0 || v > limy ? limy : v) * 2;
		v = br_ue_i(b, 1 << 20); s.crop[3] = (v < 0 || v > limy - s.crop[2] / 2 ? limy - s.crop[2] / 2 : v) * 2;
	}
	if (br_u1(b)) {   /* vui_parameters (E.1.1): walked only to reach bitstream_restriction */
		if (br_u1(b)) { if (br_u(b, 8) == 255) { br_u(b, 16); br_u(b, 16); } }
		if (br_u1(b)) br_u1(b);
		if (br_u1(b)) { br_u(b, 4); if (br_u1(b)) br_u(b, 24); }
		if (br_u1(b)) { br_ue(b); br_ue(b); }
		if (br_u1(b)) { br_u(b, 32); br_u(b, 32); br_u1(b); }
		int nal_hrd = br_u1(b); if (nal_hrd) skip_hrd(b);
		int vcl_hrd = br_u1(b); if (vcl_hrd) skip_hrd(b);
		if (nal_hrd || vcl_hrd) br_u1(b);
		br_u1(b);   /* pic_struct_present_flag */
		if (br_u1(b)) {
			br_u1(b); br_ue(b); br_ue(b); br_ue(b); br_ue(b);
			int reorder = br_ue_i(b, 17), buffering = br_ue_i(b, 17);
			if (reorder > 16 || buffering > 16) return EBADMSG;
			s.max_dec_frame_buffering = buffering > s.max_num_ref_frames ? buffering : s.max_num_ref_frames;
			s.max_num_reorder_frames = reorder < s.max_dec_frame_buffering ? reorder : s.max_dec_frame_buffering;
		}
	}
	if (subset) {   /* Multiview High and Stereo High only (reference headers.c:2002-2009) */
		if (s.profile_idc != 118 && s.profile_idc != 128 && s.profile_idc != 134) return ENOTSUP;
		br_u1(b);   /* bit_equal_to_one */
		int r = parse_sps_mvc_extension(b, s.profile_idc);
		if (r) return r;
		if (br_u1(b)) skip_mvc_vui(b);
		br_u1(b);   /* additional_extension2_flag */
	}
	if (b->overrun) return EBADMSG;
	(void)d;
	s.valid = 1;
	*out = s;
	return ret;
}

static int parse_pps(Edge264Decoder *d, BitReader *b) {
	PPS p; memset(&p, 0, sizeof(p));
	int ret = 0;
	unsigned id = br_ue(b);
	if (id >= E264_MAX_PPS || id >= 4) ret = ENOTSUP;   /* the reference supports 4 PPS ids (headers.c:1435) */
	br_ue(b);
	p.entropy_coding_mode = br_u1(b);
	p.bottom_field_pic_order_present = br_u1(b);
	if (br_ue(b) != 0) return ENOTSUP;   /* slice groups: cannot parse further */
	p.num_ref_idx_default[0] = br_ue_i(b, 32) + 1; p.num_ref_idx_default[1] = br_ue_i(b, 32) + 1;
	if (p.num_ref_idx_default[0] > 32 || p.num_ref_idx_default[1] > 32) return EBADMSG;
	p.weighted_pred_flag = br_u1(b); p.weighted_bipred_idc = br_u(b, 2);
	int q = br_se(b); if (q < -26 || q > 25) return EBADMSG;
	p.pic_init_qp = 26 + q;
	br_se(b);
	p.chroma_qp_index_offset[0] = p.chroma_qp_index_offset[1] = br_se(b);
	if (p.chroma_qp_index_offset[0] < -12 || p.chroma_qp_index_offset[0] > 12) return EBADMSG;
	p.deblocking_filter_control_present = br_u1(b);
	if (br_u1(b)) ret = ENOTSUP;   /* constrained_intra_pred_flag */
	if (br_u1(b)) ret = ENOTSUP;   /* redundant_pic_cnt_present_flag */
	int has_matrix = 0;
	if (br_more_rbsp_data(b)) {
		p.transform_8x8_mode = br_u1(b);
		has_matrix = br_u1(b);
		if (has_matrix) parse_scaling_lists(b, p.sl4x4, p.sl8x8, p.transform_8x8_mode);   /* zeros = "take the SPS list" */
		p.chroma_qp_index_offset[1] = br_se(b);
		if (p.chroma_qp_index_offset[1] < -12 || p.chroma_qp_index_offset[1] > 12) return EBADMSG;
	}
	if (b->overrun || p.weighted_bipred_idc == 3) return EBADMSG;
	p.valid = 1 + has_matrix;
	if (ret == 0) d->pps[id] = p;
	return ret;
}

/* scaling lists in force for a slice (reference merge rule, headers.c:903-915) */
static void merge_scaling(const SPS *s, const PPS *p, E264SliceRec *sr) {
	if (p->valid == 2) {
		for (int i = 0; i < 6; i++) {
			const uint8_t *fb = s->sl4x4[i < 3 ? 0 : 3];
			for (int k = 0; k < 16; k++) sr->scaling4x4[i][k] = p->sl4x4[i][k] ? p->sl4x4[i][k] : fb[k];
		}
		for (int i = 0; i < 2; i++) for (int k = 0; k < 64; k++) sr->scaling8x8[i][k] = p->sl8x8[i][k] ? p->sl8x8[i][k] : s->sl8x8[i][k];
	} else {
		memcpy(sr->scaling4x4, s->sl4x4, sizeof(sr->scaling4x4));
		memcpy(sr->scaling8x8, s->sl8x8, sizeof(sr->scaling8x8));
	}
}

/* ------------------------------------------------------------------------------------------ */
/* host mirrors and output queue                                                                */
/* ------------------------------------------------------------------------------------------ */
static void hostbuf_free(Edge264Decoder *d, HostBuf *hb) {
	if (hb->p) {
		if (d->alloc_cb) d->free_cb(hb->p, hb->mbs, d->alloc_arg);
		else d->be->host_free(d->be_ctx, hb->p);
	}
	if (hb->map) d->be->pinned_free(d->be_ctx, hb->map);
	if (hb->motion) {
		if (d->alloc_cb) d->free_cb(hb->motion, hb->motion_mbs, d->alloc_arg);
		else d->be->host_free(d->be_ctx, hb->motion);
	}
	if (hb->packed) {
		if (d->alloc_cb) d->free_cb(hb->packed, hb->packed_mbs, d->alloc_arg);
		else d->be->host_free(d->be_ctx, hb->packed);
	}
	if (hb->picstats) {
		if (d->alloc_cb) d->free_cb(hb->picstats, hb->picstats_mbs, d->alloc_arg);
		else d->be->host_free(d->be_ctx, hb->picstats);
	}
	memset(hb, 0, sizeof(*hb));
}
/* the nearest even size to s_a * t_b / s_b, within 2..16384: the resized side that keeps the aspect ratio */
static int32_t aspect_size(int64_t s_a, int64_t s_b, int64_t t_b) {
	const int64_t t = 2 * ((s_a * t_b + s_b) / (2 * s_b));
	return (int32_t)(t < 2 ? 2 : t > 16384 ? 16384 : t);
}
/* what the pictures of the active sequence are packed as: the decoder's format and scale, the sequence's cropping
 * rectangle, and for the resized output the requested size, a 0 side derived from the cropping rectangle */
static E264PackedDesc packed_desc(const Edge264Decoder *d) {
	const Edge264Frame *o = &d->out_fmt;
	E264PackedDesc k = {d->packed_format, d->packed_scale, o->frame_crop_offsets[3], o->frame_crop_offsets[0],
	                    d->w_mbs * 16 - o->frame_crop_offsets[3] - o->frame_crop_offsets[1], d->h_mbs * 16 - o->frame_crop_offsets[0] - o->frame_crop_offsets[2]};
	if (d->packed_scale < 0) {
		k.target_width = d->packed_width ? d->packed_width : aspect_size(k.width, k.height, d->packed_height);
		k.target_height = d->packed_height ? d->packed_height : aspect_size(k.height, k.width, d->packed_width);
	}
	return k;
}
/* a buffer beside the samples, of their memory kind: from the application's allocator, else from the backend's output
 * mirrors (pinned host memory, device memory with E264B_OUTPUT=device) */
static uint8_t *side_alloc(Edge264Decoder *d, size_t bytes, void **mbs) {
	void *m = NULL;
	if (d->alloc_cb) d->alloc_cb(&m, (unsigned)bytes, mbs, 0, ENOMEM, d->alloc_arg);
	else {
		pthread_mutex_lock(&d->be_lock);
		m = d->be->host_alloc(d->be_ctx, bytes);
		pthread_mutex_unlock(&d->be_lock);
	}
	return (uint8_t *)m;
}
static int hostbuf_acquire(Edge264Decoder *d) {
	for (int i = 0; i < E264_MAX_HOSTBUFS; i++) if (d->hb[i].state == 0 && d->hb[i].p) return i;
	for (int i = 0; i < E264_MAX_HOSTBUFS; i++) if (d->hb[i].state == 0) {
		HostBuf *hb = &d->hb[i];
		size_t bytes = (size_t)d->frame_bytes + 64;
		if (d->alloc_cb) {
			void *smp = NULL, *mbs = NULL;
			/* reference sizes (headers.c:113-117): samples = plane_Y + plane_C + 16, mbs = 304 * ((W+1)*H - 1) */
			d->alloc_cb(&smp, (unsigned)(d->plane_y + d->plane_c + 16), &mbs, (unsigned)(304 * ((d->w_mbs + 1) * d->h_mbs - 1)), ENOMEM, d->alloc_arg);
			if (!smp) return -1;
			hb->p = (uint8_t *)smp; hb->mbs = mbs;
		} else {
			pthread_mutex_lock(&d->be_lock);
			hb->p = (uint8_t *)d->be->host_alloc(d->be_ctx, bytes);
			pthread_mutex_unlock(&d->be_lock);
			if (!hb->p) return -1;
		}
		/* the error map stays in pinned host memory even when the samples are device memory */
		if (d->be->submit_maps) {
			pthread_mutex_lock(&d->be_lock);
			hb->map = (uint8_t *)d->be->pinned_alloc(d->be_ctx, (size_t)d->w_mbs * d->h_mbs);
			pthread_mutex_unlock(&d->be_lock);
			if (!hb->map) { hostbuf_free(d, hb); return -1; }
		}
		/* the motion export, the packed output and the statistics live where the samples live */
		if (d->motion && !(hb->motion = side_alloc(d, (size_t)d->w_mbs * d->h_mbs * E264_MOTION_BYTES, &hb->motion_mbs))) { hostbuf_free(d, hb); return -1; }
		if (d->packed) {
			const E264PackedDesc k = packed_desc(d);
			if (!(hb->packed = side_alloc(d, (size_t)e264_packed_layout(&k).bytes, &hb->packed_mbs))) { hostbuf_free(d, hb); return -1; }
		}
		if (d->picstats && !(hb->picstats = side_alloc(d, E264_PICSTATS_BYTES((size_t)d->w_mbs * d->h_mbs), &hb->picstats_mbs))) { hostbuf_free(d, hb); return -1; }
		return i;
	}
	return -1;
}
static void hostbufs_free_all(Edge264Decoder *d) {
	for (int i = 0; i < E264_MAX_HOSTBUFS; i++) hostbuf_free(d, &d->hb[i]);
	d->outq_n[0] = d->outq_n[1] = 0; d->pending_release[0] = d->pending_release[1] = -1;
}

/* DPB bookkeeping mirrors the reference's bit sets (edge264_internal.h:1217-1222):
 *   ref            <-> prev_short_term_frames / prev_long_term_frames
 *   needed_for_output <-> to_get_frames & ~output_frames */
/* slot i holds a picture of the view being worked on (d->view) */
static inline int in_view(const Edge264Decoder *d, int i) { return d->pics[i].in_use && d->pics[i].view == d->view; }
static inline const SPS *view_sps(const Edge264Decoder *d) { return d->view ? &d->ssps : &d->sps; }
static int dpb_fullness(Edge264Decoder *d) {
	int n = 0;
	for (int i = 0; i < d->n_slots; i++) if (in_view(d, i) && (d->pics[i].ref || d->pics[i].needed_for_output)) n++;
	return n;
}
static int waiting_for_output(Edge264Decoder *d) {
	int n = 0;
	for (int i = 0; i < d->n_slots; i++) if (in_view(d, i) && d->pics[i].needed_for_output) n++;
	return n;
}
static void slot_release_if_unused(Edge264Decoder *d, int i) {
	Pic *p = &d->pics[i];
	if (p->in_use && !p->ref && !p->needed_for_output && i != d->cur && i != d->base_slot) p->in_use = 0;
}
/* bumping: output the waiting picture of `view` with the lowest POC (reference bump_frame, headers.c:78-95) */
static int bump_frame(Edge264Decoder *d, int view, int ignore_slot) {
	int best = -1;
	for (int i = 0; i < d->n_slots; i++) {
		Pic *p = &d->pics[i];
		if (!p->in_use || p->view != view || !p->needed_for_output || i == ignore_slot) continue;
		if (best < 0 || p->poc_top < d->pics[best].poc_top) best = i;
	}
	if (best < 0) return 0;
	Pic *p = &d->pics[best];
	p->needed_for_output = 0;
	if (p->host_buf >= 0) {
		d->hb[p->host_buf].state = 2; d->outq[view][d->outq_n[view]++] = p->host_buf;
		if (__atomic_load_n(&d->hb[p->host_buf].submitted, __ATOMIC_ACQUIRE)) p->host_buf = -1;   /* a worker may be submitting it */
	}
	slot_release_if_unused(d, best);
	return 1;
}

/* ------------------------------------------------------------------------------------------ */
/* picture completion                                                                           */
/* ------------------------------------------------------------------------------------------ */
static void apply_marking(Edge264Decoder *d);

/* Macroblocks that no slice delivered (lost or damaged slices): give them a neutral, self-consistent record so
 * that every picture the backend sees is complete — copy of the co-located samples of the most recent reference
 * picture (a P_Skip with zero motion), or DC intra prediction when there is none.  The reference blends an
 * error-probability-weighted intra DC / re-runs P_Skip (recover_slice, edge264_headers.c:295-430); matching its
 * concealed samples is not attempted (SURVEY §8 f3), only a deterministic, safe picture. */
static void conceal_missing(Edge264Decoder *d, PicBuild *pb) {
	const int total = d->w_mbs * d->h_mbs;
	const int ref = pb->conceal_ref;
	if (pb->n_slices == 0) {   /* not one slice arrived: a neutral slice record for the concealed macroblocks to point to */
		E264SliceRec *sr = &pb->slices[0];
		memset(sr, 0, sizeof(*sr));
		memset(sr->scaling4x4, 16, sizeof(sr->scaling4x4)); memset(sr->scaling8x8, 16, sizeof(sr->scaling8x8));
		pb->n_slices = 1;
	}
	for (int a = 0; a < total; a++) {
		if (pb->mbi[a].slice_id) continue;
		E264MbRec *r = pb->recs + a;
		memset(r, 0, sizeof(*r));
		r->err = 100;                 /* made up: no slice delivered it */
		r->qp[0] = r->qp[1] = r->qp[2] = 26;
		memset(r->ref_idx, -1, sizeof(r->ref_idx)); memset(r->ref_pic, -1, sizeof(r->ref_pic));
		if (ref >= 0) {
			r->kind = MBK_INTER; r->flags = MBF_SKIP;
			for (int i8 = 0; i8 < 4; i8++) { r->ref_idx[0][i8] = 0; r->ref_pic[0][i8] = (int8_t)ref; }
		} else {
			r->kind = MBK_I16x16; r->i16_mode = IMODE(2, 1 | 2 | 8); r->chroma_mode = IMODE(0, 1 | 2 | 8);
		}
	}
}

/* the frame slot a lost macroblock is copied from: the most recent reference picture (header-time state) */
static int conceal_reference(Edge264Decoder *d) {
	int ref = -1, best = -1;
	for (int i = 0; i < d->n_slots; i++) if (i != d->cur && in_view(d, i) && d->pics[i].ref && !d->pics[i].nonexisting && d->pics[i].uid > best) { best = d->pics[i].uid; ref = i; }
	return ref;
}

/* data side of a finished picture: conceal what no slice delivered and list the intra macroblocks (build_finalize: the
 * records are complete afterwards), then hand the picture to the backend (build_submit).  build_work runs both once
 * the picture is closed and every slice of it is parsed. */
static void build_finalize(Edge264Decoder *d, PicBuild *pb, E264PicDesc *pd) {
	if (pb->mbs_done < d->w_mbs * d->h_mbs) {
		conceal_missing(d, pb);
		pb->any_err = 1;
		if (pb->conceal_ref >= 0) pb->ref_mask |= 1u << pb->conceal_ref;
	}
	memset(pd, 0, sizeof(*pd));
	pd->width_mbs = d->w_mbs; pd->height_mbs = d->h_mbs; pd->stride_y = d->stride_y; pd->stride_c = d->stride_c;
	pd->plane_y = d->plane_y; pd->frame_bytes = d->frame_bytes; pd->dst_slot = pb->slot;
	pd->n_slices = pb->n_slices; pd->n_coefs = (int32_t)pb->n_coefs; pd->any_deblock = pb->any_deblock; pd->staging = pb->staging;
	pd->luma_only = (uint8_t)d->luma_only;
	/* intra macroblocks in raster order: the device draws them from this list, so a waiting macroblock only ever waits for earlier entries */
	const int total = d->w_mbs * d->h_mbs; int n = 0;
	for (int a = 0; a < total; a++) if (pb->recs[a].kind != MBK_INTER) pb->intra_list[n++] = (uint32_t)a;
	pd->n_intra = n;
}
/* called in decoding order: whether the picture needs an error map depends on what the pictures before it left in its
 * reference slots.  A slot is tainted from the moment a picture with a map (or a non-existing frame) is written into it
 * until a picture without one is. */
static int build_submit(Edge264Decoder *d, PicBuild *pb, E264PicDesc *pd, uint64_t *ticket) {
	*ticket = 0;
	if (pb->host_buf < 0) return 0;
	pd->err_pic = d->be->submit_maps && (pb->any_err || (pb->ref_mask & d->taint) != 0);
	pd->taint = d->taint;
	if (pd->err_pic) d->taint |= 1u << pb->slot; else d->taint &= ~(1u << pb->slot);
	HostBuf *hb = &d->hb[pb->host_buf];
	hb->err_pic = pd->err_pic;
	int r;
	{
		PROF_BEGIN;
		if (d->packed || d->picstats) {   /* the picture is packed and measured when it is reconstructed, like its samples are copied then */
			const E264PackedDesc k = packed_desc(d);   /* the statistics' histograms take its cropping rectangle */
			if (d->packed) hb->pk = k;
			const E264Outputs o = {hb->map, hb->motion, pb->slot_ids, E264_MAX_SLOTS, &hb->motion_dev, hb->packed, hb->pk, &hb->packed_dev,
			                       hb->picstats, k.left, k.top, k.width, k.height, &hb->picstats_dev};
			r = d->be->submit_outputs(d->be_ctx, pd, hb->p, &o, ticket);
		} else if (d->motion) r = d->be->submit_motion(d->be_ctx, pd, hb->p, hb->map, hb->motion, pb->slot_ids, &hb->motion_dev, ticket);
		else r = d->be->submit_maps ? d->be->submit_maps(d->be_ctx, pd, hb->p, hb->map, ticket) : d->be->submit(d->be_ctx, pd, hb->p, ticket);
		PROF_END(2);
	}
	return r ? EIO : 0;
}

static int build_work(Edge264Decoder *d, PicBuild *pb);

/* Close the current picture: no later slice joins it.  With workers, one of them finalizes and submits it; with none,
 * the calling thread does it here and the backend's error is returned. */
static int finish_picture(Edge264Decoder *d) {
	if (d->cur < 0) return 0;
	Pic *p = &d->pics[d->cur];
	int ret = 0;
	d->view = p->view;
	if (d->pb) {   /* a skipped picture has no build */
		pthread_mutex_lock(&d->lock);
		if (!d->pb->closed) {   /* a worker closes a complete picture itself in low-latency output (build_work) */
			d->pb->conceal_ref = conceal_reference(d);
			d->pb->closed = 1;
			pthread_cond_broadcast(&d->work_cv);
			if (!d->n_threads) ret = build_work(d, d->pb);
		}
		pthread_mutex_unlock(&d->lock);
		d->pb = NULL;
	}
	if (p->host_buf >= 0 && !p->needed_for_output) p->host_buf = -1;   /* already in the output queue */
	apply_marking(d);
	int c = d->cur, old_base = -1;
	d->cur = -1;
	if (d->mvc && !p->view) { old_base = d->base_slot; d->base_slot = c; }   /* the reference's basePic (headers.c:73-74) */
	slot_release_if_unused(d, c);
	if (old_base >= 0 && old_base != c) slot_release_if_unused(d, old_base);
	return ret;
}

/* ------------------------------------------------------------------------------------------ */
/* picture pipeline: slices queued on builds, parsed and submitted by build_work                  */
/* ------------------------------------------------------------------------------------------ */
/* The calling thread parses headers, runs the decoded-picture-buffer logic and queues slices; build_work parses slice
 * data.  Worker threads run it, several pictures at a time; with no workers the calling thread runs it as soon as a
 * slice is queued and when the picture is closed, so every picture is submitted before the next one starts.  One thread
 * owns a picture at a time (its slices share the coefficient pool and run in order); pictures are handed to the backend
 * strictly in decoding order.  A B slice waits until its co-located picture is completely parsed (its records are the
 * motion data direct prediction reads); nothing else depends on another picture at parse time — pixels are the
 * device's business.  Reference counterpart: task dependencies + worker_loop, edge264_internal.h:1196-1226,
 * edge264_headers.c:450-603. */
static PicBuild *build_acquire(Edge264Decoder *d, int slot) {
	pthread_mutex_lock(&d->lock);
	PicBuild *pb = NULL;
	for (;;) {
		/* the slot's records may still be written by its previous picture's parser or read as co-located motion */
		if (d->slot_users[slot] == 0) for (int i = 0; i < d->n_builds && !pb; i++) if (!d->builds[i].in_use) pb = &d->builds[i];
		if (pb) break;
		/* not reached without workers: every earlier picture has been submitted, which frees its build and its slots */
		pthread_cond_wait(&d->done_cv, &d->lock);
	}
	MbInfo *mbi = pb->mbi;
	memset(pb, 0, sizeof(*pb));
	pb->mbi = mbi; pb->in_use = 1; pb->seq = d->next_seq++;
	d->slot_users[slot]++; d->slot_build[slot] = pb; d->slot_build_seq[slot] = pb->seq;
	pthread_mutex_unlock(&d->lock);
	return pb;
}
static void slice_enqueue(Edge264Decoder *d, PicBuild *pb, SliceJob *job, int col_slot) {
	pthread_mutex_lock(&d->lock);
	job->next = NULL; job->dep = NULL; job->dep_seq = 0; job->col_slot = col_slot;
	if (col_slot >= 0) {
		d->slot_users[col_slot]++;
		if (d->slot_build[col_slot] && d->slot_build[col_slot] != pb) { job->dep = d->slot_build[col_slot]; job->dep_seq = d->slot_build_seq[col_slot]; }
	}
	if (pb->tail) pb->tail->next = job; else pb->head = job;
	pb->tail = job;
	pb->held = 0;
	pthread_cond_broadcast(&d->work_cv);
	pthread_mutex_unlock(&d->lock);
}
/* wait until every picture but `except` (NULL: every picture) has been parsed and handed to the backend (flush, end of
 * stream, format change, a fill of a frame slot) */
static void threads_drain(Edge264Decoder *d, const PicBuild *except) {
	pthread_mutex_lock(&d->lock);
	for (;;) {
		int busy = 0;
		for (int i = 0; i < d->n_builds; i++) busy |= d->builds[i].in_use && &d->builds[i] != except;
		if (!busy) break;
		/* not reached without workers: the picture under construction, if any, was closed before, which submitted it */
		pthread_cond_wait(&d->done_cv, &d->lock);
	}
	pthread_mutex_unlock(&d->lock);
}
static inline int job_ready(const SliceJob *j) { return !j->dep || j->dep->seq != j->dep_seq || j->dep->parsed || !j->dep->in_use; }
/* The work of one build, called with d->lock held: parse its queued slices while they are ready; once the picture is
 * closed and completely parsed, finalize it and hand the parsed pictures to the backend in decoding order.  Returns
 * the first slice-data error (EBADMSG, ENOMEM when the coefficient pool runs out) or the backend's EIO. */
static int build_work(Edge264Decoder *d, PicBuild *pb) {
	int ret = 0;
	pb->running = 1;
	while (pb->head && job_ready(pb->head)) {
		SliceJob *job = pb->head;
		pb->head = job->next; if (!pb->head) pb->tail = NULL;
		pthread_mutex_unlock(&d->lock);
		job->sc.n_coefs = pb->n_coefs;      /* the slices of a picture share one coefficient pool */
		int n = e264_parse_slice_data(&job->sc);
		pb->n_coefs = job->sc.n_coefs; pb->n_intra += job->sc.n_intra;
		if (n > 0) pb->mbs_done += n;
		pb->any_err |= job->sc.any_err;
		if (job->sc.error && !ret) ret = job->sc.error == 2 ? ENOMEM : EBADMSG;
		free(job->rbsp);
		pthread_mutex_lock(&d->lock);
		if (job->col_slot >= 0) { d->slot_users[job->col_slot]--; pthread_cond_broadcast(&d->done_cv); }
		free(job);
	}
	/* low-latency output with workers (edge264_latency.h): the picture is closed as soon as its slices cover every
	 * macroblock, like the synchronous path does in decode_slice, instead of by the next picture's first slice */
	if (!pb->head && !pb->closed && pb->close_complete && !pb->held && pb->mbs_done >= d->w_mbs * d->h_mbs) pb->closed = 1;
	if (!pb->head && pb->closed) {
		pthread_mutex_unlock(&d->lock);
		build_finalize(d, pb, &pb->pd);
		pthread_mutex_lock(&d->lock);
		pb->parsed = 1; pb->running = 0;      /* its records are complete: B pictures may read them */
		pthread_cond_broadcast(&d->work_cv);
		/* hand parsed pictures to the backend in decoding order; whoever completes the oldest one also sends the
		 * ones that were waiting behind it, so no worker ever sleeps on the order */
		while (!d->submitting) {
			PicBuild *q = NULL;
			for (int i = 0; i < d->n_builds; i++) if (d->builds[i].in_use && d->builds[i].parsed && d->builds[i].seq == d->submit_seq) q = &d->builds[i];
			if (!q) break;
			uint64_t ticket = 0;
			d->submitting = 1;
			pthread_mutex_unlock(&d->lock);
			pthread_mutex_lock(&d->be_lock);
			int r = build_submit(d, q, &q->pd, &ticket);
			pthread_mutex_unlock(&d->be_lock);
			if (r && !ret) ret = r;
			pthread_mutex_lock(&d->lock);
			if (q->host_buf >= 0) { d->hb[q->host_buf].ticket = ticket; __atomic_store_n(&d->hb[q->host_buf].submitted, 1, __ATOMIC_RELEASE); }
			d->submit_seq++; d->submitting = 0;
			d->slot_users[q->slot]--;
			q->in_use = 0;
			pthread_cond_broadcast(&d->done_cv);
		}
	} else pb->running = 0;               /* more slices to come, or the next one waits for its co-located picture */
	return ret;
}
static void *worker_main(void *arg) {
	Edge264Decoder *d = (Edge264Decoder *)arg;
	pthread_mutex_lock(&d->lock);
	for (;;) {
		PicBuild *pb = NULL;
		while (!d->stop) {
			for (int i = 0; i < d->n_builds; i++) {     /* the oldest picture with something to do */
				PicBuild *b = &d->builds[i];
				if (!b->in_use || b->running || b->parsed) continue;
				if (!(b->head ? job_ready(b->head) : b->closed)) continue;
				if (!pb || b->seq < pb->seq) pb = b;
			}
			if (pb) break;
			pthread_cond_wait(&d->work_cv, &d->lock);
		}
		if (d->stop) break;
		build_work(d, pb);
	}
	pthread_mutex_unlock(&d->lock);
	return NULL;
}
static void threads_stop(Edge264Decoder *d) {
	threads_drain(d, NULL);
	pthread_mutex_lock(&d->lock);
	d->stop = 1;
	pthread_cond_broadcast(&d->work_cv); pthread_cond_broadcast(&d->done_cv);
	pthread_mutex_unlock(&d->lock);
	for (int i = 0; i < d->n_threads; i++) pthread_join(d->threads[i], NULL);
	d->n_threads = 0;
}

/* 8.2.5 decoded reference picture marking, applied when the picture is complete.  Mirrors the
 * reference's order of operations (headers.c:611-701): MMCO list, then sliding window whenever the
 * number of references reaches max_num_ref_frames, then the current picture is inserted. */
static void apply_marking(Edge264Decoder *d) {
	Pic *cur = &d->pics[d->cur];
	SliceHeader *h = &d->first_sh;
	if (!d->cur_nal_ref_idc) { cur->ref = 0; return; }
	int cur_long = 0;
	if (d->cur_idr) {
		for (int i = 0; i < d->n_slots; i++) if (i != d->cur && in_view(d, i)) { d->pics[i].ref = 0; slot_release_if_unused(d, i); }
		cur_long = h->long_term_reference_flag;
		cur->long_term_idx = 0;
	} else {
		for (int k = 0; k < h->n_mmco; k++) {
			int op = h->mmco[k].op;
			int target = -1;
			if (op == 1 || op == 3) {
				int fn = cur->frame_num - 1 - (int)h->mmco[k].a;
				for (int i = 0; i < d->n_slots; i++) if (i != d->cur && in_view(d, i) && d->pics[i].ref == 1 && d->pics[i].frame_num == fn) { target = i; d->pics[i].ref = 0; }
			}
			if (op == 2 || op == 3 || op == 4 || op == 6) {
				int idx = (int)(op == 3 ? h->mmco[k].b : h->mmco[k].a);
				int up = op == 4 ? INT_MAX : idx;
				if (op == 4) idx = (int)h->mmco[k].a;   /* max_long_term_frame_idx_plus1: drop idx >= a */
				for (int i = 0; i < d->n_slots; i++) if (i != d->cur && in_view(d, i) && d->pics[i].ref == 2 && d->pics[i].long_term_idx >= idx && d->pics[i].long_term_idx <= up) d->pics[i].ref = 0;
				if (op == 3 && target >= 0) { d->pics[target].ref = 2; d->pics[target].long_term_idx = idx; }
				if (op == 6) { cur_long = 1; cur->long_term_idx = idx; }
			}
			if (op == 5) {
				for (int i = 0; i < d->n_slots; i++) if (i != d->cur && in_view(d, i)) d->pics[i].ref = 0;
			}
		}
		for (int i = 0; i < d->n_slots; i++) slot_release_if_unused(d, i);
	}
	int nref = 0;
	for (int i = 0; i < d->n_slots; i++) if (i != d->cur && in_view(d, i) && d->pics[i].ref) nref++;
	if (nref >= view_sps(d)->max_num_ref_frames) {
		int best = -1;
		for (int i = 0; i < d->n_slots; i++) if (i != d->cur && in_view(d, i) && d->pics[i].ref == 1 && (best < 0 || d->pics[i].frame_num < d->pics[best].frame_num)) best = i;
		if (best >= 0) { d->pics[best].ref = 0; slot_release_if_unused(d, best); }
	}
	cur->ref = cur_long ? 2 : 1;
	for (int k = 0; k < h->n_mmco; k++) if (h->mmco[k].op == 5) cur->frame_num = 0;   /* 8.2.1: the picture is now "frame_num 0" for everything that follows */
	d->prev_ref_frame_num[d->view] = cur->frame_num;
	d->q_prev_ref_frame_num[d->view] = d->q_cur_frame_num;
	for (int k = 0; k < h->n_mmco; k++) if (h->mmco[k].op == 5) d->q_prev_ref_frame_num[d->view] = 0;
}

/* ------------------------------------------------------------------------------------------ */
/* sequence (re)configuration                                                                   */
/* ------------------------------------------------------------------------------------------ */
static int bump_all(Edge264Decoder *d) {
	if (d->cur >= 0) finish_picture(d);
	threads_drain(d, NULL);
	for (int v = 0; v < 2; v++) while (bump_frame(d, v, -1));
	if (d->outq_n[0] || d->outq_n[1]) return ENOBUFS;
	/* frames the application still holds (borrowed, or handed out until the next decode_NAL) keep their buffers: a
	 * change of format must wait for them like the reference's `to_get_frames | output_frames` test (headers.c:2005-2007) */
	for (int i = 0; i < E264_MAX_HOSTBUFS; i++) if (d->hb[i].state == 3 && d->hb[i].borrowed) return ENOBUFS;
	return 0;
}

/* keep_numbering: the frame format is unchanged and only the frame pool grows — the reference does not clear its decoder
 * then (it compares size, crop and bit depth only, headers.c:2016-2024), so FrameId numbering and the parameter sets go on */
static int configure_sequence(Edge264Decoder *d, const SPS *s, int keep_numbering) {
	int w = s->width_mbs * 16, h = s->height_mbs * 16;
	d->w_mbs = s->width_mbs; d->h_mbs = s->height_mbs;
	d->stride_y = w; if (!(d->stride_y & 2047)) d->stride_y += 16;       /* reference headers.c:2027-2029 */
	d->stride_c = w; if (!(d->stride_c & 4095)) d->stride_c += 16;       /* headers.c:2035-2037 pads by 8; 16 keeps both chroma planes 8-byte aligned for vector stores and TMA */
	d->plane_y = d->stride_y * h; d->plane_c = d->stride_c * (h >> 1);
	d->frame_bytes = d->plane_y + d->plane_c + 16;
	pthread_mutex_lock(&d->lock);      /* idle workers scan builds[0..n_builds) */
	d->n_builds = d->n_threads ? d->n_threads + 2 : 1;
	if (d->n_builds > E264_MAX_BUILDS) d->n_builds = E264_MAX_BUILDS;
	pthread_mutex_unlock(&d->lock);
	/* a picture keeps its slot (and the slot's record buffer) until it is handed to the device: parsing ahead needs one spare slot per picture in flight.
	 * A stereo sequence holds both views' references, current pictures and waiting pictures; past 32 slots it gives up the parse-ahead slack and
	 * the waiting slots before any reference slot (case 15 refuses views that do not fit). */
	const int slack = d->n_threads ? d->n_builds : 0;
	if (!d->mvc) {
		d->n_slots = s->max_num_ref_frames + 2 + slack;
		if (d->n_slots > E264_MONO_SLOTS) d->n_slots = E264_MONO_SLOTS;
	} else {
		d->n_slots = s->max_num_ref_frames + d->ssps.max_num_ref_frames + 4 + slack;
		if (d->n_slots > E264_MAX_SLOTS) d->n_slots = E264_MAX_SLOTS;
	}
	E264PicDesc g; memset(&g, 0, sizeof(g));
	g.width_mbs = d->w_mbs; g.height_mbs = d->h_mbs; g.stride_y = d->stride_y; g.stride_c = d->stride_c; g.plane_y = d->plane_y; g.frame_bytes = d->frame_bytes;
	g.staging = d->n_threads ? (d->n_threads + 2 > E264_MAX_BUILDS ? E264_MAX_BUILDS : d->n_threads + 2) + 2 : 0;   /* staging areas wanted: one per picture being parsed + two in flight on the device; 0 = the backend's default */
	hostbufs_free_all(d);
	if (d->be->configure(d->be_ctx, &g, d->n_slots)) return ENOMEM;
	int oom = 0;
	pthread_mutex_lock(&d->lock);
	for (int i = 0; i < E264_MAX_BUILDS; i++) {
		free(d->builds[i].mbi); memset(&d->builds[i], 0, sizeof(d->builds[i]));
		if (i < d->n_builds && !(d->builds[i].mbi = (MbInfo *)calloc((size_t)d->w_mbs * d->h_mbs, sizeof(MbInfo)))) oom = 1;
	}
	d->pb = NULL;
	memset(d->slot_users, 0, sizeof(d->slot_users)); memset(d->slot_build, 0, sizeof(d->slot_build));
	d->taint = 0;
	pthread_mutex_unlock(&d->lock);
	if (oom) return ENOMEM;
	memset(d->pics, 0, sizeof(d->pics));
	for (int i = 0; i < E264_MAX_SLOTS; i++) d->pics[i].host_buf = -1;
	d->cur = -1; d->base_slot = -1;
	Edge264Frame *o = &d->out_fmt; memset(o, 0, sizeof(*o));
	o->bit_depth_Y = o->bit_depth_C = 8;
	o->width_Y = (int16_t)(w - s->crop[0] - s->crop[1]); o->height_Y = (int16_t)(h - s->crop[2] - s->crop[3]);
	o->width_C = o->width_Y >> 1; o->height_C = o->height_Y >> 1;
	o->stride_Y = (int16_t)d->stride_y; o->stride_C = (int16_t)d->stride_c;
	o->stride_mb = (int16_t)(s->width_mbs * 304);   /* sizeof(Edge264Macroblock) in the reference; wraps like there */
	o->frame_crop_offsets[0] = (int16_t)s->crop[2]; o->frame_crop_offsets[1] = (int16_t)s->crop[1];
	o->frame_crop_offsets[2] = (int16_t)s->crop[3]; o->frame_crop_offsets[3] = (int16_t)s->crop[0];
	d->configured = 1;
	if (!keep_numbering) {
		for (int v = 0; v < 2; v++) { d->q_prev_ref_frame_num[v] = -1; d->prev_ref_frame_num[v] = -1; d->prev_ref_poc[v] = 0; }
		memset(d->ref_frame_view, 0, sizeof(d->ref_frame_view));
	}
	return 0;
}

static inline int clamp8(int v) { return v < -128 ? -128 : v > 127 ? 127 : v; }   /* bounded reads like the reference's get_se16(-128,127) (headers.c:721-731) */

/* ------------------------------------------------------------------------------------------ */
/* slice header                                                                                 */
/* ------------------------------------------------------------------------------------------ */
/* s: the SPS of the slice's view; idr: IdrPicFlag (nal_unit_type 5, or non_idr_flag 0 in a NAL unit 20 header) */
static int parse_slice_header(Edge264Decoder *d, const SPS *s, BitReader *b, int nal_unit_type, int idr, int nal_ref_idc, SliceHeader *h, const PPS **ppps) {
	memset(h, 0, sizeof(*h));
	h->first_mb = br_ue_i(b, 139264);   /* bounded like the reference's get_ue32(139263) (headers.c:968); anything larger fails the first_mb >= total test */
	int st = br_ue_i(b, 10);
	if (st > 9) return EBADMSG;
	if (nal_unit_type == 5 || s->max_num_ref_frames == 0) st = 2;   /* reference headers.c:983 */
	h->slice_type = st < 5 ? st : st - 5;
	h->pps_id = br_ue_i(b, 256);
	if (h->slice_type > 2 || h->pps_id >= 4) return ENOTSUP;
	const PPS *p = &d->pps[h->pps_id];
	if (!s->valid || !p->valid) return EBADMSG;
	*ppps = p;
	h->frame_num = br_u(b, s->log2_max_frame_num);
	if (idr) h->frame_num = 0;
	h->idr_pic_id = -1;
	if (idr) h->idr_pic_id = br_ue_i(b, 65536);
	if (s->poc_type == 0) {
		h->poc_lsb = br_u(b, s->log2_max_poc_lsb);
		if (p->bottom_field_pic_order_present) h->delta_poc_bottom = br_se(b);
	} else if (s->poc_type == 1 && !s->delta_pic_order_always_zero_flag) {
		h->delta_poc[0] = br_se(b);
		if (p->bottom_field_pic_order_present) h->delta_poc[1] = br_se(b);
	}
	h->num_ref[0] = p->num_ref_idx_default[0]; h->num_ref[1] = p->num_ref_idx_default[1];
	if (h->slice_type < 2) {
		if (h->slice_type == 1) h->direct_spatial = br_u1(b);
		if (br_u1(b)) {
			h->num_ref[0] = br_ue_i(b, 32) + 1;
			if (h->slice_type == 1) h->num_ref[1] = br_ue_i(b, 32) + 1;
		}
		if (h->num_ref[0] > 16) h->num_ref[0] = h->num_ref[0] > 32 ? 0 : 16;
		if (h->num_ref[1] > 16) h->num_ref[1] = h->num_ref[1] > 32 ? 0 : 16;
		if (h->num_ref[0] == 0 || h->num_ref[1] == 0) return EBADMSG;
		for (int l = 0; l <= h->slice_type; l++) {
			if (!br_u1(b)) continue;
			int n = 0;
			for (;;) {
				unsigned op = br_ue(b);
				if (op == 3) break;
				if (op > 5 || n >= 32) return EBADMSG;
				h->mod[l][n].op = (uint8_t)op; h->mod[l][n].val = (uint32_t)br_ue_i(b, 1 << 20); n++;
			}
			h->n_mod[l] = n;
		}
		int wp = h->slice_type == 0 ? p->weighted_pred_flag : p->weighted_bipred_idc;
		if (wp == 1) {
			h->luma_log2_wd = br_ue_i(b, 8); h->chroma_log2_wd = br_ue_i(b, 8);
			if (h->luma_log2_wd > 7 || h->chroma_log2_wd > 7) return EBADMSG;
			for (int l = 0; l <= h->slice_type; l++) for (int i = 0; i < h->num_ref[l]; i++) {
				if (br_u1(b)) { h->w[l][i][0] = (int16_t)clamp8(br_se(b)); h->o[l][i][0] = (int16_t)clamp8(br_se(b)); }
				else { h->w[l][i][0] = (int16_t)(1 << h->luma_log2_wd); h->o[l][i][0] = 0; }
				if (br_u1(b)) for (int c = 1; c < 3; c++) { h->w[l][i][c] = (int16_t)clamp8(br_se(b)); h->o[l][i][c] = (int16_t)clamp8(br_se(b)); }
				else for (int c = 1; c < 3; c++) { h->w[l][i][c] = (int16_t)(1 << h->chroma_log2_wd); h->o[l][i][c] = 0; }
			}
		}
	}
	if (nal_ref_idc) {
		if (idr) { h->no_output_of_prior_pics = br_u1(b); h->long_term_reference_flag = br_u1(b); }
		else if (br_u1(b)) {
			h->adaptive_marking = 1;
			int n = 0;
			for (;;) {
				unsigned op = br_ue(b);
				if (op == 0) break;
				if (op > 6 || n >= 64) return EBADMSG;
				h->mmco[n].op = (uint8_t)op;
				if (op == 1 || op == 3) h->mmco[n].a = (uint32_t)br_ue_i(b, 1 << 20);
				if (op == 2 || op == 4 || op == 6) h->mmco[n].a = (uint32_t)br_ue_i(b, 1 << 20);
				if (op == 3) h->mmco[n].b = (uint32_t)br_ue_i(b, 1 << 20);
				n++;
			}
			h->n_mmco = n;
		}
	}
	if (p->entropy_coding_mode && h->slice_type != 2) { h->cabac_init_idc = br_ue_i(b, 3); if (h->cabac_init_idc > 2) return EBADMSG; }
	int qd = br_se(b);
	h->slice_qp = p->pic_init_qp + qd;
	if (h->slice_qp < 0 || h->slice_qp > 51) return EBADMSG;
	if (p->deblocking_filter_control_present) {
		h->deblock_idc = br_ue_i(b, 3);
		if (h->deblock_idc > 2) return EBADMSG;
		if (h->deblock_idc != 1) {
			int a = br_se(b), bb = br_se(b);
			if (a < -6 || a > 6 || bb < -6 || bb > 6) return EBADMSG;
			h->filter_offset_a = a * 2; h->filter_offset_b = bb * 2;
		}
	}
	if (b->overrun) return EBADMSG;
	return 0;
}

/* 8.2.4: reference picture lists of the slice -> slots */
static void build_ref_lists(Edge264Decoder *d, const SliceHeader *h, int lists[2][32], int nlist[2]) {
	Pic *cur = &d->pics[d->cur];
	int st[E264_MAX_SLOTS], lt[E264_MAX_SLOTS], nst = 0, nlt = 0;
	for (int l = 0; l < 2; l++) for (int i = 0; i < 32; i++) lists[l][i] = -1;
	nlist[0] = nlist[1] = 0;
	for (int i = 0; i < d->n_slots && !d->cur_idr; i++) {
		Pic *p = &d->pics[i];
		if (i == d->cur || !in_view(d, i)) continue;
		if (p->ref == 1) st[nst++] = i; else if (p->ref == 2) lt[nlt++] = i;
	}
	/* long-term by LongTermFrameIdx ascending */
	for (int i = 1; i < nlt; i++) for (int j = i; j > 0 && d->pics[lt[j]].long_term_idx < d->pics[lt[j - 1]].long_term_idx; j--) { int t = lt[j]; lt[j] = lt[j - 1]; lt[j - 1] = t; }
	if (h->slice_type == 0) {
		/* short-term by FrameNum descending (absolute frame numbers, monotonic) */
		for (int i = 1; i < nst; i++) for (int j = i; j > 0 && d->pics[st[j]].frame_num > d->pics[st[j - 1]].frame_num; j--) { int t = st[j]; st[j] = st[j - 1]; st[j - 1] = t; }
		int n = 0;
		for (int i = 0; i < nst; i++) lists[0][n++] = st[i];
		for (int i = 0; i < nlt; i++) lists[0][n++] = lt[i];
		nlist[0] = n;
	} else {
		int before[E264_MAX_SLOTS], after[E264_MAX_SLOTS], nb = 0, na = 0;
		for (int i = 0; i < nst; i++) { if (d->pics[st[i]].poc_top <= cur->poc_top_dec) before[nb++] = st[i]; else after[na++] = st[i]; }
		for (int i = 1; i < nb; i++) for (int j = i; j > 0 && d->pics[before[j]].poc_top > d->pics[before[j - 1]].poc_top; j--) { int t = before[j]; before[j] = before[j - 1]; before[j - 1] = t; }
		for (int i = 1; i < na; i++) for (int j = i; j > 0 && d->pics[after[j]].poc_top < d->pics[after[j - 1]].poc_top; j--) { int t = after[j]; after[j] = after[j - 1]; after[j - 1] = t; }
		int n = 0;
		for (int i = 0; i < nb; i++) lists[0][n++] = before[i];
		for (int i = 0; i < na; i++) lists[0][n++] = after[i];
		for (int i = 0; i < nlt; i++) lists[0][n++] = lt[i];
		nlist[0] = n; n = 0;
		for (int i = 0; i < na; i++) lists[1][n++] = after[i];
		for (int i = 0; i < nb; i++) lists[1][n++] = before[i];
		for (int i = 0; i < nlt; i++) lists[1][n++] = lt[i];
		nlist[1] = n;
	}
	/* H.8.2.1: the second view appends its inter-view reference, the base view of its access unit, to both lists (reference
	 * headers.c:784-792: it keeps its place in the before/after swap) */
	if (d->view) { lists[0][nlist[0]++] = d->base_slot; if (h->slice_type == 1) lists[1][nlist[1]++] = d->base_slot; }
	if (h->slice_type == 1 && nlist[1] > 1 && lists[0][0] == lists[1][0]) { int t = lists[1][0]; lists[1][0] = lists[1][1]; lists[1][1] = t; }
	/* 8.2.4.3 modification */
	int mask = (1 << view_sps(d)->log2_max_frame_num) - 1;
	for (int l = 0; l <= (h->slice_type == 1); l++) {
		int pic_num_pred = cur->frame_num;
		for (int k = 0; k < h->n_mod[l]; k++) {
			int op = h->mod[l][k].op, pic = -1;
			if (op < 2) {
				pic_num_pred = op == 0 ? pic_num_pred - ((int)h->mod[l][k].val + 1) : pic_num_pred + ((int)h->mod[l][k].val + 1);
				for (int i = 0; i < d->n_slots; i++) if (i != d->cur && in_view(d, i) && d->pics[i].ref == 1 && !((d->pics[i].frame_num ^ pic_num_pred) & mask)) { pic = i; break; }
			} else if (op == 2) {
				for (int i = 0; i < d->n_slots; i++) if (i != d->cur && in_view(d, i) && d->pics[i].ref == 2 && d->pics[i].long_term_idx == (int)h->mod[l][k].val) { pic = i; break; }
			} else if (d->view) pic = d->base_slot;   /* idc 4 and 5 name the one inter-view reference (H.8.2.2.3; reference headers.c:848) */
			if (pic < 0) continue;
			if (k >= h->num_ref[l] || k >= 32) break;   /* more operations than list entries: the reference stops at refIdx 32 too (headers.c:817) */
			int buf = pic, c = k;
			do { int sw = lists[l][c]; lists[l][c] = buf; buf = sw; } while (++c < h->num_ref[l] && c < 32 && buf != pic);
		}
	}
}

/* ------------------------------------------------------------------------------------------ */
/* slice NAL                                                                                    */
/* ------------------------------------------------------------------------------------------ */
/* the first free slot, preferring one no parser is still using: taking a busy one would wait in build_acquire for its
 * picture to be submitted (without workers no slot is busy here, so this is the first free slot) */
static int find_free_slot(Edge264Decoder *d) {
	int pick = -1;
	pthread_mutex_lock(&d->lock);
	for (int i = 0; i < d->n_slots && pick < 0; i++) if (!d->pics[i].in_use && d->slot_users[i] == 0) pick = i;
	for (int i = 0; i < d->n_slots && pick < 0; i++) if (!d->pics[i].in_use) pick = i;
	pthread_mutex_unlock(&d->lock);
	return pick;
}

/* 8.2.1 PicOrderCnt and TopFieldOrderCnt of a frame, from its absolute (unwrapped) frame number */
static void picture_poc(const Edge264Decoder *d, const SliceHeader *h, int idr, int nal_ref_idc, int frame_num_abs, int *poc, int *poc_top) {
	const SPS *s = view_sps(d);
	if (s->poc_type == 0) {
		int sh = 32 - s->log2_max_poc_lsb;
		int prev_poc = idr ? 0 : d->prev_ref_poc[d->view];
		int inc = (int)((unsigned)(h->poc_lsb - prev_poc) << sh) >> sh;
		*poc = *poc_top = prev_poc + inc;
		if (h->delta_poc_bottom < 0) *poc += h->delta_poc_bottom;   /* PicOrderCnt = min(top, bottom) */
	} else if (s->poc_type == 1) {
		int abs_fn = s->num_ref_frames_in_poc_cycle > 0 ? frame_num_abs : 0;
		if (nal_ref_idc == 0 && abs_fn > 0) abs_fn--;
		int top = h->delta_poc[0] + (nal_ref_idc ? 0 : s->offset_for_non_ref_pic);
		if (abs_fn > 0) {
			int cyc = (abs_fn - 1) / s->num_ref_frames_in_poc_cycle, in = (abs_fn - 1) % s->num_ref_frames_in_poc_cycle, sum = 0, tot = 0;
			for (int i = 0; i < s->num_ref_frames_in_poc_cycle; i++) { tot += s->offset_for_ref_frame[i]; if (i <= in) sum += s->offset_for_ref_frame[i]; }
			top += cyc * tot + sum;
		}
		int bot = top + s->offset_for_top_to_bottom_field + h->delta_poc[1];
		*poc = top < bot ? top : bot; *poc_top = top;
	} else *poc = *poc_top = frame_num_abs * 2 + (nal_ref_idc != 0) - 1;
}

/* short-term frames the DPB has room for: max_num_ref_frames less the long-term frames */
static int short_term_room(const Edge264Decoder *d) {
	int nlong = 0;
	for (int i = 0; i < d->n_slots; i++) nlong += in_view(d, i) && d->pics[i].ref == 2;
	return view_sps(d)->max_num_ref_frames - nlong;
}

/* the reference decoder's frame buffer for a picture of d->view entering the DPB now (Edge264Decoder.ref_frame_view);
 * returns whether that buffer last held a picture of the same view */
static int take_ref_frame(Edge264Decoder *d, Pic *p) {
	uint32_t busy = 0, dropped = 0;
	const int ghosts = d->ghost_frames;
	d->ghost_frames = 0;
	if (ghosts) {   /* it makes room for them by dropping its view's oldest short-term references first (headers.c:1095-1110) */
		int excess = -short_term_room(d) + ghosts;
		for (int i = 0; i < d->n_slots; i++) excess += in_view(d, i) && d->pics[i].ref == 1 && &d->pics[i] != p;
		while (excess-- > 0) {
			int old = -1;
			for (int i = 0; i < d->n_slots; i++) if (in_view(d, i) && d->pics[i].ref == 1 && &d->pics[i] != p && !(dropped >> i & 1) &&
			                                       (old < 0 || d->pics[i].frame_num < d->pics[old].frame_num)) old = i;
			if (old >= 0) dropped |= 1u << old;
		}
	}
	for (int i = 0; i < d->n_slots; i++) if (d->pics[i].in_use && ((d->pics[i].ref && !(dropped >> i & 1)) || d->pics[i].needed_for_output)) busy |= 1u << d->pics[i].ref_frame;
	for (int i = 0; i < E264_MAX_HOSTBUFS; i++) if (d->hb[i].state == 2 || (d->hb[i].state == 3 && d->hb[i].borrowed)) busy |= 1u << d->hb[i].ref_frame;
	for (int k = 0; k < ghosts && busy != ~0u; k++) { const int g = __builtin_ctz(~busy); d->ref_frame_view[g] = (uint8_t)d->view; busy |= 1u << g; }
	const int f = busy == ~0u ? 0 : __builtin_ctz(~busy);
	const int same = d->ref_frame_view[f] == d->view;
	d->ref_frame_view[f] = (uint8_t)d->view; p->ref_frame = f;
	if (p->host_buf >= 0) d->hb[p->host_buf].ref_frame = f;
	return same;
}

/* 8.2.5.2 gaps in frame_num (a reference picture was lost): like the reference (headers.c:1095-1139) insert
 * "non-existing" short-term frames for the missing numbers — they take FrameIds and list positions and push
 * older pictures out through the sliding window, which keeps the reference indices of the surviving pictures
 * what the encoder meant.  Their samples are undefined in the reference (never-written buffers); ours are
 * cleared.  Returns the number of frames inserted. */
static int fill_frame_num_gap(Edge264Decoder *d, int frame_num_abs) {
	const SPS *s = view_sps(d);
	int prev = d->prev_ref_frame_num[d->view];
	if (prev < 0 || frame_num_abs - prev <= 1) return 0;
	int room = short_term_room(d), nshort = 0;
	for (int i = 0; i < d->n_slots; i++) nshort += in_view(d, i) && d->pics[i].ref == 1;
	int gap_frames = frame_num_abs - prev - 1 < room ? frame_num_abs - prev - 1 : room;
	if (gap_frames < 0) gap_frames = 0;
	for (; gap_frames + nshort > room && nshort > 0; nshort--) {
		int old = -1;
		for (int i = 0; i < d->n_slots; i++) if (in_view(d, i) && d->pics[i].ref == 1 && (old < 0 || d->pics[i].frame_num < d->pics[old].frame_num)) old = i;
		d->pics[old].ref = 0; slot_release_if_unused(d, old);
	}
	if (gap_frames > 0) threads_drain(d, NULL);   /* the fills below go straight to the device: every earlier picture must be on its way first */
	for (int fn = frame_num_abs - gap_frames; fn < frame_num_abs; fn++) {
		int sl = find_free_slot(d);
		while (sl < 0 && bump_frame(d, d->view, -1)) sl = find_free_slot(d);
		if (sl < 0) { d->next_uid++; continue; }   /* no room even after bumping: keep at least the FrameId numbering */
		Pic *np = &d->pics[sl];
		memset(np, 0, sizeof(*np));
		np->in_use = 1; np->ref = 1; np->nonexisting = 1; np->frame_num = fn; np->uid = d->next_uid++; np->host_buf = -1; np->view = d->view;
		take_ref_frame(d, np);
		int npoc = 0;
		if (s->poc_type == 2) npoc = fn * 2;
		else if (s->poc_type == 1 && s->num_ref_frames_in_poc_cycle > 0) {
			int tot = 0, part = 0, in = fn % s->num_ref_frames_in_poc_cycle;
			for (int i = 0; i < s->num_ref_frames_in_poc_cycle; i++) { tot += s->offset_for_ref_frame[i]; if (i < in) part += s->offset_for_ref_frame[i]; }
			npoc = (fn / s->num_ref_frames_in_poc_cycle) * tot + part;   /* as the reference computes it (headers.c:1133-1139), not as 8.2.1 does */
		}
		np->poc = np->poc_dec = np->poc_top = np->poc_top_dec = npoc;
		for (int i = 0; i < E264_MAX_SLOTS; i++) np->slot_uid[i] = -1;
		if (d->be->fill_slot) { pthread_mutex_lock(&d->be_lock); d->be->fill_slot(d->be_ctx, sl, 0, d->luma_only ? 128 : 0); pthread_mutex_unlock(&d->be_lock); }
		d->taint |= 1u << sl;   /* its error map is all 100 */
	}
	d->prev_ref_frame_num[d->view] = frame_num_abs - 1;   /* the last inserted frame is the previous reference frame now (headers.c:1131) */
	return gap_frames;
}

/* FrameId numbering: the reference keeps an absolute FrameNum across IDRs, so an IDR after other pictures looks like a
 * frame_num gap and non-existing frames take FrameIds (headers.c:1059,1095-1139) */
static void number_frame_id(Edge264Decoder *d, int frame_num, int gap_frames) {
	int q = d->q_prev_ref_frame_num[d->view];
	int qfn = q + 1 + ((frame_num - q - 1) & ((1 << view_sps(d)->log2_max_frame_num) - 1));
	int gap = qfn - q;
	if (gap > 1 && !gap_frames) {   /* a real gap has just been given its frames (and FrameIds) by fill_frame_num_gap */
		int room = short_term_room(d), n = gap - 1 < room ? gap - 1 : room;
		if (n > 0) { d->next_uid += n; d->ghost_frames = n; }
	}
	if (gap > 1) d->q_prev_ref_frame_num[d->view] = qfn - 1;
	d->q_cur_frame_num = qfn;
}

/* the data side of a decoded picture d->cur in `slot`: its host buffer, build and staging; sets d->pb */
static int start_build(Edge264Decoder *d, int slot, int hbuf) {
	Pic *cp = &d->pics[slot];
	d->hb[hbuf].state = 1; d->hb[hbuf].frame_id = cp->uid; d->hb[hbuf].borrowed = 0; d->hb[hbuf].submitted = 0; d->hb[hbuf].err_pic = 0;
	PicBuild *pb = build_acquire(d, slot);     /* may wait for a worker to finish a picture */
	E264Staging stg; memset(&stg, 0, sizeof(stg));
	int ar;
	{ PROF_BEGIN; pthread_mutex_lock(&d->be_lock); ar = d->be->acquire_staging(d->be_ctx, slot, &stg); pthread_mutex_unlock(&d->be_lock); PROF_END(1); }
	if (ar) {   /* give the build back as if it had never been taken (no later picture exists yet) */
		pthread_mutex_lock(&d->lock); d->next_seq--; d->slot_users[slot]--; d->slot_build[slot] = NULL; pb->in_use = 0; pthread_mutex_unlock(&d->lock);
		cp->in_use = 0; d->cur = -1; d->hb[hbuf].state = 0;
		return ENOMEM;
	}
	cp->recs = stg.recs;
	pb->recs = stg.recs; pb->coefs = stg.coefs; pb->slices = stg.slices; pb->intra_list = stg.intra_list; pb->staging = stg.handle;
	pb->coef_cap = stg.coef_capacity; pb->n_coefs = 0; pb->n_slices = 0; pb->mbs_done = 0; pb->n_intra = 0; pb->any_deblock = 0;
	pb->slot = slot; pb->host_buf = hbuf; pb->conceal_ref = -1; pb->slice_counter = 0;
	memcpy(pb->slot_ids, cp->slot_uid, sizeof(pb->slot_ids));   /* slots may hold other pictures by the time this one is submitted */
	{ PROF_BEGIN; memset(pb->mbi, 0, (size_t)d->w_mbs * d->h_mbs * sizeof(MbInfo)); PROF_END(4); }
	/* records need no clearing: every macroblock of a complete picture rewrites its own (sx_one_mb) */
	d->pb = pb;
	return 0;
}

/* first slice of a picture: frame number, POC, FrameId, slot, the data side (start_build) unless the picture is skipped,
 * bumping; sets d->cur, d->cur_skip */
static int start_picture(Edge264Decoder *d, const SliceHeader *h, int idr, int nal_ref_idc) {
	const SPS *s = view_sps(d);
	const int v = d->view;
	int ret;
	if (d->outq_n[v] > 16) {
		/* the frame the application is told to fetch may still be with a parser: wait for it here, not in a polling
		 * loop (without workers every queued frame has been submitted, so this does not wait) */
		pthread_mutex_lock(&d->lock);
		while (!__atomic_load_n(&d->hb[d->outq[v][0]].submitted, __ATOMIC_ACQUIRE)) pthread_cond_wait(&d->done_cv, &d->lock);
		pthread_mutex_unlock(&d->lock);
		return ENOBUFS;
	}
	/* edge264_skip.h: decided once, at the picture's first slice; in a stereo sequence once per access unit, at its base view,
	 * whose inter_view_flag makes it a reference for NONREF, and the second view follows it */
	const int reference = nal_ref_idc || (d->mvc && d->inter_view_flag);
	const int skip = v ? d->au_skip : d->skip_mode == EDGE264_SKIP_NONREF ? !reference : d->skip_mode == EDGE264_SKIP_NONKEY ? !idr && h->slice_type != 2 : 0;
	int hbuf = -1;
	if (!skip && (hbuf = hostbuf_acquire(d)) < 0) return ENOBUFS;
	if (!v) d->au_skip = skip;
	/* edge264_latency.h: read at the picture's first slice, like the skip and loop filter modes */
	const int max_reorder = d->output_latency >= 0 && d->output_latency < s->max_num_reorder_frames ? d->output_latency : s->max_num_reorder_frames;
	d->low_latency = d->output_latency >= 0;
	/* absolute (unwrapped) frame numbers like the reference (headers.c:1059) */
	int prev = d->prev_ref_frame_num[v];
	int frame_num_abs = idr ? 0 : prev + 1 + ((h->frame_num - prev - 1) & ((1 << s->log2_max_frame_num) - 1));
	if (idr) { d->prev_ref_frame_num[v] = -1; d->prev_ref_poc[v] = 0; }
	int poc, poc_top;
	picture_poc(d, h, idr, nal_ref_idc, frame_num_abs, &poc, &poc_top);
	int gap_frames = idr ? 0 : fill_frame_num_gap(d, frame_num_abs);

	int slot = find_free_slot(d);
	if (slot < 0) {   /* DPB invariant broken (stream exceeds its own limits): drop the oldest output-pending picture */
		if (!bump_frame(d, v, -1)) return EBADMSG;
		slot = find_free_slot(d);
		if (slot < 0) return ENOBUFS;
	}
	Pic *cp = &d->pics[slot];
	memset(cp, 0, sizeof(*cp));
	number_frame_id(d, idr ? 0 : h->frame_num, gap_frames);
	cp->in_use = 1; cp->frame_num = frame_num_abs; cp->poc = cp->poc_dec = poc; cp->poc_top = cp->poc_top_dec = poc_top; cp->uid = d->next_uid++; cp->host_buf = hbuf; cp->view = v;
	const int counted = take_ref_frame(d, cp);
	d->cur = slot; d->cur_idr = idr; d->cur_nal_ref_idc = nal_ref_idc; d->cur_skip = skip;
	d->first_sh = *h;
	for (int i = 0; i < E264_MAX_SLOTS; i++) cp->slot_uid[i] = d->pics[i].in_use ? d->pics[i].uid : -1;
	if (skip) {   /* no build, no staging: a non-existing frame whose slot is filled if a decoded picture ever predicts from it */
		cp->nonexisting = 1; cp->unfilled = nal_ref_idc != 0;
	} else {
		if ((ret = start_build(d, slot, hbuf))) return ret;
		/* edge264_loopfilter.h: decided once, at the picture's first slice, like the skip decision; for each view component,
		 * a base view with inter_view_flag counting as a reference */
		d->pb->no_deblock = d->loop_filter_mode == EDGE264_LOOP_FILTER_NONE || (d->loop_filter_mode == EDGE264_LOOP_FILTER_REF && !(v ? nal_ref_idc : reference));
		d->pb->close_complete = d->low_latency && d->n_threads;
	}

	/* IDR / MMCO5: every earlier picture leaves in output order first (reference headers.c:632, 680) */
	int has_mmco5 = 0;
	for (int k = 0; k < h->n_mmco; k++) if (h->mmco[k].op == 5) has_mmco5 = 1;
	if (idr || has_mmco5) {
		while (bump_frame(d, v, slot));
		if (has_mmco5) { cp->poc_top -= cp->poc; cp->poc = 0; }   /* tempPicOrderCnt subtraction (8.2.1) for output order and later pictures; frame_num restarts in apply_marking, once the picture's own lists and operations have used the real value */
	}
	/* C.4.5.3 bumping before insertion (reference headers.c:1229-1250), with max_num_reorder_frames capped by
	 * edge264_set_output_latency: the bumping of a stream whose VUI states that depth */
	int max_bump = s->max_num_ref_frames;
	if (!nal_ref_idc) {
		max_bump = 0;
		for (int i = 0; i < d->n_slots; i++) if (i != slot && in_view(d, i) && d->pics[i].needed_for_output && d->pics[i].poc_top < cp->poc_top) max_bump++;
	}
	while (dpb_fullness(d) >= s->max_dec_frame_buffering && max_bump--) bump_frame(d, v, slot);
	cp->needed_for_output = 1;   /* a skipped picture too: it leaves by bumping as in a full decode, without a buffer to queue */
	if (max_bump < 0) {   /* nothing may precede it: straight to the output queue (it is returned once decoded) */
		cp->needed_for_output = 0;
		if (!skip) { d->hb[hbuf].state = 2; d->outq[v][d->outq_n[v]++] = hbuf; }
	} else if (waiting_for_output(d) - !counted > max_reorder) bump_frame(d, v, -1);
	/* POC bookkeeping for the next picture (8.2.1.1) */
	if (nal_ref_idc) { d->prev_ref_poc[v] = has_mmco5 ? cp->poc_top : poc_top; }
	if (has_mmco5) d->prev_ref_frame_num[v] = 0;
	return 0;
}

/* 8.4.2.3.1 implicit weights from POC distances */
static void implicit_weights(const SliceCtx *c, E264SliceRec *sr) {
	for (int i0 = 0; i0 < c->num_ref[0] && i0 < 16; i0++) for (int i1 = 0; i1 < c->num_ref[1] && i1 < 16; i1++) {
		int w1 = 32;
		if (c->ref_uid[0][i0] >= 0 && c->ref_uid[1][i1] >= 0 && !c->ref_long[0][i0] && !c->ref_long[1][i1]) {
			int poc0 = c->ref_poc[0][i0], poc1 = c->ref_poc[1][i1];
			int tb = c->cur_poc - poc0, td = poc1 - poc0;
			tb = tb < -128 ? -128 : tb > 127 ? 127 : tb; td = td < -128 ? -128 : td > 127 ? 127 : td;
			if (td != 0) {
				int tx = (16384 + (td < 0 ? -td : td) / 2) / td;
				int dsf = (tb * tx + 32) >> 6; dsf = dsf < -1024 ? -1024 : dsf > 1023 ? 1023 : dsf;
				if ((dsf >> 2) >= -64 && (dsf >> 2) <= 128) w1 = dsf >> 2;
			}
		}
		sr->implicit_w1[i0][i1] = (int16_t)w1;
	}
}

/* A skipped reference picture named by a decoded picture's reference list gets its samples now, like the frames of a
 * frame_num gap (edge264_skip.h): a constant, and an error map of 100 that the taint carries into the predicting picture.
 * The fill goes straight to the device, after every earlier picture and before the current one. */
static void fill_skipped(Edge264Decoder *d, int slot) {
	if (!d->pics[slot].unfilled) return;
	d->pics[slot].unfilled = 0;
	threads_drain(d, d->pb);
	if (d->be->fill_slot) { pthread_mutex_lock(&d->be_lock); d->be->fill_slot(d->be_ctx, slot, 0, d->luma_only ? 128 : 0); pthread_mutex_unlock(&d->be_lock); }
	d->taint |= 1u << slot;
}

/* slice record (deblocking, weights, scaling lists) and parsing context (reference lists, co-located slot in *col_slot) */
static int setup_slice(Edge264Decoder *d, const PPS *p, const SliceHeader *h, const BitReader *b, SliceJob *job, int *col_slot) {
	const SPS *s = view_sps(d);
	PicBuild *pb = d->pb;
	if (pb->n_slices >= E264_MAX_SLICES) return ENOTSUP;
	Pic *cp = &d->pics[d->cur];
	if (h->first_mb >= d->w_mbs * d->h_mbs) return EBADMSG;

	/* a picture without the loop filter (edge264_loopfilter.h) gets the records of disable_deblocking_filter_idc 1; its
	 * header keeps the values it was parsed with */
	const int deblock_idc = pb->no_deblock ? 1 : h->deblock_idc;
	E264SliceRec *sr = &pb->slices[pb->n_slices];
	memset(sr, 0, sizeof(*sr));
	if (deblock_idc != 1) { sr->filter_offset_a = (int8_t)h->filter_offset_a; sr->filter_offset_b = (int8_t)h->filter_offset_b; }
	sr->deblock_idc = (uint8_t)deblock_idc; sr->slice_type = (uint8_t)h->slice_type;
	merge_scaling(s, p, sr);

	SliceCtx *c = &job->sc;
	*col_slot = -1;
	c->cabac = p->entropy_coding_mode;
	c->w_mbs = d->w_mbs; c->h_mbs = d->h_mbs;
	c->slice_type = h->slice_type; c->slice_id = ++pb->slice_counter; c->slice_idx = pb->n_slices;
	c->num_ref[0] = h->num_ref[0]; c->num_ref[1] = h->num_ref[1];
	c->direct_spatial = h->direct_spatial; c->direct_8x8_inference = s->direct_8x8_inference; c->transform_8x8_mode = p->transform_8x8_mode;
	c->qp = h->slice_qp; c->chroma_qp_offset[0] = p->chroma_qp_index_offset[0]; c->chroma_qp_offset[1] = p->chroma_qp_index_offset[1];
	c->deblock_idc = deblock_idc; c->cur_poc = cp->poc_dec;
	c->mbi = pb->mbi; c->recs = pb->recs; c->coefs = pb->coefs; c->coef_cap = pb->coef_cap;   /* n_coefs: build_work continues the pool where the previous slice ended */
	c->col_recs = NULL; c->col_slot_uid = NULL; c->error = 0; c->n_intra = 0; c->missing_ref = 0; c->any_err = 0; c->luma_only = d->luma_only;
	memset(c->ref_slot, -1, sizeof(c->ref_slot)); memset(c->ref_long, 0, sizeof(c->ref_long));
	for (int l = 0; l < 2; l++) for (int i = 0; i < 32; i++) { c->ref_uid[l][i] = -1; c->ref_poc[l][i] = 0; }
	if (h->slice_type < 2) {
		int lists[2][32], nl[2];
		build_ref_lists(d, h, lists, nl);
		for (int l = 0; l <= (h->slice_type == 1); l++) for (int i = 0; i < h->num_ref[l]; i++) if (lists[l][i] >= 0) fill_skipped(d, lists[l][i]);
		for (int l = 0; l <= (h->slice_type == 1); l++) {
			/* a missing entry (damaged or non-conforming stream) is predicted from a defined picture other than the one
			 * being decoded: the list's first present entry, else the picture concealment copies from.  It keeps
			 * ref_uid -1, so direct prediction and implicit weights still see it as missing. */
			int subst = -1;
			for (int i = 0; i < h->num_ref[l] && subst < 0; i++) subst = lists[l][i];
			if (subst < 0) subst = conceal_reference(d);
			if (subst < 0) return EBADMSG;   /* nothing to predict from: the slice is not decoded */
			for (int i = 0; i < h->num_ref[l]; i++) {
				int sl = lists[l][i];
				c->ref_slot[l][i] = (int8_t)(sl < 0 ? subst : sl);
				pb->ref_mask |= 1u << c->ref_slot[l][i];
				if (sl < 0) { c->missing_ref = 1; continue; }
				c->ref_uid[l][i] = d->pics[sl].uid; c->ref_poc[l][i] = d->pics[sl].poc; c->ref_long[l][i] = d->pics[sl].ref == 2;
			}
		}
		if (h->slice_type == 1 && lists[1][0] >= 0) {
			c->col_recs = d->pics[lists[1][0]].recs;
			if (d->pics[lists[1][0]].nonexisting) c->col_recs = NULL; else *col_slot = lists[1][0];
			/* the co-located picture's Pic entry may be recycled before this slice is parsed: keep a private copy of the uid table */
			memcpy(job->col_slot_uid, d->pics[lists[1][0]].slot_uid, sizeof(job->col_slot_uid)); c->col_slot_uid = job->col_slot_uid;
		}
		int wp = h->slice_type == 0 ? p->weighted_pred_flag : p->weighted_bipred_idc;
		sr->wp_mode = (uint8_t)wp; sr->luma_log2_wd = (uint8_t)h->luma_log2_wd; sr->chroma_log2_wd = (uint8_t)h->chroma_log2_wd;
		if (wp == 1) for (int l = 0; l < 2; l++) for (int i = 0; i < 16; i++) for (int k = 0; k < 3; k++) { sr->wp_w[l][i][k] = h->w[l][i][k]; sr->wp_o[l][i][k] = h->o[l][i][k]; }
		if (wp == 1 && d->luma_only) {   /* chroma weights that keep 128 at 128 (edge264_enable_luma_only) */
			sr->chroma_log2_wd = 0;
			for (int l = 0; l < 2; l++) for (int i = 0; i < 16; i++) for (int k = 1; k < 3; k++) { sr->wp_w[l][i][k] = 1; sr->wp_o[l][i][k] = 0; }
		}
		if (wp == 2) implicit_weights(c, sr);
	}
	pb->n_slices++;
	if (deblock_idc != 1) pb->any_deblock = 1;

	c->br = *b;
	c->mbaddr = h->first_mb;
	c->cabac_init_idc_col = h->slice_type == 2 ? 0 : 1 + h->cabac_init_idc;
	return 0;
}

/* Low-latency output with workers: a slice that continues the current picture may arrive after a worker has closed it
 * (its slices already covered every macroblock).  build_hold returns 1 when that happened: the slice then starts a new
 * picture, as it does without workers.  Otherwise the picture stays open until the slice is queued (slice_enqueue) or
 * dropped (build_release, which closes the picture if it became complete meanwhile). */
static int build_hold(Edge264Decoder *d) {
	pthread_mutex_lock(&d->lock);
	const int closed = d->pb->closed;
	d->pb->held = !closed;
	pthread_mutex_unlock(&d->lock);
	return closed;
}
static void build_release(Edge264Decoder *d) {
	PicBuild *pb = d->pb;
	if (!pb || !pb->held) return;
	pthread_mutex_lock(&d->lock);
	pb->held = 0;
	if (!pb->head && !pb->running && pb->mbs_done >= d->w_mbs * d->h_mbs) { pb->closed = 1; pthread_cond_broadcast(&d->work_cv); }
	pthread_mutex_unlock(&d->lock);
}

/* Parses the slice header, starts a picture when it is the first slice of one and queues the slice's data on the
 * picture's build.  *jobp is set to NULL once the job is queued; until then it stays the caller's. */
static int decode_slice(Edge264Decoder *d, int nal_unit_type, int nal_ref_idc, int view, int idr, BitReader *b, SliceJob **jobp) {
	SliceHeader *h = &d->sh;
	const PPS *p = NULL;
	const SPS *s = view ? &d->ssps : &d->sps;
	int ret = parse_slice_header(d, s, b, nal_unit_type, idr, nal_ref_idc, h, &p);
	if (ret) return ret;
	if (!d->configured) return EBADMSG;

	/* 7.4.1.2.4 first slice of a new picture? (same tests as the reference, headers.c:1027-1050, the view included) */
	if (d->cur >= 0) {
		const SliceHeader *f = &d->first_sh;
		int newpic = h->frame_num != f->frame_num || (nal_ref_idc > 0) != (d->cur_nal_ref_idc > 0) || h->idr_pic_id != f->idr_pic_id ||
		             (s->poc_type == 0 && h->poc_lsb != f->poc_lsb) || (s->poc_type == 1 && h->delta_poc[0] != f->delta_poc[0]) ||
		             view != d->pics[d->cur].view;
		if (!newpic && d->pb && d->pb->close_complete) newpic = build_hold(d);
		if (newpic) { ret = finish_picture(d); if (ret) return ret; }
	}
	d->view = view;
	if (d->cur < 0 && (ret = start_picture(d, h, idr, nal_ref_idc))) return ret;
	if (d->cur_skip) return h->first_mb >= d->w_mbs * d->h_mbs ? EBADMSG : 0;   /* its slice data is never parsed */
	int col_slot;
	if ((ret = setup_slice(d, p, h, b, *jobp, &col_slot))) { build_release(d); return ret; }
	PicBuild *pb = d->pb;
	slice_enqueue(d, pb, *jobp, col_slot);
	*jobp = NULL;
	/* With workers, one of them parses the slice data and errors in it are not reported; the picture is closed by the
	 * next picture's first slice, a flush, the end of the sequence or of the stream.  Without workers, the slice is
	 * parsed here, its error is returned, and the picture is closed and submitted as soon as it is complete. */
	if (d->n_threads) return 0;
	{ PROF_BEGIN; pthread_mutex_lock(&d->lock); ret = build_work(d, pb); pthread_mutex_unlock(&d->lock); PROF_END(0); }
	if (pb->mbs_done >= d->w_mbs * d->h_mbs) { int r2 = finish_picture(d); if (!ret) ret = r2; }
	return ret;
}

/* ------------------------------------------------------------------------------------------ */
/* public API                                                                                   */
/* ------------------------------------------------------------------------------------------ */
Edge264Decoder *edge264_alloc(int n_threads, Edge264LogCb log_cb, void *log_arg, int log_mbs,
                              Edge264AllocCb alloc_cb, Edge264FreeCb free_cb, void *alloc_arg) {
	(void)log_mbs;
	if (prof_on < 0) { const char *e = getenv("E264_HOST_PROFILE"); prof_on = e && atoi(e); }
	if (log_cb) return NULL;   /* like a reference build without the logs variant (edge264.c:217-220) */
	Edge264Decoder *d = (Edge264Decoder *)calloc(1, sizeof(*d));
	if (!d) return NULL;
	d->alloc_cb = (alloc_cb && free_cb) ? alloc_cb : NULL; d->free_cb = free_cb; d->alloc_arg = alloc_arg;
	d->cur = -1; d->base_slot = -1; d->inter_view_flag = 1; d->output_latency = -1;
	for (int v = 0; v < 2; v++) { d->pending_release[v] = -1; d->prev_ref_frame_num[v] = -1; d->q_prev_ref_frame_num[v] = -1; }
	d->be = e264_default_backend();
	if (!d->be || d->be->create(&d->be_ctx)) { free(d); return NULL; }
	d->n_builds = 1;
	pthread_mutex_init(&d->lock, NULL); pthread_mutex_init(&d->be_lock, NULL);
	pthread_cond_init(&d->work_cv, NULL); pthread_cond_init(&d->done_cv, NULL);
	/* n_threads as in the reference (edge264.c:223-257): 0 = parse inside edge264_decode_NAL, < 0 = one worker per CPU up
	 * to the limit, > 0 = that many workers (here they parse slice data ahead; reconstruction is the device's) */
	{ const char *e = getenv("E264_SYNC_OUTPUT"); d->sync_output = e && atoi(e) != 0; d->block_output = d->sync_output; }
	if (n_threads < 0) { long n = sysconf(_SC_NPROCESSORS_ONLN); n_threads = n < 1 ? 1 : (int)n; }
	if (n_threads > E264_MAX_THREADS) n_threads = E264_MAX_THREADS;
	for (int i = 0; i < n_threads; i++) {
		if (pthread_create(&d->threads[i], NULL, worker_main, d)) { edge264_free(&d); return NULL; }
		d->n_threads = i + 1;
	}
	return d;
}

void edge264_flush(Edge264Decoder *d) {
	if (!d) return;
	finish_picture(d);
	threads_drain(d, NULL);
	/* drop every picture and the sequence state, keep parameter sets (reference edge264.c:261-270 clears them too) */
	for (int i = 0; i < E264_MAX_SLOTS; i++) { d->pics[i].in_use = 0; d->pics[i].host_buf = -1; }
	for (int i = 0; i < E264_MAX_HOSTBUFS; i++) if (d->hb[i].state != 3 || !d->hb[i].borrowed) d->hb[i].state = 0;
	d->cur = -1; d->base_slot = -1; d->inter_view_flag = 1;
	for (int v = 0; v < 2; v++) { d->outq_n[v] = 0; d->pending_release[v] = -1; d->prev_ref_frame_num[v] = -1; d->q_prev_ref_frame_num[v] = -1; d->prev_ref_poc[v] = 0; }
	memset(&d->sps, 0, sizeof(d->sps)); memset(d->pps, 0, sizeof(d->pps));
	memset(&d->ssps, 0, sizeof(d->ssps)); d->mvc = 0;   /* stereo off, like the reference's clear_decoder (headers.c:135-141) */
	memset(d->ref_frame_view, 0, sizeof(d->ref_frame_view));
	d->configured = 0;
}

void edge264_free(Edge264Decoder **pd) {
	Edge264Decoder *d;
	if (!pd || !(d = *pd)) return;
	*pd = NULL;
	if (prof_on > 0) { for (int i = 0; i < 6; i++) if (prof_n[i]) fprintf(stderr, "host profile: %-18s %8.3f ms total %6ld calls %8.1f us/call\n", prof_names[i], 1e3 * prof_t[i], prof_n[i], 1e6 * prof_t[i] / prof_n[i]); memset(prof_t, 0, sizeof(prof_t)); memset(prof_n, 0, sizeof(prof_n)); }
	finish_picture(d);
	threads_stop(d);
	hostbufs_free_all(d);
	d->be->destroy(d->be_ctx);
	for (int i = 0; i < E264_MAX_BUILDS; i++) free(d->builds[i].mbi);
	pthread_mutex_destroy(&d->lock); pthread_mutex_destroy(&d->be_lock);
	pthread_cond_destroy(&d->work_cv); pthread_cond_destroy(&d->done_cv);
	free(d->rbsp); free(d);
}

static int decode_NAL_inner(Edge264Decoder *d, const uint8_t *buf, const uint8_t *end, Edge264UnrefCb unref_cb, void *unref_arg);
int edge264_decode_NAL(Edge264Decoder *d, const uint8_t *buf, const uint8_t *end, Edge264UnrefCb unref_cb, void *unref_arg) {
	if (!d || !buf) return EINVAL;
	const int r = decode_NAL_inner(d, buf, end, unref_cb, unref_arg);
	d->block_output = r == ENOBUFS || r == ENODATA || buf >= end || d->sync_output;
	return r;
}
static int decode_NAL_inner(Edge264Decoder *d, const uint8_t *buf, const uint8_t *end, Edge264UnrefCb unref_cb, void *unref_arg) {
	for (int v = 0; v < 2; v++) if (d->pending_release[v] >= 0) { d->hb[d->pending_release[v]].state = 0; d->pending_release[v] = -1; }
	if (buf >= end) {
		int r = bump_all(d);
		return r ? r : ENODATA;
	}
	int nal_ref_idc = buf[0] >> 5, nal_unit_type = buf[0] & 31;
	size_t n = (size_t)(end - buf) - 1;
	if (nal_unit_type == 1 || nal_unit_type == 5 || nal_unit_type == 20) {   /* the slice data is parsed from its own copy of the payload, possibly later */
		/* NAL unit 20: nal_unit_header_mvc_extension (H.7.3.1.1), then a slice of the second view with the subset SPS and its
		 * view's DPB (reference headers.c:1309-1332) */
		const int view = nal_unit_type == 20;
		if (view && !d->mvc) return EBADMSG;   /* no subset SPS: like a slice without its parameter set */
		d->slices_seen = 1;
		SliceJob *job = (SliceJob *)calloc(1, sizeof(SliceJob));
		/* slack: the slice parsers test for an overrun once per macroblock, so a damaged slice reads past its end */
		uint8_t *rb = job ? (uint8_t *)malloc(n + 4096) : NULL;
		if (!rb) { free(job); return ENOMEM; }
		size_t rn = e264_unescape(rb, buf + 1, n);
		memset(rb + rn, 0, 32);
		job->rbsp = rb;
		BitReader b; br_init(&b, rb, rn);
		int idr = nal_unit_type == 5, ret = 0;
		if (view) {
			const uint32_t x = br_u(&b, 24);
			idr = !(x >> 22 & 1);   /* non_idr_flag */
			ret = x >> 23 ? ENOTSUP : 0;   /* svc_extension_flag */
		}
		if (!(view && ret)) ret = decode_slice(d, nal_unit_type, nal_ref_idc, view, idr, &b, &job);
		if (!view) d->inter_view_flag = 1;   /* inferred for a base view slice without a prefix NAL unit (H.7.4.1.1) */
		if (job) { free(rb); free(job); }      /* not queued */
		if (ret == 0 && unref_cb) unref_cb(0, unref_arg);
		return ret;
	}
	if (d->rbsp_cap < n + 64) { free(d->rbsp); d->rbsp_cap = n * 2 + 4096; d->rbsp = (uint8_t *)malloc(d->rbsp_cap); if (!d->rbsp) { d->rbsp_cap = 0; return ENOMEM; } }
	size_t rn = e264_unescape(d->rbsp, buf + 1, n);
	memset(d->rbsp + rn, 0, 32);
	BitReader b; br_init(&b, d->rbsp, rn);
	int ret;
	switch (nal_unit_type) {
	case 7: {
		SPS s; ret = parse_sps(d, &b, &s, 0);
		if (ret == 0) {
			int same_format = d->configured && d->sps.width_mbs == s.width_mbs && d->sps.height_mbs == s.height_mbs && !memcmp(d->sps.crop, s.crop, sizeof(s.crop));
			int fits = same_format && s.max_num_ref_frames + 2 + (d->mvc ? d->ssps.max_num_ref_frames : 0) <= d->n_slots;
			if (!fits) {
				if (d->configured && bump_all(d)) return ENOBUFS;   /* frame format change: drain first (headers.c:2005-2007) */
				ret = configure_sequence(d, &s, same_format);
				if (ret) return ret;
				if (!same_format) memset(d->pps, 0, sizeof(d->pps));   /* a format change clears the decoder, PPSs included (reference clear_decoder, headers.c:133-141) */
			}
			d->sps = s;
		}
		break; }
	case 15: {   /* subset SPS: turns stereo decoding on (edge264_mvc.h) */
		SPS s; ret = parse_sps(d, &b, &s, 1);
		if (ret) break;
		/* the second view has the frame format of its base, and both views' references fit in the 32 frame slots; otherwise
		 * the stream is decoded as its base view alone */
		if (!d->configured || d->sps.width_mbs != s.width_mbs || d->sps.height_mbs != s.height_mbs || memcmp(d->sps.crop, s.crop, sizeof(s.crop)) ||
		    s.max_num_ref_frames > 15 || d->sps.max_num_ref_frames + s.max_num_ref_frames + 2 > E264_MAX_SLOTS) { ret = ENOTSUP; break; }
		if (!d->mvc || d->sps.max_num_ref_frames + s.max_num_ref_frames + 2 > d->n_slots) {   /* more frame slots: drain first, like a format change */
			if (bump_all(d)) return ENOBUFS;
			d->mvc = 1; d->ssps = s;
			if ((ret = configure_sequence(d, &d->sps, 1))) return ret;
		}
		d->ssps = s;
		break; }
	case 14: {   /* prefix NAL unit: nal_unit_header_mvc_extension of the base view slice that follows */
		const uint32_t x = br_u(&b, 24);
		if (b.overrun) { ret = EBADMSG; break; }
		if (x >> 23) { ret = ENOTSUP; break; }   /* svc_extension_flag */
		d->inter_view_flag = x >> 1 & 1;
		ret = 0;
		break; }
	case 8: ret = parse_pps(d, &b); break;
	case 10:   /* end of sequence; a stereo sequence is output in full and the decoder goes back to single view (reference headers.c:143-151) */
		if (d->mvc) {
			if (bump_all(d)) return ENOBUFS;
			const int b = d->base_slot;
			d->mvc = 0; d->base_slot = -1; memset(&d->ssps, 0, sizeof(d->ssps));
			for (int v = 0; v < 2; v++) { d->q_prev_ref_frame_num[v] = -1; d->prev_ref_poc[v] = 0; }   /* the reference clears its decoder here */
			memset(d->ref_frame_view, 0, sizeof(d->ref_frame_view));
			if (b >= 0) slot_release_if_unused(d, b);
		}
		ret = 0; if (d->cur >= 0) finish_picture(d); d->prev_ref_frame_num[0] = d->prev_ref_frame_num[1] = -1; break;
	case 6: case 9: case 11: case 12: ret = 0; break;
	default: ret = ENOTSUP;
	}
	if (ret == 0 && unref_cb) unref_cb(0, unref_arg);
	return ret;
}

/* Low-latency output: waits until the picture in host buffer hbuf has been handed to the backend if it is closed, that is
 * if no slice can join it any more and only workers still parse it.  Returns whether it has been handed over; an open
 * picture is never waited for, since its next slices have not been passed in yet. */
static int wait_submitted(Edge264Decoder *d, int hbuf) {
	pthread_mutex_lock(&d->lock);
	for (;;) {
		if (__atomic_load_n(&d->hb[hbuf].submitted, __ATOMIC_ACQUIRE)) break;
		const PicBuild *pb = NULL;
		for (int i = 0; i < d->n_builds; i++) if (d->builds[i].in_use && d->builds[i].host_buf == hbuf) pb = &d->builds[i];
		if (!pb || !pb->closed) break;
		pthread_cond_wait(&d->done_cv, &d->lock);   /* not reached without workers: closing a picture submits it */
	}
	pthread_mutex_unlock(&d->lock);
	return __atomic_load_n(&d->hb[hbuf].submitted, __ATOMIC_ACQUIRE);
}
/* 0: the picture in host buffer hbuf may be output; ENOMSG: not yet; EIO: device error.  Like the reference in threaded mode
 * (edge264.c:373: a frame whose last macroblock is not deblocked yet answers ENOMSG), a picture still on the device is "not
 * available yet" — unless the last decode_NAL told the application to fetch frames (ENOBUFS, end of stream) or the decoder
 * is in low-latency output (edge264_latency.h): then the call waits, so that no application loop ever has to poll. */
static int output_ready(Edge264Decoder *d, int hbuf) {
	HostBuf *hb = &d->hb[hbuf];
	/* queued at insertion but still being parsed */
	if (!__atomic_load_n(&hb->submitted, __ATOMIC_ACQUIRE) && !(d->low_latency && wait_submitted(d, hbuf))) return ENOMSG;
	if (!d->block_output && !d->low_latency) {
		int pr = d->be->poll(d->be_ctx, hb->ticket);
		if (pr == EAGAIN) return ENOMSG;
		if (pr) return EIO;
	}
	{ PROF_BEGIN; int wr = d->be->wait(d->be_ctx, hb->ticket); PROF_END(3); if (wr) return EIO; }
	return 0;
}
/* the samples (cropped) and error map of host buffer hb */
static void frame_planes(const Edge264Decoder *d, const HostBuf *hb, const Edge264Frame *fmt, const uint8_t *samples[3]) {
	int top = fmt->frame_crop_offsets[0], left = fmt->frame_crop_offsets[3];
	samples[0] = hb->p + top * d->stride_y + left;
	samples[1] = hb->p + d->plane_y + (top >> 1) * d->stride_c + (left >> 1);
	samples[2] = samples[1] + (d->stride_c >> 1);
}
static void frame_map(const Edge264Decoder *d, const HostBuf *hb, Edge264Frame *out) {
	out->mb_errors = NULL; out->stride_mb = d->out_fmt.stride_mb;
	/* the map was written for this picture only if some macroblock could be wrong; a map of zeros is reported as none */
	if (hb->err_pic) {
		const size_t nmb = (size_t)d->w_mbs * d->h_mbs;
		size_t k = 0;
		while (k < nmb && !hb->map[k]) k++;
		if (k < nmb) { out->mb_errors = hb->map; out->stride_mb = (int16_t)d->w_mbs; }
	}
}
/* return_arg of an output frame: host buffer + 1 of the base view in bits 0-7, of the second view in bits 8-15 */
static int frame_hostbuf(const Edge264Frame *f, int view) {
	const uintptr_t a = (uintptr_t)f->return_arg;
	return a >> 16 ? -1 : (int)(a >> (8 * view) & 255) - 1;
}

int edge264_get_frame(Edge264Decoder *d, Edge264Frame *out, int borrow) {
	if (!d || !out) return EINVAL;
	/* a stereo sequence outputs a pair once both views of the access unit are ready (reference edge264.c:365-407) */
	if (d->outq_n[0] == 0 || (d->mvc && d->outq_n[1] == 0)) return ENOMSG;
	const int pair = d->outq_n[1] > 0, h0 = d->outq[0][0], h1 = pair ? d->outq[1][0] : -1;
	int r = output_ready(d, h0);
	if (!r && pair) r = output_ready(d, h1);
	if (r) return r;
	*out = d->out_fmt;
	for (int v = 0; v <= pair; v++) {
		const int h = v ? h1 : h0;
		memmove(d->outq[v], d->outq[v] + 1, (size_t)(--d->outq_n[v]) * sizeof(int));
		d->hb[h].state = 3; d->hb[h].borrowed = borrow != 0;
		if (!borrow) d->pending_release[v] = h;   /* valid until the next decode_NAL, as in the reference */
	}
	frame_planes(d, &d->hb[h0], out, out->samples);
	out->FrameId = d->hb[h0].frame_id;
	frame_map(d, &d->hb[h0], out);
	out->return_arg = (void *)(uintptr_t)(h0 + 1);
	if (pair) {
		frame_planes(d, &d->hb[h1], out, out->samples_mvc);
		out->FrameId_mvc = d->hb[h1].frame_id;
		out->return_arg = (void *)(uintptr_t)((h0 + 1) | (h1 + 1) << 8);
	}
	return 0;
}

void edge264_return_frame(Edge264Decoder *d, void *return_arg) {
	if (!d) return;
	const Edge264Frame f = {.return_arg = return_arg};
	for (int v = 0; v < 2; v++) {
		const int i = frame_hostbuf(&f, v);
		if (i >= 0 && i < E264_MAX_HOSTBUFS && d->hb[i].state == 3) {
			d->hb[i].state = 0; d->hb[i].borrowed = 0;
			for (int w = 0; w < 2; w++) if (d->pending_release[w] == i) d->pending_release[w] = -1;
		}
	}
}

/* ------------------------------------------------------------------------------------------ */
/* stereo frames (include/edge264_mvc.h)                                                        */
/* ------------------------------------------------------------------------------------------ */
int edge264_get_second_view(Edge264Decoder *d, const Edge264Frame *frame, Edge264Frame *out) {
	if (!d || !frame || !out) return EINVAL;
	const int h0 = frame_hostbuf(frame, 0), h1 = frame_hostbuf(frame, 1);
	if (h0 < 0 || h0 >= E264_MAX_HOSTBUFS || d->hb[h0].state != 3) return EINVAL;
	if (h1 < 0) return ENOENT;
	if (h1 >= E264_MAX_HOSTBUFS || d->hb[h1].state != 3) return EINVAL;
	*out = *frame;
	for (int p = 0; p < 3; p++) { out->samples[p] = frame->samples_mvc[p]; out->samples_mvc[p] = NULL; }
	out->FrameId = frame->FrameId_mvc; out->FrameId_mvc = 0;
	frame_map(d, &d->hb[h1], out);
	out->return_arg = (void *)(uintptr_t)(h1 + 1);   /* a mono frame of its own for the output getters */
	return 0;
}

/* ------------------------------------------------------------------------------------------ */
/* motion export (include/edge264_motion.h)                                                     */
/* ------------------------------------------------------------------------------------------ */
int edge264_enable_motion(Edge264Decoder *d) {
	if (!d) return EINVAL;
	if (!d->be->submit_motion) return ENOTSUP;
	if (d->slices_seen) return EBUSY;   /* host buffers are created with the first picture: they would lack the export */
	d->motion = 1;
	return 0;
}

int edge264_get_motion(Edge264Decoder *d, const Edge264Frame *frame, Edge264Motion *out) {
	if (!d || !frame || !out) return EINVAL;
	if (!d->motion) return ENOENT;
	const int i = frame_hostbuf(frame, 0);
	if (i < 0 || i >= E264_MAX_HOSTBUFS || d->hb[i].state != 3 || !d->hb[i].motion) return EINVAL;
	const size_t nmb = (size_t)d->w_mbs * d->h_mbs;
	const uint8_t *m = d->hb[i].motion;
	out->mv = (const int16_t *)(m + E264_MOTION_MV * nmb);
	out->ref_frame_id = (const int32_t *)(m + E264_MOTION_REF * nmb);
	out->mb_type = m + E264_MOTION_TYPE * nmb;
	out->mb_qp = m + E264_MOTION_QP * nmb;
	out->width_mbs = d->w_mbs; out->height_mbs = d->h_mbs;
	out->on_device = d->hb[i].motion_dev;
	return 0;
}

/* ------------------------------------------------------------------------------------------ */
/* packed output (include/edge264_packed.h)                                                     */
/* ------------------------------------------------------------------------------------------ */
int edge264_enable_packed(Edge264Decoder *d, int format, int log2_scale) {
	if (!d || (format != EDGE264_PACKED_I420 && format != EDGE264_PACKED_NV12) || log2_scale < 0 || log2_scale > 3) return EINVAL;
	if (!d->be->submit_outputs) return ENOTSUP;
	if (d->slices_seen) return EBUSY;   /* host buffers are created with the first picture: they would lack the packed one */
	d->packed = 1; d->packed_format = format; d->packed_scale = log2_scale;
	return 0;
}

int edge264_enable_resized(Edge264Decoder *d, int format, int width, int height) {
	if (!d || (format != EDGE264_PACKED_I420 && format != EDGE264_PACKED_NV12) || ((width | height) & 1) || width < 0 || height < 0 ||
	    width > 16384 || height > 16384 || (width | height) == 0) return EINVAL;
	if (!d->be->submit_outputs) return ENOTSUP;
	if (d->slices_seen) return EBUSY;   /* host buffers are created with the first picture: they would lack the resized one */
	d->packed = 1; d->packed_format = format; d->packed_scale = -1; d->packed_width = width; d->packed_height = height;
	return 0;
}

int edge264_get_packed(Edge264Decoder *d, const Edge264Frame *frame, Edge264Packed *out) {
	if (!d || !frame || !out) return EINVAL;
	if (!d->packed) return ENOENT;
	const int i = frame_hostbuf(frame, 0);
	if (i < 0 || i >= E264_MAX_HOSTBUFS || d->hb[i].state != 3 || !d->hb[i].packed) return EINVAL;
	const HostBuf *hb = &d->hb[i];
	const E264PackedLayout l = e264_packed_layout(&hb->pk);
	memset(out, 0, sizeof(*out));
	for (int p = 0; p < (hb->pk.format == E264_PACKED_NV12 ? 2 : 3); p++) { out->planes[p] = hb->packed + l.offset[p]; out->stride[p] = l.stride[p]; }
	out->width = l.width; out->height = l.height; out->width_C = l.width_C; out->height_C = l.height_C;
	out->format = hb->pk.format; out->log2_scale = hb->pk.log2_scale;
	out->on_device = hb->packed_dev;
	return 0;
}

/* ------------------------------------------------------------------------------------------ */
/* picture statistics (include/edge264_picstats.h)                                              */
/* ------------------------------------------------------------------------------------------ */
int edge264_enable_picstats(Edge264Decoder *d) {
	if (!d) return EINVAL;
	if (!d->be->submit_outputs) return ENOTSUP;
	if (d->slices_seen) return EBUSY;   /* host buffers are created with the first picture: they would lack the statistics */
	d->picstats = 1;
	return 0;
}

int edge264_get_picstats(Edge264Decoder *d, const Edge264Frame *frame, Edge264PicStats *out) {
	if (!d || !frame || !out) return EINVAL;
	if (!d->picstats) return ENOENT;
	const int i = frame_hostbuf(frame, 0);
	if (i < 0 || i >= E264_MAX_HOSTBUFS || d->hb[i].state != 3 || !d->hb[i].picstats) return EINVAL;
	const size_t nmb = (size_t)d->w_mbs * d->h_mbs;
	const uint8_t *s = d->hb[i].picstats;
	out->hist = (const uint32_t *)(s + E264_PICSTATS_HIST);
	out->sum = (const uint32_t *)(s + E264_PICSTATS_SUM);
	out->sum_sq = (const uint32_t *)(s + E264_PICSTATS_SUM_SQ(nmb));
	out->width_mbs = d->w_mbs; out->height_mbs = d->h_mbs;
	out->on_device = d->hb[i].picstats_dev;
	return 0;
}

/* ------------------------------------------------------------------------------------------ */
/* skipped pictures (include/edge264_skip.h)                                                    */
/* ------------------------------------------------------------------------------------------ */
int edge264_set_skip(Edge264Decoder *d, int mode) {
	if (!d || mode < EDGE264_SKIP_NONE || mode > EDGE264_SKIP_NONKEY) return EINVAL;
	d->skip_mode = mode;   /* read by start_picture only: the current picture keeps its decision */
	return 0;
}

/* ------------------------------------------------------------------------------------------ */
/* luma-only decoding (include/edge264_luma.h)                                                  */
/* ------------------------------------------------------------------------------------------ */
/* The records of a luma-only picture reconstruct a chroma plane of 128 on their own, whatever backend reconstructs them:
 * no chroma levels (sx_residual), chroma samples of I_PCM macroblocks set to 128 (mb_impl.h), explicit chroma weights 1 with
 * offset 0 and log2 denominator 0 (setup_slice), filled slots at 128 (fill_slot).  With every reference at 128, intra
 * prediction of every mode, interpolation, every weighting and the deblocking filter map a plane of 128 to itself.  The
 * device's luma-only kernels leave chroma alone and set it to 128 with a memset: both give the same frame. */
int edge264_enable_luma_only(Edge264Decoder *d) {
	if (!d) return EINVAL;
	if (d->slices_seen) return EBUSY;   /* the pictures of one stream are all decoded one way */
	d->luma_only = 1;
	return 0;
}

/* ------------------------------------------------------------------------------------------ */
/* skipping the loop filter (include/edge264_loopfilter.h)                                      */
/* ------------------------------------------------------------------------------------------ */
int edge264_set_loop_filter(Edge264Decoder *d, int mode) {
	if (!d || mode < EDGE264_LOOP_FILTER_ALL || mode > EDGE264_LOOP_FILTER_NONE) return EINVAL;
	d->loop_filter_mode = mode;   /* read by start_picture only: the current picture keeps its decision */
	return 0;
}

/* ------------------------------------------------------------------------------------------ */
/* low-latency output (include/edge264_latency.h)                                               */
/* ------------------------------------------------------------------------------------------ */
int edge264_set_output_latency(Edge264Decoder *d, int max_reorder) {
	if (!d || max_reorder < -1 || max_reorder > 16) return EINVAL;
	d->output_latency = max_reorder;   /* read by start_picture only: the current picture keeps its depth */
	return 0;
}
