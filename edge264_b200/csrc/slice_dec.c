/* slice_dec.c — the product-side instantiation of the shared slice-data code (parser direction). */
#include <pthread.h>
#include "mb_impl.h"

static pthread_once_t tables_once = PTHREAD_ONCE_INIT;   /* decoders are created and run from many threads at once */

/* p^k for a probability p sampled to 0..65536 (reference ppow, edge264_headers.c:266-275) */
static unsigned ppow(unsigned p65536, unsigned k) {
	unsigned r = 65536;
	for (; k; k >>= 1) {
		if (k & 1) r = (r * p65536) >> 16;
		p65536 = (p65536 * p65536) >> 16;
	}
	return r;
}

/* Error of the i-th of the num macroblocks a slice delivered before its data ended on an error, 0..100 (reference
 * recover_slice, edge264_headers.c:305-311): CAVLC spreads the error evenly over the slice, CABAC weighs every macroblock
 * by the chance (1-p)^d, p = 342/65536, that the damage reached it without ending the slice first; the last one is 100. */
static unsigned slice_error(int cabac, unsigned i, unsigned num) {
	unsigned p12800;
	if (!cabac) p12800 = ((i + 1) * 12800 + num - 1) / num;
	else {
		unsigned div = 65536 - ppow(65194, num);
		p12800 = ((div - (65536 - ppow(65194, num - 1 - i))) * 12800 + div - 1) / div;
	}
	return p12800 >> 7;
}

/* an inter macroblock that predicts from a reference-list entry with no picture behind it (decoder.c setup_slice gave it
 * a substitute): its samples are made up */
static int uses_missing_ref(const SliceCtx *s, const E264MbRec *r) {
	for (int l = 0; l < 2; l++) for (int i8 = 0; i8 < 4; i8++) {
		int ri = r->ref_idx[l][i8];
		if (ri >= 0 && ri < 32 && s->ref_uid[l][ri] < 0) return 1;
	}
	return 0;
}

int e264_parse_slice_data(SliceCtx *s) {
	pthread_once(&tables_once, sx_init_tables);
	s->skip_run = -1; s->last_qp_delta_nz = 0; s->prev_mb_skipped = 0;
	if (s->cabac) {
		size_t byte = (s->br.pos + 7) >> 3;                 /* cabac_alignment_one_bit */
		if (byte > s->br.size) { s->error = 1; return 0; }
		cabac_init_states(s->cd.state, s->cabac_init_idc_col, s->qp);
		cabac_dec_start(&s->cd, s->br.buf + byte, s->br.buf + s->br.size);
	}
	int total = s->w_mbs * s->h_mbs, n = 0, first = s->mbaddr;
	s->any_err = 0;
	for (;;) {
		if (s->mbaddr < 0 || s->mbaddr >= total) { s->error = 1; break; }
		if (s->mbi[s->mbaddr].slice_id) { s->error = 1; break; }            /* already delivered by another slice of this picture */
		if (s->n_coefs + 408u > s->coef_cap) { s->error = 2; break; }        /* a macroblock takes at most 16+256+8+128 levels: the pool cannot overflow inside it */
		int end = sx_one_mb(s);
		/* a macroblock that failed to parse may have a partial record: it counts as not delivered, so the picture's
		 * concealment (decoder.c conceal_missing) gives it a complete one */
		if (s->error) { s->cur->slice_id = 0; break; }
		n++;
		if (s->missing_ref && s->rec->kind == MBK_INTER && uses_missing_ref(s, s->rec)) { s->rec->err = 100; s->any_err = 1; }
		if (s->cabac && cabac_dec_overrun(&s->cd)) { s->error = 1; break; }
		if (!s->cabac && s->br.overrun) { s->error = 1; break; }
		if (end) break;
		s->mbaddr++;
	}
	/* delivered macroblocks keep their samples; the error map says how likely each one is to be wrong */
	if (s->error && n > 0) {
		for (int i = 0; i < n; i++) {
			E264MbRec *r = s->recs + first + i;
			unsigned e = slice_error(s->cabac, (unsigned)i, (unsigned)n);
			if (e > r->err) r->err = (uint8_t)e;
		}
		s->any_err = 1;
	}
	return n;
}
