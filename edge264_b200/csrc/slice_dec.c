/* slice_dec.c — the product-side instantiation of the shared slice-data code (parser direction). */
#include <pthread.h>
#include "mb_impl.h"

static pthread_once_t tables_once = PTHREAD_ONCE_INIT;   /* decoders are created and run from many threads at once */

int e264_parse_slice_data(SliceCtx *s) {
	pthread_once(&tables_once, sx_init_tables);
	s->skip_run = -1; s->last_qp_delta_nz = 0; s->prev_mb_skipped = 0;
	if (s->cabac) {
		size_t byte = (s->br.pos + 7) >> 3;                 /* cabac_alignment_one_bit */
		if (byte > s->br.size) { s->error = 1; return 0; }
		cabac_init_states(s->cd.state, s->cabac_init_idc_col, s->qp);
		cabac_dec_start(&s->cd, s->br.buf + byte, s->br.buf + s->br.size);
	}
	int total = s->w_mbs * s->h_mbs, n = 0;
	for (;;) {
		if (s->mbaddr < 0 || s->mbaddr >= total) { s->error = 1; break; }
		if (s->mbi[s->mbaddr].slice_id) { s->error = 1; break; }            /* already delivered by another slice of this picture */
		if (s->n_coefs + 408u > s->coef_cap) { s->error = 2; break; }        /* a macroblock takes at most 16+256+8+128 levels: the pool cannot overflow inside it */
		int end = sx_one_mb(s);
		/* a macroblock that failed to parse may have a partial record: it counts as not delivered, so the picture's
		 * concealment (decoder.c conceal_missing) gives it a complete one */
		if (s->error) { s->cur->slice_id = 0; break; }
		n++;
		if (s->cabac && cabac_dec_overrun(&s->cd)) { s->error = 1; break; }
		if (!s->cabac && s->br.overrun) { s->error = 1; break; }
		if (end) break;
		s->mbaddr++;
	}
	return n;
}
