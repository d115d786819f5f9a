/* port_dbk_backend.c — TEST INFRASTRUCTURE ONLY.  The CPU restatement's backend (oracle/port_backend.c) with every picture
 * written out for the deblocking test (tests/test_deblock_spec.py): when E264_DBK_DUMP names a file, each submit appends
 * the picture's E264PicDesc, records, slice records and levels, then the picture before deblocking, then the picture itself
 * (tests/picture_dumps.py reads the file).  Each configure and each fill_slot (the frames of a frame_num gap, decoder.c
 * fill_frame_num_gap, and skipped references, fill_skipped) is written as an entry of its own, so that the file says what every frame slot holds.  The
 * picture before deblocking is the same picture reconstructed from its records with MBF_DEBLOCK / MBF_EDGE_* cleared and
 * any_deblock 0 (a picture the record contract allows); it goes to a buffer of its own, and the picture is then
 * reconstructed as parsed, so the frame slots hold what they hold without the dump.  The test links this file with the
 * product's host sources (decoder.c, slice_dec.c) and -Wl,--wrap=e264_default_backend. */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../../edge264_b200/csrc/dec.h"

const E264Backend *__real_e264_default_backend(void);
static E264Backend dbk_backend;
static E264Staging staged[64];   /* by handle: what acquire_staging handed out */

enum { DUMP_PICTURE = 1, DUMP_FILL = 2, DUMP_CONFIGURE = 3 };   /* the tag before each entry */
static FILE *dump_open(void) {
	const char *path = getenv("E264_DBK_DUMP");
	return path && *path ? fopen(path, "ab") : NULL;
}
static int dbk_configure(void *ctx, const E264PicDesc *g, int n_slots) {
	const int r = __real_e264_default_backend()->configure(ctx, g, n_slots);
	FILE *f = r ? NULL : dump_open();
	if (f) { uint32_t tag = DUMP_CONFIGURE; int32_t n = n_slots; fwrite(&tag, 4, 1, f); fwrite(g, sizeof(*g), 1, f); fwrite(&n, 4, 1, f); fclose(f); }
	return r;
}
static int dbk_fill(void *ctx, int slot, int y, int c) {
	const int r = __real_e264_default_backend()->fill_slot(ctx, slot, y, c);
	FILE *f = r ? NULL : dump_open();
	if (f) { uint32_t tag = DUMP_FILL; int32_t v[3] = {slot, y, c}; fwrite(&tag, 4, 1, f); fwrite(v, 4, 3, f); fclose(f); }
	return r;
}
static int dbk_acquire(void *ctx, int slot, E264Staging *out) {
	const int r = __real_e264_default_backend()->acquire_staging(ctx, slot, out);
	if (!r && out->handle >= 0 && out->handle < 64) staged[out->handle] = *out;
	return r;
}
static int dbk_submit(void *ctx, const E264PicDesc *pd, uint8_t *host_out, uint64_t *ticket) {
	const E264Backend *real = __real_e264_default_backend();
	const char *path = getenv("E264_DBK_DUMP");
	if (!path || !*path || pd->staging < 0 || pd->staging >= 64) return real->submit(ctx, pd, host_out, ticket);
	const E264Staging *st = staged + pd->staging;
	const size_t nmb = (size_t)pd->width_mbs * pd->height_mbs;
	E264MbRec *recs = malloc(nmb * sizeof(E264MbRec));
	uint8_t *pre = malloc((size_t)pd->frame_bytes);
	if (!recs || !pre) return -1;
	memcpy(recs, st->recs, nmb * sizeof(E264MbRec));
	for (size_t a = 0; a < nmb; a++) st->recs[a].flags &= (uint8_t)~(MBF_DEBLOCK | MBF_EDGE_L | MBF_EDGE_T);
	E264PicDesc p0 = *pd; p0.any_deblock = 0;
	uint64_t t0;
	int r = real->submit(ctx, &p0, pre, &t0);
	memcpy(st->recs, recs, nmb * sizeof(E264MbRec));
	if (!r) r = real->wait(ctx, t0);
	if (!r) r = real->submit(ctx, pd, host_out, ticket);
	if (!r) r = real->wait(ctx, *ticket);
	FILE *f = r ? NULL : fopen(path, "ab");
	if (f) {
		uint32_t tag = DUMP_PICTURE;
		fwrite(&tag, 4, 1, f);
		fwrite(pd, sizeof(*pd), 1, f); fwrite(recs, sizeof(E264MbRec), nmb, f); fwrite(st->slices, sizeof(E264SliceRec), (size_t)pd->n_slices, f);
		fwrite(st->coefs, 2, (size_t)pd->n_coefs, f);
		fwrite(pre, 1, (size_t)pd->frame_bytes, f); fwrite(host_out, 1, (size_t)pd->frame_bytes, f);
		fclose(f);
	} else if (!r) r = -1;
	free(recs); free(pre);
	return r;
}
const E264Backend *__wrap_e264_default_backend(void) {
	dbk_backend = *__real_e264_default_backend();
	dbk_backend.name = "port-dbk";
	dbk_backend.configure = dbk_configure;
	dbk_backend.fill_slot = dbk_fill;
	dbk_backend.acquire_staging = dbk_acquire;
	dbk_backend.submit = dbk_submit;
	return &dbk_backend;
}
