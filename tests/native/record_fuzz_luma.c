/* record_fuzz_luma — the record fuzzer (record_fuzz.c, included as it is: same generator, same draws from the same seeds,
 * same geometries, contexts and pictures in flight) with luma-only pictures among the colour ones: each picture is drawn
 * luma-only (E264PicDesc.luma_only) or colour at random, from a random stream of its own so the records stay exactly
 * those record_fuzz draws.  The records keep their chroma coded bits and levels: the luma-only kernels must skip them.
 * record_fuzz.c compares the device's slot with the port's after every picture; here the port's slot of a luma-only
 * picture gets its chroma plane set to 128 (port_recon_luma), so that comparison covers the luma samples and the
 * chroma fill.
 * tests/test_luma_only.py builds and runs it.
 *   record_fuzz_luma [--cpu-only] [--lib libedge264_b200.so] [--seeds A-B] [--contexts M] [--inflight K] ...
 * Prints record_fuzz's coverage counters, then "luma_only_pictures" and "colour_pictures". */
#include <stdint.h>
#include "../../edge264_b200/csrc/records.h"
/* every picture record_fuzz.c draws passes through its record check, just after the draw and before the port and the
 * device see it: that is where the mode is drawn.  Its port reconstruction goes through port_recon_luma below. */
#define e264_check_records record_fuzz_check_hook
#define port_recon_picture port_recon_luma
#include "record_fuzz.c"
#undef e264_check_records
#undef port_recon_picture
void port_recon_picture(uint8_t *frames, const E264PicDesc *pd, const E264MbRec *recs, const int16_t *coefs, const E264SliceRec *slices);
int e264_check_records(const E264PicDesc *pd, const E264MbRec *recs, const int16_t *coefs, const E264SliceRec *slices,
                       const uint32_t *intra_list, int n_slots, char *why, int why_len);

static _Thread_local uint64_t rng_l = 0x94D049BB133111EBull;
static long n_luma, n_colour;
int record_fuzz_check_hook(const E264PicDesc *pd, const E264MbRec *recs, const int16_t *coefs, const E264SliceRec *slices,
                           const uint32_t *intra_list, int n_slots, char *why, int why_len) {
	rng_l ^= rng_l >> 12; rng_l ^= rng_l << 25; rng_l ^= rng_l >> 27;
	const int luma = (int)((rng_l * 0x2545F4914F6CDD1Dull) >> 63);
	((E264PicDesc *)pd)->luma_only = (uint8_t)luma;   /* run_picture's own local: it goes on to the port and the device */
	__atomic_add_fetch(luma ? &n_luma : &n_colour, 1, __ATOMIC_RELAXED);
	return e264_check_records(pd, recs, coefs, slices, intra_list, n_slots, why, why_len);
}

/* The drawn records of a luma-only picture carry chroma levels, chroma PCM samples and chroma weights (the decoder's
 * parser leaves none that would change a chroma plane of 128, decoder.c edge264_enable_luma_only).  The mode's
 * definition on the restatement: its reconstruction of every plane, then the chroma plane set to 128; no luma sample
 * depends on chroma. */
void port_recon_luma(uint8_t *frames, const E264PicDesc *pd, const E264MbRec *recs, const int16_t *coefs, const E264SliceRec *slices) {
	port_recon_picture(frames, pd, recs, coefs, slices);
	if (pd->luma_only) memset(frames + (size_t)pd->dst_slot * pd->frame_bytes + pd->plane_y, 128, (size_t)(pd->frame_bytes - pd->plane_y));
}

__attribute__((destructor)) static void print_modes(void) {
	printf("cov luma_only_pictures %ld\ncov colour_pictures %ld\n", n_luma, n_colour);
}
