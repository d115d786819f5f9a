/* record_fuzz_maps — the record fuzzer (record_fuzz.c, included as it is: same generator, same draws from the same seeds)
 * with error maps on top: every picture may get E264MbRec.err values and an E264PicDesc.err_pic / taint mask, drawn from a
 * random stream of their own so the records stay exactly those record_fuzz draws; after every picture the device's map
 * of the slot (e264b_slot_map) must equal the CPU restatement's (port_error_map.c), next to the samples record_fuzz
 * compares.  tests/test_mb_errors.py builds and runs it.
 *   record_fuzz_maps [--cpu-only] [--lib libedge264_b200.so] [--seeds A-B]
 * Prints record_fuzz's coverage counters and the "map_*" ones. */
#define main record_fuzz_main
#include "record_fuzz.c"
#undef main

void port_error_map(uint8_t *maps, const E264PicDesc *pd, const E264MbRec *recs);
extern long port_cov_map[12];

static int (*slot_map)(void *, int, uint8_t *);
static int (*submit_maps)(void *, const E264PicDesc *, uint8_t *, uint8_t *, uint64_t *);
static uint64_t rng_e;
static uint32_t e32(void) { rng_e ^= rng_e >> 12; rng_e ^= rng_e << 25; rng_e ^= rng_e >> 27; return (uint32_t)((rng_e * 0x2545F4914F6CDD1Dull) >> 32); }
static int erand(int n) { return n > 0 ? (int)(e32() % (unsigned)n) : 0; }
static long cov_int16, cov_unread_taint;
static uint8_t *port_maps, *dev_map, *host_out;

/* one picture through both sides (run_picture of record_fuzz.c, plus the maps); 0 when they agree */
static int run_picture_maps(Ctx *c, int pic, int dst, int pcm_content, int cpu_only) {
	E264PicDesc pd;
	draw_picture(c, &pd, dst, pcm_content);
	if (erand(2)) {   /* a picture with an error map: own errors on some records, a drawn set of tainted slots */
		pd.err_pic = 1;
		pd.taint = e32() & ((1u << c->n_slots) - 1);
		int dens = erand(3) == 0 ? 0 : erand(40);
		for (int a = 0; a < c->nmb; a++) c->recs[a].err = (uint8_t)(erand(100) < dens ? (erand(2) ? 100 : erand(101)) : 0);
		uint32_t read = 0;
		for (int a = 0; a < c->nmb; a++) {
			const E264MbRec *r = c->recs + a;
			if (r->kind != MBK_INTER) continue;
			for (int l = 0; l < 2; l++) for (int b = 0; b < 16; b++) if (r->ref_idx[l][b >> 2] >= 0) {
				int s = r->ref_pic[l][b >> 2];
				read |= 1u << s;
				cov_int16 += (pd.taint >> s & 1) && (r->mv[l][b][0] <= -32767 || r->mv[l][b][0] >= 32764 || r->mv[l][b][1] <= -32767 || r->mv[l][b][1] >= 32764);
			}
		}
		cov_unread_taint += (pd.taint & ~read & ~(1u << dst)) != 0;
	}
	char why[256];
	if (e264_check_records(&pd, c->recs, c->coefs, c->slices, c->intra_list, c->n_slots, why, sizeof(why))) { fprintf(stderr, "generator broke the record contract, picture %d: %s\n", pic, why); exit(2); }
	count_picture(c);
	cov[C_PICTURES]++;
	port_recon_picture(c->port_frames, &pd, c->recs, c->coefs, c->slices);
	port_error_map(port_maps, &pd, c->recs);
	if (cpu_only) return 0;
	E264Staging st;
	if (D.acquire(c->dev, dst, &st)) { fprintf(stderr, "acquire_staging failed\n"); exit(3); }
	memcpy(st.recs, c->recs, (size_t)c->nmb * sizeof(E264MbRec));
	memcpy(st.coefs, c->coefs, (size_t)pd.n_coefs * 2);
	memcpy(st.slices, c->slices, (size_t)pd.n_slices * sizeof(E264SliceRec));
	memcpy(st.intra_list, c->intra_list, (size_t)pd.n_intra * 4);
	pd.staging = st.handle;
	uint64_t t;
	if (submit_maps(c->dev, &pd, host_out, NULL, &t) || D.wait(c->dev, t)) { fprintf(stderr, "picture %d: submit/wait failed\n", pic); return 1; }
	if (D.error_flag(c->dev)) { fprintf(stderr, "picture %d: device error flag %d\n", pic, D.error_flag(c->dev)); return 1; }
	const uint8_t *port = c->port_frames + (size_t)dst * c->g.frame_bytes;
	const int W = c->g.width_mbs, H = c->g.height_mbs;
	for (int pl = 0; pl < 3; pl++) {
		int w = pl ? W * 8 : W * 16, h = pl ? H * 8 : H * 16, stride = pl ? c->g.stride_c : c->g.stride_y;
		size_t base = pl == 0 ? 0 : (size_t)c->g.plane_y + (pl == 2 ? c->g.stride_c / 2 : 0);
		for (int y = 0; y < h; y++) for (int x = 0; x < w; x++) {
			size_t o = base + (size_t)y * stride + x;
			if (host_out[o] == port[o]) continue;
			fprintf(stderr, "MISMATCH picture %d (slot %d) plane %d x %d y %d: device %d port %d\n", pic, dst, pl, x, y, host_out[o], port[o]);
			dump_mb(c->recs, c->slices, W, (y / (pl ? 8 : 16)) * W + x / (pl ? 8 : 16));
			return 1;
		}
	}
	if (pd.err_pic) {
		if (slot_map(c->dev, dst, dev_map)) { fprintf(stderr, "picture %d: e264b_slot_map failed\n", pic); return 1; }
		const uint8_t *pm = port_maps + (size_t)dst * c->nmb;
		for (int a = 0; a < c->nmb; a++) if (dev_map[a] != pm[a]) {
			fprintf(stderr, "MAP MISMATCH picture %d (slot %d, taint %#x) mb %d: device %d port %d\n", pic, dst, pd.taint, a, dev_map[a], pm[a]);
			dump_mb(c->recs, c->slices, W, a);
			return 1;
		}
	}
	return 0;
}

int main(int argc, char **argv) {
	int cpu_only = 0, s0 = 1, s1 = 1;
	const char *lib = NULL;
	for (int i = 1; i < argc; i++) {
		if (!strcmp(argv[i], "--cpu-only")) cpu_only = 1;
		else if (!strcmp(argv[i], "--lib") && i + 1 < argc) lib = argv[++i];
		else if (!strcmp(argv[i], "--seeds") && i + 1 < argc) { if (sscanf(argv[++i], "%d-%d", &s0, &s1) == 1) s1 = s0; }
		else { fprintf(stderr, "usage: %s [--cpu-only] [--lib path] [--seeds A-B]\n", argv[0]); return 2; }
	}
	if (!cpu_only) {
		if (!lib) { fprintf(stderr, "--lib is needed without --cpu-only\n"); return 2; }
		load_device(lib);
		void *h = dlopen(lib, RTLD_NOW);
		if (!h || !(*(void **)&slot_map = dlsym(h, "e264b_slot_map")) || !(*(void **)&submit_maps = dlsym(h, "e264b_submit_maps"))) { fprintf(stderr, "missing e264b_slot_map / e264b_submit_maps\n"); return 3; }
	}
	/* the geometries, slot counts, fills and picture sequence of record_fuzz.c with one picture in flight */
	const int n_geoms = sizeof(geoms) / sizeof(geoms[0]);
	int fails = 0, total = 0;
	for (int seed = s0; seed <= s1; seed++) {
		rng = 0x9E3779B97F4A7C15ull * (uint64_t)(seed + 1) ^ 0xD1B54A32D192ED03ull;
		rng_e = 0xBF58476D1CE4E5B9ull * (uint64_t)(seed + 1) ^ 0x94D049BB133111EBull;
		int W = geoms[seed % n_geoms][0], H = geoms[seed % n_geoms][1];
		Ctx c; memset(&c, 0, sizeof(c));
		geometry(&c, W, H, 2 + rnd(MAX_SLOTS - 1));
		port_maps = calloc((size_t)c.nmb * c.n_slots, 1); dev_map = calloc(c.nmb, 1);
		int n_pics = W * H >= 4096 ? 3 : W * H >= 100 ? 12 : 24;
		if (!cpu_only) {
			if (D.create(&c.dev)) { fprintf(stderr, "e264b_create failed\n"); return 3; }
			if (D.configure(c.dev, &c.g, c.n_slots)) { fprintf(stderr, "e264b_configure failed\n"); return 3; }
			host_out = D.host_alloc(c.dev, c.g.frame_bytes);
		}
		for (int s = 0; s < c.n_slots; s++) {   /* every slot starts identical on both sides; fill_slot makes its map all 100 */
			int y = rnd(256), cc = rnd(256);
			uint8_t *f = c.port_frames + (size_t)s * c.g.frame_bytes;
			memset(f, y, c.g.plane_y); memset(f + c.g.plane_y, cc, c.g.frame_bytes - c.g.plane_y);
			memset(port_maps + (size_t)s * c.nmb, 100, c.nmb);
			if (!cpu_only) D.fill(c.dev, s, y, cc);
		}
		int bad = 0;
		for (int s = 0; s < c.n_slots && !bad; s++) bad = run_picture_maps(&c, total++, s, s % 3, cpu_only);
		for (int p = 0; p < n_pics && !bad; p++) bad = run_picture_maps(&c, total++, rnd(c.n_slots), -1, cpu_only);
		if (bad) { fprintf(stderr, "seed %d (%dx%d, %d slots) failed\n", seed, W, H, c.n_slots); fails++; }
		if (!cpu_only) { D.host_free(c.dev, host_out); D.destroy(c.dev); }
		free(port_maps); free(dev_map);
		free(c.port_alloc); free(c.recs); free(c.coefs); free(c.slices); free(c.intra_list);
	}
	static const char *mn[12] = {"map_clamp_left", "map_clamp_right", "map_clamp_top", "map_clamp_bottom", "map_window_1mb", "map_window_2mb", NULL,
		"map_window_4mb", "map_max_from_list1", "map_read_all100_slot", "map_intra_c_4x4_blk5", "map_intra_c_8x8_blk1"};
	for (int i = 0; i < 12; i++) if (mn[i]) printf("cov %s %ld\n", mn[i], port_cov_map[i]);
	printf("cov map_int16_vector %ld\ncov map_tainted_slot_unread %ld\ncov pictures %ld\n", cov_int16, cov_unread_taint, cov[C_PICTURES]);
	printf("%d pictures, %d failing seeds\n", total, fails);
	return fails ? 1 : 0;
}
