// Host check of edge264_b200/csrc/mc_math.cuh (the per-thread 4x4 interpolation of the inter kernel) against the oracle's
// per-sample restatement oracle/port_recon.c (itself pinned to the reference's decode_inter_luma by ref_kat fuzz):
// every fractional position, random and extreme (0/255 period-3, the int16 wrap of the centre sample) windows.
// Build + run: tests/test_mc_math.py.  Test infrastructure.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "../../edge264_b200/csrc/mc_math.cuh"
extern "C" {
typedef struct { const uint8_t *p; int stride, w, h; } Plane;
int port_mc_luma_sample(const Plane *r, int x, int y, int fx, int fy);
int port_mc_chroma_sample(const Plane *r, int x, int y, int fx, int fy);
}
static uint32_t rng = 12345;
static uint32_t rnd() { rng = rng * 1664525u + 1013904223u; return rng >> 8; }
int main() {
	enum { S = 32 };
	uint8_t img[S * S];
	long bad = 0, n = 0;
	for (int it = 0; it < 40000; it++) {
		int mode = it % 5;
		for (int i = 0; i < S * S; i++) {
			int x = i % S, y = i / S;
			if (mode == 0) img[i] = (uint8_t)rnd();
			else if (mode == 1) img[i] = (uint8_t)((((x + it) % 3 == 1) == ((y + it / 3) % 3 == 1)) ? 255 : 0);       // period-3 checkerboards
			else if (mode == 2) img[i] = (uint8_t)(((x + (it & 1)) % 3 == 1) ? 255 : 0) ^ (uint8_t)(rnd() % 37 == 0 ? 3 : 0);
			else if (mode == 3) img[i] = (uint8_t)(rnd() & 1 ? 255 : 0);
			else img[i] = (uint8_t)(128 + (int)(rnd() % 9) - 4);
		}
		Plane P = {img, S, S, S};
		int X = 8 + (int)(rnd() % 12), Y = 8 + (int)(rnd() % 12);     // block origin, window stays inside the image
		// window rows y = Y-2..Y+6, 12 bytes from x = X-2, read through an aligned word + byte offset like the kernel
		uint32_t w[9][3];
		for (int r = 0; r < 9; r++) {
			const uint8_t *row = img + (Y - 2 + r) * S;
			uint32_t a[4]; int x0 = X - 2, al = x0 & ~3, sh = (x0 & 3) * 8;
			for (int k = 0; k < 4; k++) memcpy(&a[k], row + al + 4 * k, 4);
			for (int k = 0; k < 3; k++) w[r][k] = sh ? mc_fsr(a[k], a[k + 1], sh) : a[k];
		}
		for (int fy = 0; fy < 4; fy++) for (int fx = 0; fx < 4; fx++) {
			uint32_t out[4];
			mc_luma4x4(w, fx, fy, out);
			for (int y = 0; y < 4; y++) for (int x = 0; x < 4; x++) {
				int want = port_mc_luma_sample(&P, X + x, Y + y, fx, fy), got = (out[y] >> (8 * x)) & 255;
				n++;
				if (want != got && bad++ < 10) printf("luma mismatch it %d mode %d frac (%d,%d) at (%d,%d): want %d got %d\n", it, mode, fx, fy, x, y, want, got);
			}
		}
		for (int fy = 0; fy < 8; fy++) for (int fx = 0; fx < 8; fx++) {
			uint32_t c[3];
			for (int r = 0; r < 3; r++) { c[r] = 0; for (int k = 0; k < 3; k++) c[r] |= (uint32_t)img[(Y + r) * S + X + k] << (8 * k); c[r] |= (rnd() & 255u) << 24; }
			uint32_t o = mc_chroma2x2(c[0], c[1], c[2], fx, fy);
			for (int y = 0; y < 2; y++) for (int x = 0; x < 2; x++) {
				int want = port_mc_chroma_sample(&P, X + x, Y + y, fx, fy), got = (o >> (8 * (y * 2 + x))) & 255;
				n++;
				if (want != got && bad++ < 10) printf("chroma mismatch frac (%d,%d) at (%d,%d): want %d got %d\n", fx, fy, x, y, want, got);
			}
		}
	}
	// prediction + residual (every reconstruction kernel): per sample the oracle's clip255((int16_t)(p + r)) (port_recon.c),
	// residuals over the whole int16 range, near zero and at the wrap
	for (int it = 0; it < 1000000; it++) {
		const uint32_t p = rnd() ^ rnd() << 8;
		int16_t r[4];
		for (int k = 0; k < 4; k++) { const int m = rnd() % 3; r[k] = (int16_t)(m == 0 ? rnd() : m == 1 ? (int)(rnd() % 600) - 300 : 32767 - (int)(rnd() % 300)); }
		const uint32_t got = mc_add_res4(p, (uint16_t)r[0] | (uint32_t)(uint16_t)r[1] << 16, (uint16_t)r[2] | (uint32_t)(uint16_t)r[3] << 16);
		for (int k = 0; k < 4; k++) {
			const int s = (int16_t)(((p >> (8 * k)) & 255) + r[k]), want = s < 0 ? 0 : s > 255 ? 255 : s;
			n++;
			if ((int)((got >> (8 * k)) & 255) != want && bad++ < 10) printf("add_res4 mismatch p %08x r %d: want %d got %d\n", p, r[k], want, (int)((got >> (8 * k)) & 255));
		}
	}
	printf("%ld samples checked, %ld mismatches\n", n, bad);
	return bad != 0;
}
