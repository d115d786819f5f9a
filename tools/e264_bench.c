/* e264_bench — multi-stream decode driver over the edge264 C API (bench/test infrastructure).
 * Compiled twice from this one source: against libedge264_b200.so (tools/libe264bench.so) and against
 * the compiled reference (oracle/_ref/libe264bench_ref.so), so both arms of bench.py run the SAME
 * application loop (reference README.md:117-156) with one decoder instance per stream and one POSIX
 * thread per decoder.  Every output frame is read back on the host (64-bit word sum of the cropped
 * planes) so that the GPU arm's device->host copies are inside the timed region. */
#define _GNU_SOURCE
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include "edge264.h"

/* include/edge264_luma.h, include/edge264_loopfilter.h and include/edge264_latency.h; weak: the reference's library has no
 * such entry points */
int edge264_enable_luma_only(Edge264Decoder *dec) __attribute__((weak));
int edge264_set_loop_filter(Edge264Decoder *dec, int mode) __attribute__((weak));
int edge264_set_output_latency(Edge264Decoder *dec, int max_reorder) __attribute__((weak));

typedef struct Job {
	const uint8_t *buf; size_t size;
	long frames; uint64_t sum; int last_ret;
	Edge264Decoder *dec; int keep;
} Job;
typedef struct Pool { Job *jobs; int n, next; pthread_mutex_t mu; pthread_barrier_t *bar; } Pool;

static uint64_t frame_sum(const Edge264Frame *f) {
	uint64_t s = 0;
	for (int pl = 0; pl < 3; pl++) {
		int w = pl ? f->width_C : f->width_Y, h = pl ? f->height_C : f->height_Y, st = pl ? f->stride_C : f->stride_Y;
		for (int y = 0; y < h; y++) {
			const uint8_t *r = f->samples[pl] + (size_t)y * st;
			int x = 0; uint64_t a = 0;
			for (; x + 8 <= w; x += 8) { uint64_t v; memcpy(&v, r + x, 8); a += v; }
			for (; x < w; x++) a += r[x];
			s = s * 1000003u + a;
		}
	}
	return s;
}

static void decode_stream(Job *j) {
	const uint8_t *buf = j->buf, *end = buf + j->size;
	const uint8_t *nal = buf + 3 + (buf[2] == 0);
	/* E264_BENCH_DEC_THREADS: n_threads of every decoder (0 = parse inside decode_NAL; the GPU library parses pictures ahead on
	 * worker threads otherwise; the reference's threaded mode hangs here, SURVEY section 0.7, so its arm stays at 0) */
	const char *nt = getenv("E264_BENCH_DEC_THREADS");
	Edge264Decoder *dec = edge264_alloc(nt ? atoi(nt) : 0, NULL, NULL, 0, NULL, NULL, NULL);
	Edge264Frame f; int res, drained = 0; long frames = 0; uint64_t sum = 0;
	if (!dec) { j->last_ret = -1; return; }
	/* E264_BENCH_LUMA_ONLY=1: every decoder decodes the Y plane only (tools/luma_only_cost.py) */
	const char *lo = getenv("E264_BENCH_LUMA_ONLY");
	if (lo && atoi(lo) && (!edge264_enable_luma_only || edge264_enable_luma_only(dec))) { edge264_free(&dec); j->last_ret = -1; return; }
	/* E264_BENCH_LOOP_FILTER=<mode>: edge264_set_loop_filter on every decoder (tools/loop_filter_cost.py) */
	const char *lf = getenv("E264_BENCH_LOOP_FILTER");
	if (lf && atoi(lf) && (!edge264_set_loop_filter || edge264_set_loop_filter(dec, atoi(lf)))) { edge264_free(&dec); j->last_ret = -1; return; }
	/* E264_BENCH_OUTPUT_LATENCY=<n>: edge264_set_output_latency on every decoder (tools/latency_cost.py) */
	const char *ol = getenv("E264_BENCH_OUTPUT_LATENCY");
	if (ol && *ol && (!edge264_set_output_latency || edge264_set_output_latency(dec, atoi(ol)))) { edge264_free(&dec); j->last_ret = -1; return; }
	for (;;) {
		const uint8_t *sc = nal < end ? edge264_find_start_code(nal, end, 0) : end;
		long before = frames;
		res = edge264_decode_NAL(dec, nal, sc, NULL, NULL);
		if (nal >= end) drained = 1;
		while (!edge264_get_frame(dec, &f, 0)) { sum = sum * 31 + frame_sum(&f); frames++; }
		if (res == ENOBUFS) { if (frames == before) break; continue; }
		if (res == ENOTSUP || res == EBADMSG) res = 0;
		nal = sc + 3 < end ? sc + 3 : end;
		if (res != 0 || drained) break;
	}
	j->frames = frames; j->sum = sum; j->last_ret = res;
	if (j->keep) j->dec = dec; else edge264_free(&dec);
}

static void *worker(void *arg) {
	Pool *p = (Pool *)arg;
	pthread_barrier_wait(p->bar);
	for (;;) {
		pthread_mutex_lock(&p->mu);
		int i = p->next < p->n ? p->next++ : -1;
		pthread_mutex_unlock(&p->mu);
		if (i < 0) break;
		decode_stream(&p->jobs[i]);
	}
	return NULL;
}

/* Decode n_streams buffers with n_threads threads.  Returns wall seconds of the decode region.
 * frames[i], sums[i] per stream; decoders[i] kept alive when keep != 0 (caller frees with e264bench_free). */
double e264bench_run(const uint8_t **bufs, const size_t *sizes, int n_streams, int n_threads, int keep,
                     long *frames, uint64_t *sums, void **decoders) {
	Job *jobs = (Job *)calloc((size_t)n_streams, sizeof(Job));
	for (int i = 0; i < n_streams; i++) { jobs[i].buf = bufs[i]; jobs[i].size = sizes[i]; jobs[i].keep = keep; }
	if (n_threads > n_streams) n_threads = n_streams;
	if (n_threads < 1) n_threads = 1;
	pthread_barrier_t bar; pthread_barrier_init(&bar, NULL, (unsigned)n_threads + 1);
	Pool p = {jobs, n_streams, 0, PTHREAD_MUTEX_INITIALIZER, &bar};
	pthread_t *th = (pthread_t *)calloc((size_t)n_threads, sizeof(pthread_t));
	for (int i = 0; i < n_threads; i++) pthread_create(&th[i], NULL, worker, &p);
	struct timespec t0, t1;
	pthread_barrier_wait(&bar);
	clock_gettime(CLOCK_MONOTONIC, &t0);
	for (int i = 0; i < n_threads; i++) pthread_join(th[i], NULL);
	clock_gettime(CLOCK_MONOTONIC, &t1);
	for (int i = 0; i < n_streams; i++) { if (frames) frames[i] = jobs[i].frames; if (sums) sums[i] = jobs[i].sum; if (decoders) decoders[i] = jobs[i].dec; }
	free(th); free(jobs); pthread_barrier_destroy(&bar);
	return (t1.tv_sec - t0.tv_sec) + 1e-9 * (t1.tv_nsec - t0.tv_nsec);
}
void e264bench_free(void **decoders, int n) { for (int i = 0; i < n; i++) { Edge264Decoder *d = (Edge264Decoder *)decoders[i]; edge264_free(&d); decoders[i] = NULL; } }
