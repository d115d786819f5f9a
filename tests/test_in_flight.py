"""Reconstruction with many pictures in flight, the way the product runs: several device contexts submitting from several
host threads, each with several pictures queued ahead of the one it waits for, contexts returning to the process-wide
pool and coming back with another geometry or the same one, and the benchmark's replay of 16 decoders at once.

Every other test reconstructs one picture of one decoder at a time.  Here, kernels of different contexts share the SMs
while their in-kernel waits (flags, row progress, ticket-ordered bands) must still make progress; a picture reads a
frame slot that an earlier picture still in flight writes, or overwrites a slot that one still reads; the host refills
a staging area as soon as the picture that used it has been uploaded.  The outputs are compared with the CPU
restatement (oracle/port_recon.c) and with the golden digests of the reference decoder's frames."""
import ctypes, errno, json, os, random, re, subprocess, threading
from concurrent.futures import ThreadPoolExecutor
import numpy as np
import pytest
from conftest import ROOT, STREAMS, DPB_STREAMS, make_stream, md5_frames
from checkers import decode_bytes, load
from test_record_fuzz import FUZZ_SRC, _counters

GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "streams.json")))
ALL_STREAMS = STREAMS + DPB_STREAMS
INFLIGHT_COUNTERS = ("inflight_max", "ref_slot_in_flight", "dst_slot_read_in_flight", "staging_wrapped", "contexts")
# 8 contexts on 8 host threads, 6 pictures in flight each; seeds 0-15 take geometries 0-15 of the fuzzer's list
# (120x68 and 256x2 among them)
FUZZ_ARGS = ["--contexts", "8", "--inflight", "6", "--seeds", "0-15"]


@pytest.fixture(scope="module")
def fuzzer(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("fuzz") / "record_fuzz")
    subprocess.run(["gcc", "-O2", "-std=gnu11", "-w", "-pthread"] + FUZZ_SRC + ["-o", exe, "-ldl"], check=True)
    return exe


def test_threaded_fuzzer_reaches_the_overlaps(fuzzer):
    """CPU only: the concurrent draw still reaches every arithmetic edge, and the submission sequence it would hand the
    device has pictures that read or overwrite the slots of pictures still in flight, and pictures that find every
    staging area of their context in use."""
    r = subprocess.run([fuzzer, "--cpu-only"] + FUZZ_ARGS, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    cov = _counters(r.stdout)
    assert len(cov) >= 75 and set(INFLIGHT_COUNTERS) <= set(cov), r.stdout
    zero = [k for k, v in cov.items() if v == 0]
    assert not zero, "never reached: %s" % zero
    assert cov["inflight_max"] == 6 and cov["contexts"] == 8
    per_context = [int(m.group(2)) for m in re.finditer(r"^context (\d+): (\d+) pictures, 0 failing seeds$", r.stdout, re.M)]
    total = int(re.search(r"^(\d+) pictures, 0 failing seeds$", r.stdout, re.M).group(1))
    assert len(per_context) == 8 and sum(per_context) == total == cov["pictures"]


def _frames_ids(frames):
    return [f[0] for f in frames]


def test_concurrent_port_decoders_match_golden(workdir):
    """The host parser from many threads at once (its lazily built tables, the decoder's own locks): every stream through
    the CPU restatement, 8 decoders at a time, half of them parsing ahead on 2 worker threads.  ctypes releases the GIL
    during each call, so the decoders really run side by side."""
    load("port")   # bound once, before the threads
    data = {name: open(make_stream(workdir, name, w, h, args), "rb").read() for name, w, h, args in ALL_STREAMS}
    solo = {name: _frames_ids(decode_bytes(data[name], "port")[0]) for name, *_ in ALL_STREAMS}
    jobs = [(name, 2 if i % 2 else 0) for i, (name, *_) in enumerate(ALL_STREAMS)]
    with ThreadPoolExecutor(8) as ex:
        out = list(ex.map(lambda j: decode_bytes(data[j[0]], "port", j[1])[0], jobs))
    for (name, threads), frames in zip(jobs, out):
        assert md5_frames(frames) == GOLD[name]["md5"], "%s (%d workers)" % (name, threads)
        assert _frames_ids(frames) == solo[name], "%s (%d workers)" % (name, threads)


@pytest.mark.gpu
def test_device_matches_port_with_pictures_in_flight(fuzzer):
    """8 device contexts from 8 host threads, 6 pictures queued ahead in each, against the port byte for byte; every
    context's device error word stays 0."""
    lib = os.path.join(ROOT, "edge264_b200", "libedge264_b200.so")
    r = subprocess.run([fuzzer, "--lib", lib] + FUZZ_ARGS, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-800:], r.stderr[-3000:])
    cov = _counters(r.stdout)
    assert cov["pictures"] >= 500 and cov["inflight_max"] == 6 and cov["ref_slot_in_flight"] > 0 and cov["staging_wrapped"] > 0


def _core():
    core = ctypes.CDLL(os.path.join(ROOT, "edge264_b200", "libedge264_b200.so"))
    core.e264b_of_decoder.restype = ctypes.c_void_p; core.e264b_of_decoder.argtypes = [ctypes.c_void_p]
    core.e264b_slot_hash.restype = ctypes.c_uint64; core.e264b_slot_hash.argtypes = [ctypes.c_void_p, ctypes.c_int]
    core.e264b_slot_count.argtypes = [ctypes.c_void_p]
    core.e264b_error_flag.argtypes = [ctypes.c_void_p]
    core.e264b_kept_count.argtypes = [ctypes.c_void_p]
    core.e264b_stats.argtypes = [ctypes.c_void_p] + [ctypes.POINTER(ctypes.c_uint64)] * 3
    core.e264b_picture_bytes.restype = ctypes.c_longlong; core.e264b_picture_bytes.argtypes = [ctypes.c_void_p]
    core.e264b_replay_frames.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    return core


# decoders that also ask for the optional outputs: (packed format, log2 scale)
EXTRAS = {"b_explicit": (1, 0), "ragged_2xN": (0, 1), "pb_intra_heavy": (1, 2), "mixed_slices_cabac": (0, 0), "dpb_ipb_spatial": (1, 1)}


def _decode_concurrently(lib, core, order, data):
    """Decode the streams of `order` ((name, n_threads) pairs) all at once, one Python thread each.  The decoders are
    allocated and freed on this thread in list order, so each takes the oldest context of the pool and gives it back in
    the same order.  Returns the frames of each and the device context it ran on."""
    import edge264_b200 as pkg
    decs = []
    for name, threads in order:
        dec = lib.edge264_alloc(threads, None, None, 0, None, None, None)
        assert dec, "edge264_alloc failed"
        if name in EXTRAS:
            assert lib.edge264_enable_motion(dec) == 0 and lib.edge264_enable_packed(dec, *EXTRAS[name]) == 0
        decs.append(dec)
    results = [None] * len(order)
    start = threading.Barrier(len(order))

    def run(k):
        name, dec = order[k][0], decs[k]
        extra = name in EXTRAS
        buf = ctypes.create_string_buffer(data[name], len(data[name]) + 64)
        base = ctypes.addressof(buf); end = base + len(data[name])
        nal = base + 3 + (1 if data[name][2] == 0 else 0)
        frames, f, drained = [], pkg.Edge264Frame(), False
        start.wait()
        while True:
            sc = lib.edge264_find_start_code(nal, end, 0) if nal < end else end
            before = len(frames)
            res = lib.edge264_decode_NAL(dec, nal, sc, None, None)
            drained |= nal >= end
            while lib.edge264_get_frame(dec, ctypes.byref(f), 0) == 0:
                frames.append((f.FrameId, f.width_Y, f.height_Y, pkg._frame_bytes(f)) + (
                    (pkg._frame_errors(f), pkg.frame_motion(lib, dec, f), pkg.frame_packed(lib, dec, f)) if extra else ()))
            if res == errno.ENOBUFS:
                if len(frames) == before:
                    break
                continue
            if res in (errno.ENOTSUP, errno.EBADMSG):
                res = 0
            nal = sc + 3 if sc + 3 < end else end
            if res != 0 or drained:
                break
        results[k] = frames

    threads = [threading.Thread(target=run, args=(k,)) for k in range(len(order))]
    for t in threads: t.start()
    for t in threads: t.join()
    ctxs = [core.e264b_of_decoder(d) for d in decs]
    for d in decs:
        p = ctypes.c_void_p(d)
        lib.edge264_free(ctypes.byref(p))
    return results, ctxs


def _same_extras(a, b):
    """mb_errors, motion export and packed output of two decodes of one stream."""
    assert len(a) == len(b)
    for fa, fb in zip(a, b):
        assert fa[4] == fb[4], "mb_errors"
        assert fa[5].keys() == fb[5].keys() and all(np.array_equal(fa[5][k], fb[5][k]) for k in fa[5]), "motion export"
        assert fa[6].keys() == fb[6].keys() and all(np.array_equal(fa[6][k], fb[6][k]) for k in fa[6]), "packed output"


@pytest.mark.gpu
def test_concurrent_decoders_match_golden(workdir):
    """Every test stream on the GPU at once, one decoder and one Python thread each, with 0, 2 or 4 parse-ahead workers;
    a few also export mb_errors, motion and packed output.  Then the same streams again in another order, so that the
    pooled device contexts come back with other geometries (reallocated) or with the same one (kept as they are)."""
    import edge264_b200 as pkg
    lib, core = pkg.load(), _core()
    data = {name: open(make_stream(workdir, name, w, h, args), "rb").read() for name, w, h, args in ALL_STREAMS}
    size = {name: (w, h) for name, w, h, _ in ALL_STREAMS}
    threads = {name: (0, 2, 4)[i % 3] for i, (name, *_) in enumerate(ALL_STREAMS)}
    alone = {name: pkg.decode_bytes(data[name], None, threads[name], errors=True, motion=True, packed=EXTRAS[name]) for name in EXTRAS}
    order1 = [(name, threads[name]) for name, *_ in ALL_STREAMS]
    order2 = list(order1)
    random.Random(5).shuffle(order2)   # leaves b_pcm_checker where it was: its context comes back with the same geometry
    rounds = []
    for order in (order1, order2):
        frames, ctxs = _decode_concurrently(lib, core, order, data)
        for (name, nt), fr in zip(order, frames):
            assert md5_frames(fr) == GOLD[name]["md5"], "%s (%d workers)" % (name, nt)
            if name in EXTRAS:
                assert [f[:4] for f in fr] == [f[:4] for f in alone[name][0]], name
                _same_extras(fr, alone[name][0])
        rounds.append(dict(zip(ctxs, (name for name, _ in order))))
    first, second = rounds
    assert len(first) == len(second) == len(ALL_STREAMS), "two decoders alive at once shared a device context"
    assert set(second) <= set(first), "round 2 created device contexts although the pool held enough"
    # the same stream with the same workers configures the same geometry and slot count: e264b_configure keeps everything
    assert any(first[c] == second[c] for c in second), "no context came back with its geometry (seed of the shuffle)"
    assert any(size[first[c]] != size[second[c]] for c in second), "no context came back with another geometry"


def _frame_sum(frame):
    """frame_sum of tools/e264_bench.c over the cropped planes of one frame (FrameId, width, height, I420 bytes): per row,
    the 64-bit sum of its little-endian 8-byte words and of the bytes left over; the rows folded as s = s * 1000003 + row."""
    _, w, h, raw = frame
    wc, hc = (w + 1) // 2, (h + 1) // 2
    assert len(raw) == w * h + 2 * wc * hc
    buf = np.frombuffer(raw, np.uint8)
    planes = [buf[:w * h].reshape(h, w), buf[w * h:w * h + wc * hc].reshape(hc, wc), buf[w * h + wc * hc:].reshape(hc, wc)]
    s, M = 0, (1 << 64) - 1
    for p in planes:
        n8 = p.shape[1] // 8 * 8
        rows = np.ascontiguousarray(p[:, :n8]).view("<u8").sum(axis=1, dtype=np.uint64) + p[:, n8:].sum(axis=1, dtype=np.uint64)
        for a in rows.tolist():
            s = (s * 1000003 + a) & M
    return s


def _stream_sum(frames):
    s = 0
    for f in frames:
        s = (s * 31 + _frame_sum(f)) & ((1 << 64) - 1)
    return s


@pytest.mark.gpu
def test_replay_at_the_benchmark_shape(workdir):
    """16 streams of the benchmark's 1080p workload (8 frames each) decoded through tools/libe264bench.so as bench.py does
    (8 application threads, 2 parse-ahead workers per decoder, records kept): each stream's e2e checksum equals the one
    of the port's frames.  Then the kept records are replayed with all 16 decoders in flight as CUDA graphs, with 3 in
    flight (event-chained), and as plain launches from 4 host threads: each replay leaves every frame slot as the live
    decode did, raises no error word and runs exactly the kept pictures' kernels."""
    from bench import CONFIGS, ReplayStats
    cfg = CONFIGS["1080p"]
    N, F = 16, 8
    paths = [make_stream(workdir, "bench_%d" % (cfg["seed0"] + i), cfg["w"], cfg["h"], "-n %d -s %d %s" % (F, cfg["seed0"] + i, cfg["gen"])) for i in range(N)]
    data = [open(p, "rb").read() for p in paths]
    with ThreadPoolExecutor(8) as ex:
        port_sums = list(ex.map(lambda d: _stream_sum(decode_bytes(d, "port")[0]), data))
    core = _core()
    core.e264b_replay.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ReplayStats)]
    bench = ctypes.CDLL(os.path.join(ROOT, "tools", "libe264bench.so"))
    bench.e264bench_run.restype = ctypes.c_double
    bench.e264bench_run.argtypes = [ctypes.POINTER(ctypes.c_char_p), ctypes.POINTER(ctypes.c_size_t), ctypes.c_int, ctypes.c_int,
                                    ctypes.c_int, ctypes.POINTER(ctypes.c_long), ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_void_p)]
    bench.e264bench_free.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int]
    saved = {k: os.environ.get(k) for k in ("E264B_KEEP", "E264_BENCH_DEC_THREADS", "E264B_REPLAY_INFLIGHT", "E264B_REPLAY_GRAPH")}
    decs = (ctypes.c_void_p * N)()
    try:
        os.environ["E264B_KEEP"] = "1"; os.environ["E264_BENCH_DEC_THREADS"] = "2"
        os.environ.pop("E264B_REPLAY_INFLIGHT", None); os.environ.pop("E264B_REPLAY_GRAPH", None)
        bufs = (ctypes.c_char_p * N)(*data); sizes = (ctypes.c_size_t * N)(*map(len, data))
        frames = (ctypes.c_long * N)(); sums = (ctypes.c_uint64 * N)()
        bench.e264bench_run(bufs, sizes, N, 8, 1, frames, sums, decs)
        assert list(frames) == [F] * N
        assert list(sums) == port_sums, "the e2e checksums differ from the port's frames"
        devs = [core.e264b_of_decoder(d) for d in decs]
        assert len(set(devs)) == N and all(core.e264b_kept_count(d) == F for d in devs)
        live_launches = 0
        for d in devs:
            n = ctypes.c_uint64()
            core.e264b_stats(d, ctypes.byref(n), None, None)
            live_launches += n.value
        hashes = [[core.e264b_slot_hash(d, s) for s in range(core.e264b_slot_count(d))] for d in devs]
        arr = (ctypes.c_void_p * N)(*devs)
        for env, reps, launch_threads, inflight in (({}, 2, 1, N), ({"E264B_REPLAY_INFLIGHT": "3"}, 2, 1, 3),
                                                    ({"E264B_REPLAY_GRAPH": "0"}, 2, 4, None)):
            os.environ.pop("E264B_REPLAY_INFLIGHT", None); os.environ.pop("E264B_REPLAY_GRAPH", None)
            os.environ.update(env)
            st = ReplayStats()
            assert core.e264b_replay(arr, N, reps, launch_threads, ctypes.byref(st)) == 0, env
            assert [core.e264b_error_flag(d) for d in devs] == [0] * N, env
            assert [[core.e264b_slot_hash(d, s) for s in range(core.e264b_slot_count(d))] for d in devs] == hashes, env
            assert st.launches == live_launches * reps, env
            if inflight is None:
                assert st.threads == launch_threads
            else:
                assert st.threads == 0 and st.inflight == inflight, env
        for d in devs:
            out = ctypes.create_string_buffer(F * core.e264b_picture_bytes(d))
            assert core.e264b_replay_frames(d, out) == 0
    finally:
        for k, v in saved.items():
            if v is None: os.environ.pop(k, None)
            else: os.environ[k] = v
        os.environ["E264B_KEEP"] = "0"
        if any(decs):
            bench.e264bench_free(decs, N)
