"""Luma-only decoding (include/edge264_luma.h): the kernels reconstruct and deblock the Y plane only, and the chroma plane
of every output frame is 128.  In 4:2:0 8-bit decoding no luma sample depends on chroma, so the oracle is the decoder's
own full decode (pinned to the reference elsewhere): a luma-only decode must give the same frames, FrameIds, order and
return codes, the same Y plane byte for byte, chroma all 128, and the same error maps and motion export.

CPU tests run the product's host sources over the plain-C restatement (oracle/liboracle_dec.so, and the test backend
with every optional output, tests/native/port_outputs_backend.c); the GPU tests compare the device with the device's
full decode and with the restatement's luma-only decode."""
import ctypes, errno, os, pickle, random, re, subprocess, sys, threading
from concurrent.futures import ThreadPoolExecutor
import numpy as np
import pytest
from conftest import ROOT, STREAMS, DPB_STREAMS, make_stream, have
from test_limits import LIMITS, FULL_LIMITS
from test_gpu_parity import FULL
from api_helpers import _damaged
from checkers import port_outputs_lib
import edge264_b200 as pkg
import checkers

GOLDEN = os.path.join(ROOT, "tests", "golden")
STORED = [os.path.join(GOLDEN, "reference_streams", f) for f in sorted(os.listdir(os.path.join(GOLDEN, "reference_streams")))] + \
         [os.path.join(GOLDEN, "gen_avc_1080p_intra_cavlc.264")]
GENERATED = STREAMS + DPB_STREAMS + LIMITS


def _data(workdir, s):
    return open(make_stream(workdir, *s) if isinstance(s, tuple) else s, "rb").read()


def _id(s):
    return s[0] if isinstance(s, tuple) else os.path.basename(s)


ALL = GENERATED + STORED
IDS = [_id(s) for s in ALL]


def same_as_full(full, luma, label=""):
    """full, luma: decode_bytes results of one stream.  Same frames, FrameIds, order, sizes and return codes; Y equal, the
    chroma of every frame 128; any further fields of the frame tuples (error map, motion export) equal."""
    (ff, fc), (lf, lc) = full, luma
    assert fc == lc, "%s: return codes" % label
    assert [f[:3] for f in ff] == [f[:3] for f in lf], "%s: frames" % label
    for a, b in zip(ff, lf):
        n = a[1] * a[2]
        assert a[3][:n] == b[3][:n], "%s: Y of frame %d" % (label, a[0])
        assert len(b[3]) == len(a[3]) and b[3][n:] == b"\x80" * (len(b[3]) - n), "%s: chroma of frame %d" % (label, a[0])
        for x, y in zip(a[4:], b[4:]):
            if isinstance(x, dict):
                assert x.keys() == y.keys() and all(np.array_equal(x[k], y[k]) for k in x), "%s: motion export of frame %d" % (label, a[0])
            else:
                assert x == y, "%s: error map of frame %d" % (label, a[0])


# ---- CPU: the restatement ----
@pytest.mark.parametrize("stream", ALL, ids=IDS)
def test_port_luma_only_equals_full_decode(workdir, stream):
    data, lib = _data(workdir, stream), checkers.load("port")
    same_as_full(pkg.decode_bytes(data, lib), pkg.decode_bytes(data, lib, luma_only=True), _id(stream))


@pytest.mark.parametrize("stream", STREAMS + DPB_STREAMS, ids=[s[0] for s in STREAMS + DPB_STREAMS])
def test_port_worker_counts_give_identical_output(workdir, stream):
    data, lib = _data(workdir, stream), checkers.load("port")
    runs = [pkg.decode_bytes(data, lib, t, luma_only=True) for t in (0, 1, 3)]
    assert runs[1] == runs[0] and runs[2] == runs[0]


@pytest.mark.parametrize("stream", STREAMS + DPB_STREAMS + LIMITS, ids=[s[0] for s in STREAMS + DPB_STREAMS + LIMITS])
def test_port_error_maps_and_motion_export_equal_full_decode(workdir, stream):
    data, lib = _data(workdir, stream), port_outputs_lib()
    same_as_full(pkg.decode_bytes(data, lib, errors=True, motion=True), pkg.decode_bytes(data, lib, errors=True, motion=True, luma_only=True), stream[0])


@pytest.mark.parametrize("skip", [pkg.SKIP_NONREF, pkg.SKIP_NONKEY], ids=["nonref", "nonkey"])
def test_port_with_skipped_pictures_equals_skip_decode(workdir, skip):
    lib = checkers.load("port")
    for s in STREAMS + DPB_STREAMS:
        data = _data(workdir, s)
        same_as_full(pkg.decode_bytes(data, lib, skip=skip), pkg.decode_bytes(data, lib, skip=skip, luma_only=True), s[0])


def test_port_damaged_streams_equal_full_decode_and_keep_the_record_contract(workdir, monkeypatch):
    """Error maps included; with E264_CHECK_RECORDS=1 every luma-only picture submitted keeps the record contract."""
    lib = port_outputs_lib()
    monkeypatch.setenv("E264_CHECK_RECORDS", "1")
    before, n = lib.e264_test_record_violations(), 0
    for name, seed, data in _damaged(workdir):
        same_as_full(pkg.decode_bytes(data, lib, errors=True), pkg.decode_bytes(data, lib, errors=True, luma_only=True), "%s seed %d" % (name, seed))
        n += 1
    assert n == 75
    assert lib.e264_test_record_violations() == before, lib.e264_test_last_violation()


def _first_slice(data):
    """Offsets (start, end) of the NAL units of an Annex-B stream up to and including its first slice."""
    starts = [m.end() for m in re.finditer(b"\x00\x00\x01", data)]
    out = []
    for k, s in enumerate(starts):
        e = starts[k + 1] - 3 if k + 1 < len(starts) else len(data)
        while e > s and data[e - 1] == 0:
            e -= 1
        out.append((s, e))
        if data[s] & 31 in (1, 5):
            return out
    return out


def test_api_contract(workdir):
    """0 before the first slice (and again), EBUSY once a slice has been decoded, EINVAL for NULL; the reference's
    library has no such entry point."""
    lib = checkers.load("port")
    assert lib.edge264_enable_luma_only(None) == errno.EINVAL
    data = _data(workdir, STREAMS[0])
    buf = ctypes.create_string_buffer(data, len(data) + 64)
    base = ctypes.addressof(buf)
    dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
    assert lib.edge264_enable_luma_only(dec) == 0 and lib.edge264_enable_luma_only(dec) == 0
    for s, e in _first_slice(data):
        assert lib.edge264_enable_luma_only(dec) == 0   # parameter sets are not slices
        lib.edge264_decode_NAL(dec, base + s, base + e, None, None)
    assert lib.edge264_enable_luma_only(dec) == errno.EBUSY
    d = ctypes.c_void_p(dec)
    lib.edge264_free(ctypes.byref(d))
    if have("ref"):
        assert not hasattr(checkers.load("ref"), "edge264_enable_luma_only")


def test_packed_and_resized_outputs_follow_their_definitions(workdir):
    """CPU restatement of the packed and resized outputs: Y plane equal to the full decode's, chroma planes 128."""
    lib = port_outputs_lib()
    for s in (next(x for x in DPB_STREAMS if x[0] == "crop_rect"), next(x for x in STREAMS if x[0] == "b_explicit")):
        data = _data(workdir, s)
        for kw in ({"packed": (pkg.PACKED_NV12, 0)}, {"packed": (pkg.PACKED_NV12, 2)}, {"packed": (pkg.PACKED_I420, 1)},
                   {"resized": (pkg.PACKED_NV12, 224, 224)}, {"resized": (pkg.PACKED_I420, 40, 26)}):
            _same_packed(pkg.decode_bytes(data, lib, **kw)[0], pkg.decode_bytes(data, lib, luma_only=True, **kw)[0], "%s %s" % (s[0], kw))


def _same_packed(full, luma, label):
    assert [f[0] for f in full] == [f[0] for f in luma], label
    for a, b in zip(full, luma):
        pa, pb = a[-1], b[-1]
        assert np.array_equal(pa["y"], pb["y"]), "%s: Y of frame %d" % (label, a[0])
        for k in ("cb", "cr", "cbcr"):
            if k in pb:
                assert pb[k].shape == pa[k].shape and (pb[k] == 128).all(), "%s: %s of frame %d" % (label, k, a[0])


# ---- the record fuzzer with luma-only pictures ----
FUZZ_SRC = [os.path.join(ROOT, "tests", "native", "record_fuzz_luma.c"), os.path.join(ROOT, "oracle", "port_recon.c"), os.path.join(ROOT, "oracle", "record_check.c")]
SEEDS = "0-35"


@pytest.fixture(scope="module")
def fuzzer(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("fuzz") / "record_fuzz_luma")
    subprocess.run(["gcc", "-O2", "-std=gnu11", "-w", "-pthread"] + FUZZ_SRC + ["-o", exe, "-ldl"], check=True)
    return exe


def _counters(out):
    return {m.group(1): int(m.group(2)) for m in re.finditer(r"^cov (\S+) (\d+)$", out, re.M)}


def _check_fuzz_run(r):
    assert r.returncode == 0, (r.stdout[-500:], r.stderr[-3000:])
    cov = _counters(r.stdout)
    zero = [k for k, v in cov.items() if v == 0]
    assert not zero, "edges never drawn: %s" % zero
    assert len(cov) >= 72 and cov["pictures"] >= 500
    assert cov["luma_only_pictures"] >= 200 and cov["colour_pictures"] >= 200
    assert cov["luma_only_pictures"] + cov["colour_pictures"] == cov["pictures"]


def test_fuzzer_draws_both_modes_and_reaches_every_edge(fuzzer):
    _check_fuzz_run(subprocess.run([fuzzer, "--cpu-only", "--seeds", SEEDS], capture_output=True, text=True, timeout=600))


def test_fuzzer_leaves_the_record_draws_alone(fuzzer, tmp_path):
    """record_fuzz's counters, picture for picture the same draws: every counter equal but the two of this driver and
    wp_bi_sat16, which the port counts on predicted samples (chroma predicted from a luma-only reference reads 128)."""
    plain = str(tmp_path / "record_fuzz")
    subprocess.run(["gcc", "-O2", "-std=gnu11", "-w", "-pthread", os.path.join(ROOT, "tests", "native", "record_fuzz.c")] + FUZZ_SRC[1:] + ["-o", plain, "-ldl"], check=True)
    a = _counters(subprocess.run([plain, "--cpu-only", "--seeds", "0-17"], capture_output=True, text=True, timeout=600).stdout)
    b = _counters(subprocess.run([fuzzer, "--cpu-only", "--seeds", "0-17"], capture_output=True, text=True, timeout=600).stdout)
    b = {k: v for k, v in b.items() if k not in ("luma_only_pictures", "colour_pictures")}
    assert a.pop("wp_bi_sat16") > 0 and b.pop("wp_bi_sat16") > 0
    assert a == b


# ---- GPU ----
@pytest.mark.gpu
@pytest.mark.parametrize("stream", ALL, ids=IDS)
def test_device_luma_only_equals_device_full_and_port(workdir, stream):
    data = _data(workdir, stream)
    luma = pkg.decode_bytes(data, luma_only=True)
    same_as_full(pkg.decode_bytes(data), luma, _id(stream))
    assert luma == pkg.decode_bytes(data, checkers.load("port"), luma_only=True), "%s: device and port luma-only frames differ" % _id(stream)


@pytest.mark.gpu
@pytest.mark.parametrize("stream", FULL_LIMITS + FULL, ids=[s[0] for s in FULL_LIMITS + FULL])
def test_device_full_size(workdir, stream):
    data = _data(workdir, stream)
    same_as_full(pkg.decode_bytes(data, n_threads=2), pkg.decode_bytes(data, n_threads=2, luma_only=True), stream[0])


@pytest.mark.gpu
def test_device_error_maps_motion_skip_threads_and_damage(workdir):
    lib = pkg.load()
    for s in STREAMS + DPB_STREAMS:
        data = _data(workdir, s)
        for t in (0, 3):
            same_as_full(pkg.decode_bytes(data, lib, t, errors=True, motion=True), pkg.decode_bytes(data, lib, t, errors=True, motion=True, luma_only=True), s[0])
        for skip in (pkg.SKIP_NONREF, pkg.SKIP_NONKEY):
            same_as_full(pkg.decode_bytes(data, lib, skip=skip), pkg.decode_bytes(data, lib, skip=skip, luma_only=True), s[0])
    port = port_outputs_lib()
    for name, seed, data in _damaged(workdir):
        luma = pkg.decode_bytes(data, lib, errors=True, luma_only=True)
        same_as_full(pkg.decode_bytes(data, lib, errors=True), luma, "%s seed %d" % (name, seed))
        assert luma == pkg.decode_bytes(data, port, errors=True, luma_only=True), "%s seed %d: device and port differ" % (name, seed)


@pytest.mark.gpu
def test_device_matches_port_on_fuzzed_records(fuzzer):
    """Every picture drawn luma-only or colour; one picture in flight, then four contexts with three pictures in flight."""
    lib = os.path.join(ROOT, "edge264_b200", "libedge264_b200.so")
    _check_fuzz_run(subprocess.run([fuzzer, "--lib", lib, "--seeds", SEEDS], capture_output=True, text=True, timeout=900))
    r = subprocess.run([fuzzer, "--lib", lib, "--seeds", SEEDS, "--contexts", "4", "--inflight", "3"], capture_output=True, text=True, timeout=900)
    _check_fuzz_run(r)
    assert _counters(r.stdout)["ref_slot_in_flight"] > 0


@pytest.mark.gpu
def test_many_decoders_in_flight(workdir):
    """8 host threads decode luma-only and colour at once, twice, in shuffled orders; then a few streams alternate colour
    and luma-only decoders.  The pooled device contexts pass from one mode to the other and back (a context keeps its
    geometry's buffers between decoders).  Each output equals its decoder's output alone."""
    lib = pkg.load()
    streams = STREAMS + DPB_STREAMS
    data = {s[0]: _data(workdir, s) for s in streams}
    alone = {(n, lo): pkg.decode_bytes(data[n], lib, 2 if lo else 0, luma_only=lo) for n in data for lo in (False, True)}
    jobs = [(n, lo) for n in data for lo in (False, True)]
    for r in range(2):
        random.Random(r).shuffle(jobs)
        with ThreadPoolExecutor(8) as ex:
            got = list(ex.map(lambda j: pkg.decode_bytes(data[j[0]], lib, 2 if j[1] else 0, luma_only=j[1]), jobs))
        for j, g in zip(jobs, got):
            assert g == alone[j], j
    for n in ("b_explicit", "pb_intra_heavy", "mixed_slices_cabac"):
        for lo in (False, True, False, True):
            assert pkg.decode_bytes(data[n], lib, luma_only=lo) == alone[(n, lo)], (n, lo)


# the samples are device memory: only the packed pictures are read (through torch)
_SUB = """
import sys, ctypes, errno, pickle
sys.path.insert(0, sys.argv[3])
import edge264_b200 as pkg
lib = pkg.load()
data = open(sys.argv[1], 'rb').read()
buf = ctypes.create_string_buffer(data, len(data) + 64); base = ctypes.addressof(buf); end = base + len(data)
dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
a = [int(x) for x in sys.argv[5:]]
assert (lib.edge264_enable_resized(dec, *a) if len(a) == 3 else lib.edge264_enable_packed(dec, *a)) == 0
if sys.argv[4] == '1':
    assert lib.edge264_enable_luma_only(dec) == 0
nal, out, f = base + 3 + (1 if data[2] == 0 else 0), [], pkg.Edge264Frame()
while True:
    sc = lib.edge264_find_start_code(nal, end, 0) if nal < end else end
    res = lib.edge264_decode_NAL(dec, nal, sc, None, None)
    while lib.edge264_get_frame(dec, ctypes.byref(f), 0) == 0:
        out.append((f.FrameId, pkg.frame_packed(lib, dec, f)))
    if res == errno.ENOBUFS:
        continue
    if nal >= end:
        break
    nal = sc + 3 if sc + 3 < end else end
pickle.dump(out, open(sys.argv[2], 'wb'))
"""


@pytest.mark.gpu
def test_device_packed_and_resized_outputs(workdir):
    """NV12 at k = 0 and 2 and NV12 resized to 224x224, in host memory and (E264B_OUTPUT=device) in device memory: Y plane
    equal to the full decode's, chroma 128."""
    lib = pkg.load()
    for s in (next(x for x in DPB_STREAMS if x[0] == "crop_rect"), next(x for x in STREAMS if x[0] == "b_explicit")):
        data = _data(workdir, s)
        src = os.path.join(workdir, "luma_dev.264")
        open(src, "wb").write(data)
        for key, arg in (("packed", (pkg.PACKED_NV12, 0)), ("packed", (pkg.PACKED_NV12, 2)), ("resized", (pkg.PACKED_NV12, 224, 224))):
            full = pkg.decode_bytes(data, lib, **{key: arg})[0]
            luma = pkg.decode_bytes(data, lib, luma_only=True, **{key: arg})[0]
            _same_packed(full, luma, "%s %s host" % (s[0], arg))
            assert all(f[-1]["on_device"] == 0 for f in luma)
            dev = {}
            for lo in (0, 1):
                out = os.path.join(workdir, "luma_dev_%d.pkl" % lo)
                subprocess.run([sys.executable, "-c", _SUB, src, out, ROOT, str(lo)] + [str(x) for x in arg], check=True, env=dict(os.environ, E264B_OUTPUT="device"), timeout=300)
                dev[lo] = pickle.load(open(out, "rb"))
                assert all(p["on_device"] == 1 for _, p in dev[lo])
            _same_packed([(i, p) for i, p in dev[0]], [(i, p) for i, p in dev[1]], "%s %s device" % (s[0], arg))
            assert [p["y"].tobytes() for _, p in dev[1]] == [f[-1]["y"].tobytes() for f in luma]


def _bench_decode(data, luma, keep):
    """The benchmark's application loop (tools/libe264bench.so: 8 application threads, 2 parse-ahead workers per decoder)
    over the streams; returns (frames, checksums, decoders).  E264_BENCH_LUMA_ONLY selects the mode."""
    bench = ctypes.CDLL(os.path.join(ROOT, "tools", "libe264bench.so"))
    bench.e264bench_run.restype = ctypes.c_double
    bench.e264bench_run.argtypes = [ctypes.POINTER(ctypes.c_char_p), ctypes.POINTER(ctypes.c_size_t), ctypes.c_int, ctypes.c_int,
                                    ctypes.c_int, ctypes.POINTER(ctypes.c_long), ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_void_p)]
    N = len(data)
    saved = {k: os.environ.get(k) for k in ("E264B_KEEP", "E264_BENCH_DEC_THREADS", "E264_BENCH_LUMA_ONLY")}
    try:
        os.environ["E264B_KEEP"] = "1" if keep else "0"; os.environ["E264_BENCH_DEC_THREADS"] = "2"; os.environ["E264_BENCH_LUMA_ONLY"] = "1" if luma else "0"
        bufs = (ctypes.c_char_p * N)(*data); sizes = (ctypes.c_size_t * N)(*map(len, data))
        frames = (ctypes.c_long * N)(); sums = (ctypes.c_uint64 * N)(); decs = (ctypes.c_void_p * N)()
        bench.e264bench_run(bufs, sizes, N, 8, 1, frames, sums, decs)
        return list(frames), list(sums), decs, bench
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


@pytest.mark.gpu
def test_replay_and_counts_at_the_benchmark_shape(workdir):
    """16 streams of the benchmark's 1080p workload through the benchmark's loop: luma-only checksums equal the port's
    luma-only frames; the same kernel launches per picture as a full decode, fewer bytes to the device, the same bytes
    back; a kernel-only replay of the luma-only decoders leaves every frame slot as the live decode did."""
    from bench import CONFIGS, ReplayStats
    from test_in_flight import _core, _stream_sum
    cfg = CONFIGS["1080p"]
    N, F = 16, 8
    paths = [make_stream(workdir, "bench_%d" % (cfg["seed0"] + i), cfg["w"], cfg["h"], "-n %d -s %d %s" % (F, cfg["seed0"] + i, cfg["gen"])) for i in range(N)]
    data = [open(p, "rb").read() for p in paths]
    port = checkers.load("port")
    with ThreadPoolExecutor(8) as ex:
        port_sums = list(ex.map(lambda d: _stream_sum(pkg.decode_bytes(d, port, luma_only=True)[0]), data))
    core = _core()
    core.e264b_replay.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ReplayStats)]
    stats = {}
    for luma in (False, True):
        frames, sums, decs, bench = _bench_decode(data, luma, keep=luma)
        assert frames == [F] * N
        devs = [core.e264b_of_decoder(d) for d in decs]
        tot = [0, 0, 0]
        for d in devs:
            v = [ctypes.c_uint64() for _ in range(3)]
            core.e264b_stats(d, *[ctypes.byref(x) for x in v])
            tot = [a + b.value for a, b in zip(tot, v)]
        stats[luma] = tot
        if luma:
            assert sums == port_sums, "the luma-only checksums differ from the port's luma-only frames"
            hashes = [[core.e264b_slot_hash(d, s) for s in range(core.e264b_slot_count(d))] for d in devs]
            arr = (ctypes.c_void_p * N)(*devs)
            st = ReplayStats()
            assert core.e264b_replay(arr, N, 2, 1, ctypes.byref(st)) == 0
            assert [core.e264b_error_flag(d) for d in devs] == [0] * N
            assert [[core.e264b_slot_hash(d, s) for s in range(core.e264b_slot_count(d))] for d in devs] == hashes
            assert st.launches == tot[0] * 2
        bench.e264bench_free.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int]
        bench.e264bench_free(decs, N)
    (lf, hf, df), (ll, hl, dl) = stats[False], stats[True]
    print("per picture: launches %.2f / %.2f, H2D %.0f / %.0f bytes, D2H %.0f / %.0f bytes (full / luma only)" % (
        lf / (N * F), ll / (N * F), hf / (N * F), hl / (N * F), df / (N * F), dl / (N * F)))
    assert ll == lf and dl == df and hl < hf
