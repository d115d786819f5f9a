"""Edge264Frame.mb_errors: the per-macroblock error map (0..100 per macroblock of the coded picture, NULL when every value
is 0).  Sources: 100 for concealed macroblocks and for inter macroblocks predicted from a missing reference, the
reference decoder's ramp for the macroblocks a broken slice delivered; the device carries them forward through motion
vectors and intra neighbours.  CPU tests run the product's host sources over the plain-C restatement of the
reconstruction (oracle/port_recon.c) and of the error maps (tests/native/port_error_map.c), bound by
tests/native/port_outputs_backend.c into a library built here; the GPU tests compare the device's maps and samples with it."""
import ctypes, errno, os, subprocess
import pytest
from conftest import ROOT, STREAMS, DPB_STREAMS, make_stream
from api_helpers import lib_of, new_decoder, free_decoder, loop, _ALLOC, _FREE, _cudart, _damaged
import edge264_b200 as pkg
import checkers


def _nals(data):
    """(start, end) of every NAL unit payload of an Annex-B stream (start points at the NAL header byte)."""
    out, i, n = [], 0, len(data)
    starts = []
    while True:
        j = data.find(b"\x00\x00\x01", i)
        if j < 0:
            break
        starts.append(j + 3)
        i = j + 3
    for k, s in enumerate(starts):
        e = starts[k + 1] - 3 if k + 1 < len(starts) else n
        while k + 1 < len(starts) and e > s and data[e - 1] == 0:
            e -= 1
        out.append((s, e))
    return out


def _ue(bits, pos):
    z = 0
    while bits[pos + z] == "0":
        z += 1
    return int(bits[pos + z:pos + 2 * z + 1], 2) - 1, pos + 2 * z + 1


def _slice_head(nal):
    """(nal_ref_idc, nal_unit_type, first_mb_in_slice, slice_type % 5) of a slice NAL unit."""
    rb = nal[1:40].replace(b"\x00\x00\x03", b"\x00\x00")
    bits = "".join(format(b, "08b") for b in rb)
    first, p = _ue(bits, 0)
    st, _ = _ue(bits, p)
    return nal[0] >> 5, nal[0] & 31, first, st % 5


NATIVE = os.path.join(ROOT, "tests", "native")
def decode(data, backend="port", n_threads=0, samples=True):
    """The README loop; per frame (FrameId, samples or None, map bytes or None, stride_mb), and per NAL its return code.
    backend: "port" (CPU, with error maps), "gpu", or "oracle" (oracle/liboracle_dec.so: a backend without error maps)."""
    lib = checkers.load("port") if backend == "oracle" else lib_of(backend)
    buf = ctypes.create_string_buffer(data, len(data) + 64)
    base = ctypes.addressof(buf); end = base + len(data)
    dec = lib.edge264_alloc(n_threads, None, None, 0, None, None, None)
    assert dec
    nal = base + 3 + (1 if data[2] == 0 else 0)
    frames, codes, f = [], [], pkg.Edge264Frame()
    while True:
        sc = lib.edge264_find_start_code(nal, end, 0) if nal < end else end
        before = len(frames)
        res = lib.edge264_decode_NAL(dec, nal, sc, None, None)
        while lib.edge264_get_frame(dec, ctypes.byref(f), 0) == 0:
            frames.append((f.FrameId, pkg._frame_bytes(f) if samples else None, pkg._frame_errors(f), f.stride_mb))
        if res == errno.ENOBUFS:
            if len(frames) == before:
                break
            continue
        codes.append(res)
        if nal >= end:
            break
        nal = sc + 3 if sc + 3 < end else end
    d = ctypes.c_void_p(dec)
    lib.edge264_free(ctypes.byref(d))
    return frames, codes


def ramp(n, cabac):
    """Error of the macroblocks 0..n-1 a broken slice delivered: a literal restatement of the reference's recover_slice
    (edge264_headers.c:305-311) with its ppow (:266-275)."""
    def ppow(p, k):
        r = 65536
        while k:
            if k & 1:
                r = (r * p) >> 16
            p = (p * p) >> 16
            k >>= 1
        return r
    out = []
    div = 65536 - ppow(65194, n)
    for i in range(n):
        p12800 = ((i + 1) * 12800 + n - 1) // n if not cabac else ((div - (65536 - ppow(65194, n - 1 - i))) * 12800 + div - 1) // div
        out.append(p12800 >> 7)
    return out


# ---- 1. clean streams: no map, stride_mb as before ----
@pytest.mark.parametrize("name,w,h,args", STREAMS + DPB_STREAMS, ids=[s[0] for s in STREAMS + DPB_STREAMS])
def test_clean_streams_have_no_error_map(workdir, name, w, h, args):
    data = open(make_stream(workdir, name, w, h, args), "rb").read()
    frames, _ = decode(data)
    assert frames
    for fid, _, m, stride in frames:
        assert m is None, "frame %d has an error map" % fid
        assert stride == ctypes.c_int16(w * 304).value, stride


def test_backend_without_maps_reports_none(workdir):
    """A backend that keeps no error maps (oracle/port_backend.c) yields NULL maps, even on a truncated slice."""
    name, w, h, args, _ = TRUNC_STREAMS[0]
    for frac, dmg, _ in _truncations(workdir, name, w, h, args)[4]:
        frames, _ = decode(dmg, "oracle")
        assert frames and all(f[2] is None for f in frames), frac


# ---- 2. truncated slices ----
TRUNC_STREAMS = [
    ("mberr_cavlc", 8, 6, "-n 14 -s 201 --gop IPB --slices 3 --idr 8 --cavlc --deblock 0", False),
    ("mberr_cabac", 8, 6, "-n 14 -s 202 --gop IPB --slices 3 --idr 8 --deblock 0 --t8x8 50", True),
]


def _truncations(workdir, name, w, h, args):
    """The stream, the index of the picture (decoding order) whose second slice is cut, that slice's macroblock range,
    and the damaged streams at several cut offsets with the index of the cut NAL unit."""
    data = open(make_stream(workdir, name, w, h, args), "rb").read()
    nals = _nals(data)
    pic, target, pics_seen, idr_after = -1, None, [], None
    for k, (s, e) in enumerate(nals):
        if data[s] & 31 not in (1, 5):
            continue
        ref, typ, first, st = _slice_head(data[s:e])
        if first == 0:
            pic += 1
            pics_seen.append((pic, typ))
        if target is None and pic > 0 and ref and st == 0 and first != 0 and typ == 1:
            target = (k, pic, first)
        elif target and typ == 5 and first == 0 and idr_after is None and pic > target[1]:
            idr_after = pic
    assert target and idr_after, "stream without a reference P picture before an IDR"
    k, pic, first = target
    s_next = None
    for s, e in nals[k + 1:]:
        if data[s] & 31 in (1, 5):
            r2, _, f2, _ = _slice_head(data[s:e])
            s_next = f2 if f2 != 0 else w * h
            break
    s, e = nals[k]
    cuts = []
    for frac in (0.3, 0.45, 0.6, 0.75, 0.9):
        cut = s + max(6, int((e - s) * frac))
        cuts.append((frac, data[:cut] + data[e:], k))
    return data, pic, (first, s_next), idr_after, cuts


@pytest.mark.parametrize("name,w,h,args,cabac", TRUNC_STREAMS, ids=[t[0] for t in TRUNC_STREAMS])
def test_truncated_slice_ramp(workdir, name, w, h, args, cabac):
    data, pic, (s0, s1), idr_after, cuts = _truncations(workdir, name, w, h, args)
    clean, _ = decode(data)
    ids = sorted(f[0] for f in clean)      # FrameIds grow in decoding order: picture k has ids[k]
    checked = 0
    for frac, dmg, k in cuts:
        frames, codes = decode(dmg)
        if codes[k] != errno.EBADMSG:
            continue
        checked += 1
        by_id = {f[0]: f[2] for f in frames}
        maps = {k: by_id[i] for k, i in enumerate(ids)}
        m = maps[pic]
        assert m is not None and len(m) == w * h
        region = list(m[s0:s1])
        n = next((n for n in range(len(region) + 1) if region == ramp(n, cabac) + [100] * (len(region) - n)), None)
        assert n is not None, (frac, region)
        assert not any(m[:s0]) and not any(m[s1:]), frac
        assert any(maps[p] is not None for p in range(pic + 1, idr_after)), frac
        assert all(maps[p] is None for p in maps if p >= idr_after), frac
    assert checked >= 2, "too few cuts answered EBADMSG"


def test_ramp_restatement_matches_the_reference_formula():
    assert ramp(1, False) == [100] and ramp(1, True) == [100]
    assert ramp(4, False) == [25, 50, 75, 100]
    c = ramp(200, True)
    assert c[-1] == 100 and all(a <= b for a, b in zip(c, c[1:]))


# ---- 3. damaged streams ----
def test_damaged_streams_maps(workdir):
    """Values in 0..100, the same on a second run; where the samples agree across worker counts the maps agree too."""
    agree = total = 0
    for name, seed, data in _damaged(workdir):
        runs = {t: decode(data, n_threads=t)[0] for t in (0, 1, 3)}
        again = decode(data)[0]
        assert [f[2] for f in again] == [f[2] for f in runs[0]], "%s seed %d: maps differ on a second run" % (name, seed)
        for t, frames in runs.items():
            for f in frames:
                assert f[2] is None or max(f[2]) <= 100
        total += 1
        base = runs[0]
        if all([(f[0], f[1]) for f in fr] == [(f[0], f[1]) for f in base] for fr in runs.values()):
            agree += 1
            for t, fr in runs.items():
                assert [f[2] for f in fr] == [f[2] for f in base], "%s seed %d: maps differ with %d workers" % (name, seed, t)
    print("damaged streams whose samples agree for 0, 1 and 3 workers: %d of %d" % (agree, total))
    assert total == 75


def test_damaged_streams_keep_the_err_contract(workdir, monkeypatch):
    """E264_CHECK_RECORDS=1: every picture the parser submits keeps the record contract, err <= 100 included."""
    lib = checkers.port_outputs_lib()
    monkeypatch.setenv("E264_CHECK_RECORDS", "1")
    for name, seed, data in _damaged(workdir):
        for t in (0, 1, 3):
            decode(data, n_threads=t, samples=False)
            assert lib.e264_test_record_violations() == 0, "%s seed %d (%d workers): %s" % (name, seed, t, lib.e264_test_last_violation())


# ---- 5. the device against the port ----
def _all_inputs(workdir):
    for name, w, h, args in STREAMS + DPB_STREAMS:
        yield name, open(make_stream(workdir, name, w, h, args), "rb").read()
    for name, w, h, args, _ in TRUNC_STREAMS:
        for frac, dmg, _ in _truncations(workdir, name, w, h, args)[4]:
            yield "%s@%.2f" % (name, frac), dmg
    for name, seed, data in _damaged(workdir):
        yield "%s/%d" % (name, seed), data


@pytest.mark.gpu
def test_device_maps_match_port(workdir):
    for label, data in _all_inputs(workdir):
        for t in (0, 3):
            g, gc = decode(data, "gpu", t)
            p, pc = decode(data, "port", t)
            assert [f[0] for f in g] == [f[0] for f in p], (label, t)
            for a, b in zip(g, p):
                assert a[1] == b[1], "%s (%d workers) frame %d: samples differ" % (label, t, a[0])
                assert a[2] == b[2], "%s (%d workers) frame %d: maps differ" % (label, t, a[0])
                assert a[3] == b[3], (label, t, a[0])


# ---- 7. device memory output: the map stays in host memory ----
def _maps_with_device_samples(data):
    """Decode with alloc_cb handing out device memory (cudaMalloc); returns the maps only."""
    cudart = _cudart()

    def alloc(samples, size, mbs, mbs_size, err, arg):
        p = ctypes.c_void_p()
        assert cudart.cudaMalloc(ctypes.byref(p), ctypes.c_size_t(size)) == 0
        samples[0] = p.value
    def free(samples, mbs, arg):
        cudart.cudaFree(ctypes.c_void_p(samples))
    cbs = (_ALLOC(alloc), _FREE(free))
    lib = pkg.load()
    dec, maps = new_decoder(lib, alloc=cbs), []
    loop(lib, dec, data, lambda f: maps.append((f.FrameId, pkg._frame_errors(f))))   # host memory: readable without a copy
    free_decoder(lib, dec)
    return maps


@pytest.mark.gpu
def test_device_memory_output_keeps_host_maps(workdir):
    name, w, h, args, _ = TRUNC_STREAMS[1]
    cuts = _truncations(workdir, name, w, h, args)[4]
    for frac, dmg, _ in cuts:
        host = [(f[0], f[2]) for f in decode(dmg, "gpu")[0]]
        assert _maps_with_device_samples(dmg) == host, frac
        code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import test_mb_errors as t; "
                "open(sys.argv[1], 'wb').write(repr([(f[0], f[2]) for f in t.decode(open(sys.argv[2], 'rb').read(), 'gpu', samples=False)[0]]).encode())"
                % (ROOT, os.path.join(ROOT, "tests")))
        src = os.path.join(workdir, "mberr_dev.264"); out = os.path.join(workdir, "mberr_dev.txt")
        open(src, "wb").write(dmg)
        subprocess.run([__import__("sys").executable, "-c", code, out, src], check=True, env=dict(os.environ, E264B_OUTPUT="device"), timeout=300)
        assert open(out).read() == repr(host), frac


# ---- 4 / 6. the record fuzzer with error maps ----
FUZZ_SRC = [os.path.join(NATIVE, "record_fuzz_maps.c"), os.path.join(NATIVE, "port_error_map.c"), os.path.join(ROOT, "oracle", "port_recon.c"),
            os.path.join(ROOT, "oracle", "record_check.c")]
MAP_COUNTERS = ["map_clamp_left", "map_clamp_right", "map_clamp_top", "map_clamp_bottom", "map_window_1mb", "map_window_2mb", "map_window_4mb",
                "map_int16_vector", "map_max_from_list1", "map_tainted_slot_unread", "map_intra_c_4x4_blk5", "map_intra_c_8x8_blk1", "map_read_all100_slot"]


@pytest.fixture(scope="module")
def fuzzer(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("mberr_fuzz") / "record_fuzz_maps")
    subprocess.run(["gcc", "-O2", "-std=gnu11", "-w"] + FUZZ_SRC + ["-o", exe, "-ldl"], check=True)
    return exe


def _counters(out):
    import re
    return {m.group(1): int(m.group(2)) for m in re.finditer(r"^cov (\S+) (\d+)$", out, re.M)}


def test_fuzzer_error_map_draws_reach_every_case(fuzzer):
    r = subprocess.run([fuzzer, "--cpu-only", "--seeds", "0-35"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    cov = _counters(r.stdout)
    zero = [k for k in MAP_COUNTERS if not cov.get(k)]
    assert not zero, "error-map cases never drawn: %s" % zero


def test_fuzzer_error_map_draws_leave_the_record_draws_alone(fuzzer, tmp_path):
    """The error-map draws come from a stream of their own: the driver runs record_fuzz's pictures, as many of them."""
    plain = str(tmp_path / "record_fuzz")
    subprocess.run(["gcc", "-O2", "-std=gnu11", "-w", os.path.join(NATIVE, "record_fuzz.c"), os.path.join(ROOT, "oracle", "port_recon.c"),
                    os.path.join(ROOT, "oracle", "record_check.c"), "-o", plain, "-ldl"], check=True)
    a = subprocess.run([plain, "--cpu-only", "--seeds", "0-7"], capture_output=True, text=True, timeout=600)
    b = subprocess.run([fuzzer, "--cpu-only", "--seeds", "0-7"], capture_output=True, text=True, timeout=600)
    assert a.returncode == 0 and b.returncode == 0
    assert _counters(a.stdout)["pictures"] == _counters(b.stdout)["pictures"] > 0
    assert a.stdout.splitlines()[-1] == b.stdout.splitlines()[-1]


@pytest.mark.gpu
def test_device_maps_match_port_on_fuzzed_records(fuzzer):
    lib = os.path.join(ROOT, "edge264_b200", "libedge264_b200.so")
    r = subprocess.run([fuzzer, "--lib", lib, "--seeds", "0-35"], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-500:], r.stderr[-3000:])
    assert _counters(r.stdout)["pictures"] >= 500
