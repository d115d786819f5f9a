"""Skipping the loop filter (include/edge264_loopfilter.h): EDGE264_LOOP_FILTER_REF outputs every non-reference picture
without deblocking, EDGE264_LOOP_FILTER_NONE every picture.  A picture whose filter is skipped is defined as the same
picture with disable_deblocking_filter_idc 1 in every slice, so the oracle is a twin stream: tools/gen264 --deblock-off
nonref|all writes the same stream with idc 1 in the slices of those pictures and every other bit unchanged.
  - The mode's decode of a stream equals the full decode of its twin, on the restatement and on the device, and the
    compiled reference decoder (oracle/_ref) decodes the twins to the same frames, so the oracle is not this project's
    code alone.
  - Under REF every reference picture is the full decode's, and every non-reference frame is the picture before
    deblocking, which tests/spec_picture.py composes from the picture's records (the statement the pictures before
    deblocking are judged by in tests/test_picture_spec.py).

CPU tests run the product's host sources over the plain-C restatement (oracle/liboracle_dec.so, and the test backends
of tests/checkers.py and tests/picture_dumps.py); the GPU tests compare the device with the restatement and with the
device's own decode of the twins, and count its launches."""
import ctypes, errno, os, pickle, random, subprocess, sys
from concurrent.futures import ThreadPoolExecutor
import numpy as np
import pytest
from conftest import ROOT, STREAMS, DPB_STREAMS, make_stream, have
from test_limits import LIMITS, FULL_LIMITS
from test_gpu_parity import FULL
from test_skip import pictures, decode, stats_per_nal
from api_helpers import _damaged
from checkers import port_outputs_lib
from picture_dumps import load_dump, port_dbk_lib
import spec_deblock as sd
import edge264_b200 as pkg
import checkers

ALL, REF, NONE = pkg.LOOP_FILTER_ALL, pkg.LOOP_FILTER_REF, pkg.LOOP_FILTER_NONE
TWIN = {REF: "nonref", NONE: "all"}
SETS = STREAMS + DPB_STREAMS + LIMITS
IDS = [s[0] for s in SETS]


def _data(workdir, s, mode=ALL):
    """The stream s (name, width_mbs, height_mbs, generator arguments), or its twin for mode (REF / NONE)."""
    name, w, h, args = s
    if mode == ALL:
        return open(make_stream(workdir, name, w, h, args), "rb").read()
    return open(make_stream(workdir, "%s_off_%s" % (name, TWIN[mode]), w, h, "%s --deblock-off %s" % (args, TWIN[mode])), "rb").read()


def _by_name(name):
    return next(s for s in SETS + FULL + FULL_LIMITS if s[0] == name)


def _set_at(hooks):
    """a before hook of test_skip.decode: edge264_set_loop_filter(dec, hooks[k]) before NAL unit k"""
    return lambda k, lib, dec: k in hooks and lib.edge264_set_loop_filter(dec, hooks[k])


# ---- CPU: the twin streams ----
def test_twins_differ_from_their_stream_in_slice_headers_only(workdir):
    """With --deblock 1 every slice already has idc 1: both twins are the stream byte for byte (the generator draws the
    filter offsets either way).  Otherwise the twins are as long as the stream or shorter, with as many NAL units."""
    plain = ("plain_idc1", 9, 7, "-n 10 -s 15 --gop IPB --deblock 1 --wp 1")
    assert _data(workdir, plain, REF) == _data(workdir, plain) == _data(workdir, plain, NONE)
    s = _by_name("b_explicit")
    d, n, a = _data(workdir, s), _data(workdir, s, REF), _data(workdir, s, NONE)
    assert len(a) < len(n) < len(d) and d.count(b"\x00\x00\x01") == n.count(b"\x00\x00\x01") == a.count(b"\x00\x00\x01")
    r = subprocess.run([os.path.join(ROOT, "tools", "gen264"), "-o", os.path.join(workdir, "bad.264"), "--deblock-off", "some"], capture_output=True, text=True)
    assert r.returncode == 2 and "--deblock-off" in r.stderr


@pytest.mark.parametrize("stream", SETS, ids=IDS)
def test_port_modes_equal_the_full_decode_of_the_twins(workdir, stream):
    """REF and NONE equal the full decode of the nonref and all twins, frames and return codes, with 0 and 3 workers;
    the compiled reference decodes the twins to the same frames."""
    lib = checkers.load("port")
    data = _data(workdir, stream)
    for mode in (REF, NONE):
        twin = pkg.decode_bytes(_data(workdir, stream, mode), lib)
        for t in (0, 3):
            assert pkg.decode_bytes(data, lib, t, loop_filter=mode) == twin, (stream[0], TWIN[mode], t)
        if have("ref"):
            ref = pkg.decode_bytes(_data(workdir, stream, mode), checkers.load("ref"))[0]
            assert [f[:4] for f in ref] == [f[:4] for f in twin[0]], "%s: the reference decodes the %s twin differently" % (stream[0], TWIN[mode])


@pytest.mark.parametrize("stream", SETS, ids=IDS)
def test_port_ref_mode_keeps_every_reference_picture(workdir, stream):
    """Under REF the frame of every reference picture is the full decode's (no drift); only non-reference frames change,
    and some do wherever the filter changes a non-reference picture (at QP 2 it changes none)."""
    lib = checkers.load("port")
    data = _data(workdir, stream)
    pics = pictures(data)
    full, got = pkg.decode_bytes(data, lib)[0], pkg.decode_bytes(data, lib, loop_filter=REF)[0]
    assert [f[:3] for f in got] == [f[:3] for f in full] and len(full) == len(pics)
    ref_of = dict(zip(sorted(f[0] for f in full), (p["ref"] for p in pics)))   # FrameIds grow in decoding order
    changed = [a[0] for a, b in zip(full, got) if a != b]
    assert not [i for i in changed if ref_of[i]], "%s: reference frames changed" % stream[0]
    if pkg.decode_bytes(_data(workdir, stream, REF), lib)[0] != full:
        assert changed, "%s: no non-reference frame changed" % stream[0]


# streams without cropping whose non-reference pictures are deblocked
COMPOSED = ["b_default", "b_explicit", "b_implicit_temporal", "b_cavlc_all", "ragged_2xN", "pb_intra_heavy", "nonref_p",
            "mixed_slices_cabac", "direct4x4_temporal", "bref_implicit"]


def composed_pictures(workdir, tmp_path, name):
    """The stream's pictures under REF through the parser and the restatement's dump backend (tests/picture_dumps.py),
    decoding order, with each picture's nal_ref_idc and output frame; the full decode's frames."""
    s = _by_name(name)
    data = _data(workdir, s)
    dump = str(tmp_path / (name + ".dbk"))
    os.environ["E264_DBK_DUMP"] = dump
    try:
        frames = pkg.decode_bytes(data, port_dbk_lib(), loop_filter=REF)[0]
    finally:
        del os.environ["E264_DBK_DUMP"]
    pics, heads = load_dump(dump), pictures(data)
    assert len(pics) == len(heads) == len(frames)
    by_id = {f[0]: f for f in frames}
    out = [(p, h["ref"], by_id[i]) for p, h, i in zip(pics, heads, sorted(by_id))]
    return out, pkg.decode_bytes(data, checkers.load("port"))[0]


def frame_of(pic):
    """the I420 bytes of a dumped picture before deblocking (no cropping)"""
    g = {k: int(pic.pd[k]) for k in ("width_mbs", "height_mbs", "stride_y", "stride_c", "plane_y")}
    return b"".join(p[0].astype(np.uint8).tobytes() for p in sd.planes_of(pic.pre[None], g))


def test_port_non_reference_frames_are_the_composition(workdir, tmp_path):
    """Under REF a non-reference picture carries no deblocking (any_deblock 0, after == before), its frame is the picture
    before deblocking, and tests/spec_picture.py composes that picture from its records; every reference picture keeps its
    deblocking and its frame is the full decode's."""
    from test_picture_spec import judge
    n = 0
    for name in COMPOSED:
        pics, full = composed_pictures(workdir, tmp_path, name)
        full = {f[0]: f for f in full}
        nonref = [p for p, ref, _ in pics if not ref]
        for p, ref, f in pics:
            assert f[1] == 16 * int(p.pd["width_mbs"]) and f[2] == 16 * int(p.pd["height_mbs"])
            if ref:
                assert int(p.pd["any_deblock"]) == 1 and f == full[f[0]], "%s: reference frame %d" % (name, f[0])
            else:
                assert int(p.pd["any_deblock"]) == 0 and np.array_equal(p.pre, p.post), "%s: frame %d was deblocked" % (name, f[0])
                assert f[3] == frame_of(p), "%s: frame %d is not its picture before deblocking" % (name, f[0])
        r = judge(nonref, name)
        assert not r["failures"], "\n".join(r["failures"][:5])
        n += len(nonref)
    assert n >= 60


# ---- CPU: switching modes ----
def test_port_mode_switches_apply_from_the_next_picture(workdir):
    """ALL -> REF between the two slices of a non-reference picture, then back to ALL and to REF again at later pictures:
    a picture keeps the mode of its first slice, for 0, 1 and 3 workers alike."""
    s = _by_name("b_scaling_mv")   # two slices per picture
    data = _data(workdir, s)
    pics = pictures(data)
    nonref = [p for p in pics if p["ref"] == 0]
    assert len(nonref) >= 5 and len(nonref[0]["nals"]) == 2
    hooks = {nonref[0]["nals"][1]: REF, nonref[2]["nals"][0]: ALL, nonref[3]["nals"][1]: REF}
    def mode_at(k):   # the mode when decode_NAL of NAL unit k runs
        return ([ALL] + [m for j, m in sorted(hooks.items()) if j <= k])[-1]
    mode_of = [mode_at(p["nals"][0]) for p in pics]
    assert [m for m, p in zip(mode_of, pics) if not p["ref"]][:5] == [ALL, REF, ALL, ALL, REF]
    full = {f[0]: f for f in decode(data)[0]}
    twin = {f[0]: f for f in decode(_data(workdir, s, REF))[0]}
    want = {i: (twin if m == REF else full)[i] for i, m in zip(sorted(full), mode_of)}
    runs = []
    for t in (0, 1, 3):
        got, codes = decode(data, n_threads=t, before=_set_at(hooks))
        assert [f[0] for f in got] == list(full) and all(f == want[f[0]] for f in got), "%d workers" % t
        runs.append((got, codes))
    assert runs[1] == runs[0] and runs[2] == runs[0]


def test_port_switch_to_none_and_back(workdir):
    """NONE from the first picture, ALL from an IDR picture on: before it the all twin's frames, from it the full
    decode's."""
    s = _by_name("dpb_mmco_cabac")   # IDR pictures every 17
    data = _data(workdir, s)
    pics = pictures(data)
    idr = [i for i, p in enumerate(pics) if p["type"] == 5]
    assert len(idr) >= 2
    k = pics[idr[1]]["nals"][0]
    full, _ = decode(data)
    twin, _ = decode(_data(workdir, s, NONE))
    ids = sorted(f[0] for f in full)
    first_after = ids[idr[1]]
    for t in (0, 3):
        got, _ = decode(data, n_threads=t, before=_set_at({0: NONE, k: ALL}))
        src = {f[0]: f for f in twin if f[0] < first_after}
        src.update({f[0]: f for f in full if f[0] >= first_after})
        assert [f[0] for f in got] == [f[0] for f in full]
        assert all(f == src[f[0]] for f in got), t


# ---- CPU: the mode with the other features ----
def _same_outputs(a, b, label):
    assert [f[:4] for f in a[0]] == [f[:4] for f in b[0]] and a[1] == b[1], label
    for x, y in zip(a[0], b[0]):
        for u, v in zip(x[4:], y[4:]):
            if isinstance(u, dict):
                assert u.keys() == v.keys() and all(np.array_equal(u[k], v[k]) if isinstance(u[k], np.ndarray) else u[k] == v[k] for k in u), "%s: frame %d" % (label, x[0])
            else:
                assert u == v, "%s: frame %d" % (label, x[0])


COMBOS = [dict(skip=pkg.SKIP_NONREF), dict(skip=pkg.SKIP_NONKEY), dict(luma_only=True), dict(errors=True, motion=True),
          dict(packed=(pkg.PACKED_NV12, 0)), dict(packed=(pkg.PACKED_I420, 1)), dict(resized=(pkg.PACKED_NV12, 40, 26)),
          dict(picstats=True), dict(luma_only=True, errors=True, picstats=True, skip=pkg.SKIP_NONKEY)]


@pytest.mark.parametrize("kw", COMBOS, ids=["-".join(sorted(k)) + "-%d" % i for i, k in enumerate(COMBOS)])
def test_port_combinations_equal_the_twins(workdir, kw):
    """With skip, luma-only, error maps, the motion export and the packed, resized and statistics outputs, each output of
    the mode's decode equals the same output of the twin's full decode: each follows its definition on the frame as
    output."""
    lib = port_outputs_lib()
    for name in ("b_explicit", "crop_rect", "mixed_slices_cavlc", "bref_spatial", "pb_intra_heavy"):
        s = _by_name(name)
        data = _data(workdir, s)
        for mode in (REF, NONE):
            _same_outputs(pkg.decode_bytes(data, lib, loop_filter=mode, **kw), pkg.decode_bytes(_data(workdir, s, mode), lib, **kw), "%s %s %s" % (name, TWIN[mode], kw))
    if kw.get("skip") == pkg.SKIP_NONREF:   # nothing left to leave unfiltered under REF
        data = _data(workdir, _by_name("b_explicit"))
        assert pkg.decode_bytes(data, lib, loop_filter=REF, **kw) == pkg.decode_bytes(data, lib, **kw)


# ---- CPU: damaged streams ----
def test_port_damaged_streams(workdir, tmp_path, monkeypatch):
    """The damaged streams of test_robustness.py under REF and NONE: every picture submitted keeps the record contract;
    return codes, FrameIds and error maps are the full decode's.  Under REF, through the dump backend, every picture is
    constructed as in the full decode (no drift) and is output either deblocked as in the full decode or, when its
    deblocking was left out, as its picture before deblocking."""
    lib = port_outputs_lib()
    monkeypatch.setenv("E264_CHECK_RECORDS", "1")
    before, n, unfiltered = lib.e264_test_record_violations(), 0, 0
    for name, seed, data in _damaged(workdir):
        for t in (0, 3):
            full = pkg.decode_bytes(data, lib, t, errors=True)
            for mode in (REF, NONE):
                got = pkg.decode_bytes(data, lib, t, errors=True, loop_filter=mode)
                assert got[1] == full[1] and [(f[0], f[4]) for f in got[0]] == [(f[0], f[4]) for f in full[0]], "%s seed %d" % (name, seed)
        dumps = {}
        for mode in (ALL, REF):
            monkeypatch.setenv("E264_DBK_DUMP", str(tmp_path / ("%d.dbk" % mode)))
            pkg.decode_bytes(data, port_dbk_lib(), loop_filter=mode)
            monkeypatch.delenv("E264_DBK_DUMP")
            dumps[mode] = load_dump(str(tmp_path / ("%d.dbk" % mode)))
        assert len(dumps[ALL]) == len(dumps[REF])
        for a, b in zip(dumps[ALL], dumps[REF]):
            assert np.array_equal(a.pre, b.pre), "%s seed %d: a picture is constructed differently" % (name, seed)
            if int(b.pd["any_deblock"]):
                assert np.array_equal(a.post, b.post)
            else:
                assert np.array_equal(b.post, b.pre)
                unfiltered += int(a.pd["any_deblock"])
        n += 1
    assert n == 75 and unfiltered > 0
    assert lib.e264_test_record_violations() == before, lib.e264_test_last_violation()


# ---- CPU: API ----
def test_api_contract(workdir):
    lib = port_outputs_lib()
    assert lib.edge264_set_loop_filter(None, REF) == errno.EINVAL
    dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
    for mode in (3, -1, 100):
        assert lib.edge264_set_loop_filter(dec, mode) == errno.EINVAL
    for mode in (ALL, REF, NONE, ALL):
        assert lib.edge264_set_loop_filter(dec, mode) == 0
    d = ctypes.c_void_p(dec)
    lib.edge264_free(ctypes.byref(d))
    # ALL is the decoder without the call, the hook of every NAL unit included
    for name in ("b_explicit", "mixed_slices_cabac"):
        data = _data(workdir, _by_name(name))
        assert decode(data, n_threads=3, before=lambda k, lib, dec: lib.edge264_set_loop_filter(dec, ALL)) == decode(data, n_threads=3)
    if have("ref"):
        ref = checkers.load("ref")
        assert not hasattr(ref, "edge264_set_loop_filter")
        with pytest.raises(RuntimeError, match="ENOTSUP"):
            pkg.decode_bytes(_data(workdir, _by_name("b_default")), ref, loop_filter=REF)


# ---- GPU ----
@pytest.mark.gpu
@pytest.mark.parametrize("stream", SETS, ids=IDS)
def test_device_equals_port_and_twins(workdir, stream):
    """colour and luma-only, REF and NONE: the device equals the restatement and its own full decode of the twin"""
    lib, port = pkg.load(), checkers.load("port")
    data = _data(workdir, stream)
    for mode in (REF, NONE):
        twin = _data(workdir, stream, mode)
        for lo in (False, True):
            got = pkg.decode_bytes(data, lib, loop_filter=mode, luma_only=lo)
            assert got == pkg.decode_bytes(data, port, loop_filter=mode, luma_only=lo), "%s %s luma_only %s: device and port differ" % (stream[0], TWIN[mode], lo)
            assert got == pkg.decode_bytes(twin, lib, luma_only=lo), "%s %s luma_only %s: device and twin differ" % (stream[0], TWIN[mode], lo)


@pytest.mark.gpu
def test_device_non_reference_frames_are_the_composition(workdir, tmp_path):
    """The device's REF frames: every non-reference frame is the picture before deblocking that tests/spec_picture.py
    composes (judged on the restatement's dump of the same pictures), every reference frame the device's full decode's."""
    from test_picture_spec import judge
    lib = pkg.load()
    for name in COMPOSED:
        pics, _ = composed_pictures(workdir, tmp_path, name)
        data = _data(workdir, _by_name(name))
        full = {f[0]: f for f in pkg.decode_bytes(data, lib)[0]}
        dev = {f[0]: f for f in pkg.decode_bytes(data, lib, 2, loop_filter=REF)[0]}
        assert len(dev) == len(pics)
        for p, ref, f in pics:
            assert dev[f[0]][3] == (full[f[0]][3] if ref else frame_of(p)), "%s frame %d (reference %d)" % (name, f[0], ref)
        r = judge([p for p, ref, _ in pics if not ref], name)
        assert not r["failures"], "\n".join(r["failures"][:5])


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["1080p_ipb", "lim_1080p_qp_levels"])
def test_device_full_size(workdir, name):
    s = _by_name(name)
    lib = pkg.load()
    data = _data(workdir, s)
    for mode in (REF, NONE):
        got = pkg.decode_bytes(data, lib, 2, loop_filter=mode)
        assert got[0] and got[0][0][1:3] == (1920, 1080)
        assert got == pkg.decode_bytes(_data(workdir, s, mode), lib, 2), (name, TWIN[mode])
    assert pkg.decode_bytes(data, lib, loop_filter=REF, luma_only=True) == pkg.decode_bytes(_data(workdir, s, REF), lib, luma_only=True)


@pytest.mark.gpu
def test_many_decoders_in_flight(workdir):
    """8 host threads decode every stream in the three modes at once, twice, in shuffled orders, with 0 or 2 workers; each
    output equals its decoder's output alone."""
    lib = pkg.load()
    streams = STREAMS + DPB_STREAMS
    data = {s[0]: _data(workdir, s) for s in streams}
    jobs = [(n, m) for n in data for m in (ALL, REF, NONE)]
    alone = {j: pkg.decode_bytes(data[j[0]], lib, 0, loop_filter=j[1]) for j in jobs}
    for r in range(2):
        random.Random(r).shuffle(jobs)
        with ThreadPoolExecutor(8) as ex:
            got = list(ex.map(lambda ij: pkg.decode_bytes(data[ij[1][0]], lib, 2 * (ij[0] & 1), loop_filter=ij[1][1]), enumerate(jobs)))
        for j, g in zip(jobs, got):
            assert g == alone[j], j


# the samples are device memory: only the packed pictures are read (through torch)
_SUB = """
import sys, ctypes, errno, pickle
sys.path.insert(0, sys.argv[3])
import edge264_b200 as pkg
lib = pkg.load()
data = open(sys.argv[1], 'rb').read()
buf = ctypes.create_string_buffer(data, len(data) + 64); base = ctypes.addressof(buf); end = base + len(data)
dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
assert lib.edge264_enable_packed(dec, pkg.PACKED_NV12, 0) == 0 and lib.edge264_set_loop_filter(dec, int(sys.argv[4])) == 0
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
def test_device_memory_output(workdir):
    """E264B_OUTPUT=device: the packed NV12 output of the mode's decode equals that of the twin's full decode."""
    for name in ("b_explicit", "crop_rect"):
        s = _by_name(name)
        for mode in (REF, NONE):
            runs = []
            for src, m in ((_data(workdir, s), mode), (_data(workdir, s, mode), ALL)):
                path, out = os.path.join(workdir, "lf_dev.264"), os.path.join(workdir, "lf_dev.pkl")
                open(path, "wb").write(src)
                subprocess.run([sys.executable, "-c", _SUB, path, out, ROOT, str(m)], check=True, env=dict(os.environ, E264B_OUTPUT="device"), timeout=300)
                runs.append(pickle.load(open(out, "rb")))
            assert runs[0] and all(p["on_device"] == 1 for _, p in runs[0])
            assert [i for i, _ in runs[0]] == [i for i, _ in runs[1]]
            for (i, a), (_, b) in zip(*runs):
                assert np.array_equal(a["y"], b["y"]) and np.array_equal(a["cbcr"], b["cbcr"]), (name, TWIN[mode], i)


@pytest.mark.gpu
def test_launch_counts(workdir):
    """e264b_stats per picture: a picture whose filter is skipped has one launch fewer than in the full decode (no
    deblocking launch; a stream of disable_deblocking_filter_idc 1 has none to leave out) and the same copies; every other picture the full decode's launches and copies.  With ALL set on
    every NAL unit the counts and frames are those of a decoder that never made the call."""
    for name in ("b_default", "b_scaling_mv", "bref_spatial", "mixed_slices_cavlc", "nonref_p", "i_cabac_4x4"):
        data = _data(workdir, _by_name(name))
        pics = pictures(data)
        full, ffull = stats_per_nal(data, pkg.SKIP_NONE)
        same, fsame = stats_per_nal(data, pkg.SKIP_NONE, lambda k, lib, dec: lib.edge264_set_loop_filter(dec, ALL))
        assert same == full and fsame == ffull, name
        for mode in (REF, NONE):
            part, _ = stats_per_nal(data, pkg.SKIP_NONE, _set_at({0: mode}))
            for p in pics:
                a = [sum(full[k][i] for k in p["nals"]) for i in range(3)]
                b = [sum(part[k][i] for k in p["nals"]) for i in range(3)]
                off = (mode == NONE or not p["ref"]) and "--deblock 1" not in _by_name(name)[3]   # --deblock 1: nothing to leave out
                assert b == [a[0] - 1 if off else a[0], a[1], a[2]], (name, TWIN[mode], p["nals"], a, b)


def _bench_decode(data, mode):
    """The benchmark's application loop (tools/libe264bench.so: 8 application threads, 2 parse-ahead workers per decoder,
    records kept) with E264_BENCH_LOOP_FILTER=mode; returns (frames, checksums, decoders, library)."""
    bench = ctypes.CDLL(os.path.join(ROOT, "tools", "libe264bench.so"))
    bench.e264bench_run.restype = ctypes.c_double
    bench.e264bench_run.argtypes = [ctypes.POINTER(ctypes.c_char_p), ctypes.POINTER(ctypes.c_size_t), ctypes.c_int, ctypes.c_int,
                                    ctypes.c_int, ctypes.POINTER(ctypes.c_long), ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_void_p)]
    N = len(data)
    saved = {k: os.environ.get(k) for k in ("E264B_KEEP", "E264_BENCH_DEC_THREADS", "E264_BENCH_LOOP_FILTER")}
    try:
        os.environ["E264B_KEEP"] = "1"; os.environ["E264_BENCH_DEC_THREADS"] = "2"; os.environ["E264_BENCH_LOOP_FILTER"] = str(mode)
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
def test_replay_equals_the_live_decode(workdir):
    """8 streams of the benchmark's 1080p workload through the benchmark's loop in each mode: the checksums equal the
    device's decode of the twins (REF, NONE) and of the streams (ALL); a kernel-only replay leaves every frame slot as the
    live decode did; the REF and NONE decoders launch fewer kernels than the ALL ones, with the same copies."""
    from bench import CONFIGS, ReplayStats
    from test_in_flight import _core, _stream_sum
    cfg = CONFIGS["1080p"]
    N, F = 8, 8
    streams = [("bench_%d" % (cfg["seed0"] + i), cfg["w"], cfg["h"], "-n %d -s %d %s" % (F, cfg["seed0"] + i, cfg["gen"])) for i in range(N)]
    lib = pkg.load()
    core = _core()
    core.e264b_replay.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ReplayStats)]
    stats = {}
    for mode in (ALL, REF, NONE):
        data = [_data(workdir, s) for s in streams]
        want = [_stream_sum(pkg.decode_bytes(_data(workdir, s, mode), lib)[0]) for s in streams]
        frames, sums, decs, bench = _bench_decode(data, mode)
        assert frames == [F] * N and sums == want, TWIN.get(mode, "all")
        devs = [core.e264b_of_decoder(d) for d in decs]
        tot = [0, 0, 0]
        for d in devs:
            v = [ctypes.c_uint64() for _ in range(3)]
            core.e264b_stats(d, *[ctypes.byref(x) for x in v])
            tot = [a + b.value for a, b in zip(tot, v)]
        stats[mode] = tot
        hashes = [[core.e264b_slot_hash(d, s) for s in range(core.e264b_slot_count(d))] for d in devs]
        arr = (ctypes.c_void_p * N)(*devs)
        st = ReplayStats()
        assert core.e264b_replay(arr, N, 2, 1, ctypes.byref(st)) == 0
        assert [core.e264b_error_flag(d) for d in devs] == [0] * N
        assert [[core.e264b_slot_hash(d, s) for s in range(core.e264b_slot_count(d))] for d in devs] == hashes
        assert st.launches == tot[0] * 2
        bench.e264bench_free.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int]
        bench.e264bench_free(decs, N)
    print("launches, H2D, D2H bytes per picture (all / ref / none):", [[v / (N * F) for v in stats[m]] for m in (ALL, REF, NONE)])
    assert stats[NONE][0] < stats[REF][0] < stats[ALL][0]
    assert stats[ALL][1:] == stats[REF][1:] == stats[NONE][1:]
