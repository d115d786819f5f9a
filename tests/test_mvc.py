"""Stereo (MVC) streams (include/edge264_mvc.h): both views decoded, paired in Edge264Frame.samples_mvc.

The oracle is the compiled reference decoder, which decodes both views bit-exactly: tests/golden/mvc.json holds what it
outputs on every stream here (frames of both views, FrameId and FrameId_mvc, the return code of every NAL unit) and in
the API cases below (tests/make_mvc_golden.py records it).  CPU tests run the product's host sources over the plain-C
restatement (oracle/liboracle_dec.so, and the restatement with every optional output); the GPU tests compare the device
with them and with the goldens."""
import ctypes, errno, functools, hashlib, json, os, subprocess
import numpy as np
import pytest
from conftest import ROOT, make_stream
from checkers import load, port_outputs_lib, Edge264Frame, _frame_bytes
from api_helpers import lib_of
from test_mb_errors import _nals
import edge264_b200 as pkg

GOLDEN = os.path.join(ROOT, "tests", "golden")
STORED = ["supp-nals.264", "nal-ref-idc-0.264"]   # the reference's own stereo streams (tests/golden/reference_streams/)

# (name, width_mbs, height_mbs, generator arguments): tools/gen264 --mvc, second views of every kind the options reach
MVC_STREAMS = [
    ("mvc_i_cabac",        6, 4, "-n 6 -s 2001 --gop I --deblock 0 --t8x8 50 --mvc 1"),
    ("mvc_ip_cavlc",       7, 5, "-n 12 -s 2002 --gop IP --refs 2 --cavlc --deblock 2 --mvc 2"),
    ("mvc_ipb",            9, 7, "-n 14 -s 2003 --gop IPB --deblock 0 --t8x8 50 --mvc 3"),
    ("mvc_dpb_refs4",      5, 4, "-n 40 -s 2004 --gop IP --refs 4 --dpb --idr 17 --deblock 0 --wp 1 --mvc 4"),
    ("mvc_dpb_ipb",        5, 4, "-n 40 -s 2005 --gop IPB --refs 4 --dpb --idr 23 --wp 2 --mvc 5"),
    ("mvc_temporal",       8, 6, "-n 24 -s 2006 --gop IPB --refs 3 --temporal --wp 2 --idr 13 --deblock 0 --mvc 6"),
    ("mvc_scaling_slices", 9, 7, "-n 12 -s 2007 --gop IPB --t8x8 60 --scaling 3 --slices 4 --wp 1 --mvc 7"),
    ("mvc_crop_bref",      6, 5, "-n 20 -s 2008 --gop IPB --i-period 5 --bref --refs 3 --crop-left 4 --crop-bottom 6 --deblock 2 --mvc 8"),
    ("mvc_nonref_cavlc",   6, 5, "-n 20 -s 2009 --gop IP --nonref-p --extra-nals --ps-update --cavlc --mvc 9"),
    ("mvc_ipb_cavlc",      7, 6, "-n 16 -s 2011 --gop IPB --refs 2 --cavlc --slices 2 --deblock 0 --wp 2 --temporal --mvc 11"),
]
# 1920x1088 (cropped to 1080): decoded on the GPU only
MVC_1080P = ("mvc_1080p_ipb", 120, 68, "-n 8 -s 2010 --gop IPB --refs 2 --t8x8 50 --density 40 --mvc 10")


@functools.lru_cache(None)
def gold():
    """Read on first use, so that tests/make_mvc_golden.py can import this module without the file."""
    return json.load(open(os.path.join(GOLDEN, "mvc.json")))


def _md5(b):
    return hashlib.md5(b).hexdigest()


def stream(workdir, s):
    return open(make_stream(workdir, *s), "rb").read()


def stored(name):
    return open(os.path.join(GOLDEN, "reference_streams", name), "rb").read()


def strip_mvc(data):
    """The stream without its prefix NAL units, subset SPSs and second-view slices (NAL unit types 14, 15, 20)."""
    return b"".join(b"\x00\x00\x00\x01" + data[a:b] for a, b in _nals(data) if data[a] & 31 not in (14, 15, 20))


def summary(frames):
    """decode_bytes(second_view=True) frames as [FrameId, md5, FrameId_mvc, md5_mvc] (the last two None for a mono frame)."""
    return [[f[0], _md5(f[3])] + ([f[-1][0], _md5(f[-1][3])] if f[-1] else [None, None]) for f in frames]


def decode(data, backend="port", n_threads=0, **kw):
    lib = None if backend == "gpu" else lib_of(backend) if backend == "outputs" else load(backend)
    frames, codes = pkg.decode_bytes(data, lib, n_threads, second_view=True, **kw)
    return frames, codes


def pair_bytes(f):
    return [_frame_bytes(f), _frame_bytes(f, True) if f.samples_mvc[0] else None]


def observe(data, backend, hold=0, flush_at=None):
    """The README loop over the C API with every frame borrowed and handed back `hold` frames later (at once when the
    decoder answers ENOBUFS without output), and edge264_flush after NAL unit `flush_at`.  Returns per decode_NAL call
    [return code, frames output after it] and per frame [FrameId, md5, FrameId_mvc, md5_mvc]; a borrowed pair must stay
    unchanged until it is returned."""
    lib = load(backend)
    buf = ctypes.create_string_buffer(data, len(data) + 64)
    base = ctypes.addressof(buf); end = base + len(data)
    dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
    assert dec
    nal = base + 3 + (1 if data[2] == 0 else 0)
    held, out, calls, f, n_nal, drained = [], [], [], Edge264Frame(), 0, False

    def give_back():
        fr, snap = held.pop(0)
        assert pair_bytes(fr) == snap, "a borrowed pair changed while it was held"
        out.append([fr.FrameId, _md5(snap[0]), fr.FrameId_mvc if snap[1] else None, snap[1] and _md5(snap[1])])
        lib.edge264_return_frame(dec, fr.return_arg)
    while True:
        sc = lib.edge264_find_start_code(nal, end, 0) if nal < end else end
        res = lib.edge264_decode_NAL(dec, nal, sc, None, None)
        drained |= nal >= end
        got = 0
        while lib.edge264_get_frame(dec, ctypes.byref(f), 1) == 0:
            fr = Edge264Frame.from_buffer_copy(bytes(f))
            held.append((fr, pair_bytes(fr)))
            got += 1
            while len(held) > hold:
                give_back()
        calls.append([res, got])
        if res == errno.ENOBUFS:
            if not got:
                if not held:
                    break
                give_back()
            continue
        n_nal += 1
        if flush_at is not None and n_nal == flush_at:
            while held:
                give_back()
            lib.edge264_flush(dec)
        nal = sc + 3 if sc + 3 < end else end
        if res not in (0, errno.ENOTSUP, errno.EBADMSG) or drained:
            break
    while held:
        give_back()
    d = ctypes.c_void_p(dec)
    lib.edge264_free(ctypes.byref(d))
    return {"calls": calls, "frames": out}


def _bits_ue(v):
    v += 1
    return "0" * (v.bit_length() - 1) + format(v, "b")


def subset_sps(w, h, num_views=2, max_num_ref_frames=2):
    """A subset SPS NAL unit (Stereo High, level 4.0, frame_num and POC lsb of 8 and 10 bits as tools/gen264 writes them
    without --dpb) for w x h macroblocks with `num_views` views, view i predicting from view 0."""
    b = format(128, "08b") + "00000000" + format(40, "08b") + _bits_ue(0)
    b += _bits_ue(1) + _bits_ue(0) + _bits_ue(0) + "0" + "0"                       # 4:2:0, 8 bits, no bypass, no matrices
    b += _bits_ue(4) + _bits_ue(0) + _bits_ue(6)                                  # log2_max_frame_num 8, POC type 0, lsb 10 bits
    b += _bits_ue(max_num_ref_frames) + "0" + _bits_ue(w - 1) + _bits_ue(h - 1) + "1" + "1" + "0" + "0"
    b += "1" + _bits_ue(num_views - 1) + "".join(_bits_ue(i) for i in range(num_views))
    b += "".join(_bits_ue(1) + _bits_ue(0) + _bits_ue(0) for _ in range(1, num_views))
    b += "".join(_bits_ue(1) + _bits_ue(0) + _bits_ue(0) for _ in range(1, num_views))
    b += _bits_ue(0) + format(40, "08b") + _bits_ue(0) + "000" + _bits_ue(num_views - 1) + "".join(_bits_ue(i) for i in range(num_views)) + _bits_ue(num_views - 1)
    b += "0" + "0" + "1"
    b += "0" * (-len(b) % 8)
    rbsp = bytes(int(b[i:i + 8], 2) for i in range(0, len(b), 8))
    esc, zeros = bytearray(), 0
    for x in rbsp:
        if zeros >= 2 and x <= 3:
            esc.append(3); zeros = 0
        esc.append(x); zeros = zeros + 1 if x == 0 else 0
    return b"\x00\x00\x00\x01\x6f" + bytes(esc)


def replace_subset_sps(data, nal):
    """The stream with every subset SPS replaced by `nal`."""
    starts = [s - 3 for s, _ in _nals(data)] + [len(data)]
    return b"".join(nal if data[a + 3] & 31 == 15 else data[a:b] for a, b in zip(starts, starts[1:]))


def api_cases(workdir):
    """name -> stream of the API observations: a stereo stream with End of sequence then a single-view stream after it,
    and a stream whose subset SPS lists 3 views."""
    by = {s[0]: s for s in MVC_STREAMS}
    ipb = stream(workdir, by["mvc_ipb"])
    mono = open(make_stream(workdir, "mvc_eos_mono", 9, 7, "-n 6 -s 2012 --gop IPB --deblock 0"), "rb").read()
    ip = stream(workdir, by["mvc_ip_cavlc"])
    return {"eos_to_mono": ipb + b"\x00\x00\x00\x01\x0a" + mono,
            "three_views": replace_subset_sps(ip, subset_sps(7, 5, num_views=3))}


HOLDS = (0, 1, 3)
FLUSH_AT = (9, 20)


# ---- CPU: the reference's stored stereo streams ----
@pytest.mark.parametrize("name", STORED)
@pytest.mark.parametrize("threads", [0, 1, 3])
def test_stored_stereo_streams(name, threads):
    """Both views, FrameId, FrameId_mvc and every return code equal the reference's."""
    frames, codes = decode(stored(name), "port", threads)
    g = gold()["stored"][name]
    assert summary(frames) == g["frames"] and codes == g["codes"]
    assert [f[0] for f in frames][:2] in ([0, 2], [0])   # base views take FrameIds 0 and 2 now: the second view numbers in between


# ---- CPU: generated stereo streams ----
@pytest.mark.parametrize("threads", [0, 1, 3])
@pytest.mark.parametrize("s", MVC_STREAMS, ids=[s[0] for s in MVC_STREAMS])
def test_generated_stereo_streams(workdir, s, threads):
    data = stream(workdir, s)
    g = gold()["streams"][s[0]]
    assert g["args"] == "-W %d -H %d %s" % s[1:] and g["stream_md5"] == _md5(data), "tools/gen264 no longer writes the stream of the golden"
    frames, codes = decode(data, "port", threads)
    assert summary(frames) == g["frames"] and codes == g["codes"]
    assert all(f[-1] for f in frames) and len(frames) == int(s[3].split()[1])


@pytest.mark.parametrize("s", MVC_STREAMS, ids=[s[0] for s in MVC_STREAMS])
def test_base_view_is_the_stream_without_its_second_view(workdir, s):
    """Stereo decoding changes nothing in the base view: its frames are those of the stream with NAL units 14, 15 and 20
    removed (tools/gen264 --mvc writes the base view's NAL units of the same stream without --mvc)."""
    data = stream(workdir, s)
    frames, _ = decode(data)
    mono, _ = decode(strip_mvc(data))
    assert [f[3] for f in frames] == [f[3] for f in mono] and all(f[-1] is None for f in mono)
    plain = open(make_stream(workdir, s[0] + "_plain", s[1], s[2], s[3].split(" --mvc")[0]), "rb").read()
    nal_units = lambda d: [d[a:b] for a, b in _nals(d)]
    assert nal_units(strip_mvc(data)) == nal_units(plain)


def test_stored_streams_base_view_against_stripped():
    for name in STORED:
        frames, _ = decode(stored(name))
        mono, _ = decode(strip_mvc(stored(name)))
        assert [f[3] for f in frames] == [f[3] for f in mono]


# ---- CPU: the API against the reference's observations ----
def test_borrowing_and_returning_pairs(workdir):
    """Pairs borrowed and handed back 0, 1 or 3 frames later: every decode_NAL return code, ENOBUFS included (when the
    decoder waits for held pairs and at the end of the stream), the pairs each call lets out, and the pairs themselves."""
    by = {s[0]: s for s in MVC_STREAMS}
    assert [c[0] for c in gold()["api"]["borrowed"]["mvc_ipb/3"]["calls"]].count(errno.ENOBUFS) > 0
    for name in ("mvc_ipb", "mvc_dpb_ipb"):
        data = stream(workdir, by[name])
        for hold in HOLDS:
            assert observe(data, "port", hold) == gold()["api"]["borrowed"]["%s/%d" % (name, hold)], (name, hold)


def test_flush_mid_stream(workdir):
    data = stream(workdir, MVC_STREAMS[2])
    for at in FLUSH_AT:
        assert observe(data, "port", 1, flush_at=at) == gold()["api"]["flush"][str(at)], at


def test_end_of_sequence_and_three_views(workdir):
    """End of sequence turns stereo off: the frames after it are single view.  A subset SPS with 3 views answers ENOTSUP
    and the stream is decoded as its base view alone."""
    cases = api_cases(workdir)
    for name, data in cases.items():
        assert observe(data, "port") == gold()["api"][name], name
    eos = observe(cases["eos_to_mono"], "port")["frames"]
    assert eos[0][2] is not None and eos[-1][2] is None
    three = decode(cases["three_views"])
    assert errno.ENOTSUP in three[1] and all(f[-1] is None for f in three[0])
    assert [f[3] for f in three[0]] == [f[3] for f in decode(strip_mvc(cases["three_views"]))[0]]


def test_subset_sps_beyond_32_frame_slots(workdir):
    """max_num_ref_frames 16 in the subset SPS: the two views do not fit in 32 frame slots, the subset SPS answers ENOTSUP
    and the stream decodes as its base view alone."""
    data = replace_subset_sps(stream(workdir, MVC_STREAMS[1]), subset_sps(7, 5, max_num_ref_frames=16))
    frames, codes = decode(data)
    assert codes[[data[a] & 31 for a, _ in _nals(data)].index(15)] == errno.ENOTSUP
    assert all(f[-1] is None for f in frames) and [f[3] for f in frames] == [f[3] for f in decode(strip_mvc(data))[0]]
    ok = replace_subset_sps(stream(workdir, MVC_STREAMS[1]), subset_sps(7, 5, max_num_ref_frames=15))
    assert all(f[-1] for f in decode(ok)[0])


# ---- CPU: modes ----
def _with_second_views(frames):
    return [(f[0], f[3], f[-1][0], f[-1][3]) for f in frames]


@pytest.mark.parametrize("s", [MVC_STREAMS[i] for i in (2, 4, 7, 8)], ids=[MVC_STREAMS[i][0] for i in (2, 4, 7, 8)])
def test_luma_only_both_views(workdir, s):
    data = stream(workdir, s)
    full, codes = decode(data)
    luma, lcodes = decode(data, luma_only=True)
    assert lcodes == codes and len(luma) == len(full)
    for a, b in zip(full, luma):
        for x, y in ((a, b), (a[-1], b[-1])):
            n = x[1] * x[2]
            assert x[0] == y[0] and x[3][:n] == y[3][:n] and set(y[3][n:]) == {128}


@pytest.mark.parametrize("mode,twin", [(pkg.LOOP_FILTER_REF, "nonref"), (pkg.LOOP_FILTER_NONE, "all")])
@pytest.mark.parametrize("s", [MVC_STREAMS[i] for i in (2, 5, 8)], ids=[MVC_STREAMS[i][0] for i in (2, 5, 8)])
def test_loop_filter_modes(workdir, s, mode, twin):
    """A decode without the loop filter of the non-reference view components (a base view with inter_view_flag 1 counts
    as a reference) or of all of them equals the full decode of the twin stream with disable_deblocking_filter_idc 1 in
    those slices; the reference decodes the twins to the same frames (golden).  REF leaves every reference unchanged."""
    name, w, h, args = s
    data = stream(workdir, s)
    tw = open(make_stream(workdir, name + "_off_" + twin, w, h, args + " --deblock-off " + twin), "rb").read()
    got = decode(data, loop_filter=mode)
    assert _with_second_views(got[0]) == _with_second_views(decode(tw)[0]) and got[1] == decode(tw)[1]
    assert summary(decode(tw)[0]) == gold()["twins"][name + "/" + twin]


def _au_kept(data, mode):
    """Per access unit of a gen264 --mvc stream, in decoding order: whether the skip mode keeps it (decided at its base
    view: NONREF keeps a reference or inter-view reference, NONKEY an IDR or I picture)."""
    from test_mb_errors import _slice_head
    keep, prefix = [], None
    for s, e in _nals(data):
        t = data[s] & 31
        if t == 14:
            prefix = data[s + 3]
        if t in (1, 5):
            ref, typ, first, st = _slice_head(data[s:e])
            if first == 0:
                keep.append(ref > 0 or prefix >> 1 & 1 if mode == pkg.SKIP_NONREF else typ == 5 or st == 2)
    return keep


@pytest.mark.parametrize("mode", [pkg.SKIP_NONREF, pkg.SKIP_NONKEY])
@pytest.mark.parametrize("s", [MVC_STREAMS[i] for i in (2, 7, 8)], ids=[MVC_STREAMS[i][0] for i in (2, 7, 8)])
def test_skip_modes_pairs(workdir, s, mode):
    """A skip mode outputs the full decode's pairs less those of the skipped access units, in order; the second view of a
    kept access unit is never skipped."""
    data = stream(workdir, s)
    full = _with_second_views(decode(data)[0])
    part = _with_second_views(decode(data, skip=mode)[0])
    it = iter(full)
    assert all(any(p == f for f in it) for p in part), "not an in-order subset of the full decode"
    assert 0 < len(part) <= len(full)
    if mode == pkg.SKIP_NONKEY:
        assert len(part) == sum(_au_kept(data, mode))


# ---- CPU: edge264_get_second_view and the optional outputs ----
def test_second_view_api(workdir):
    lib = port_outputs_lib()
    data = stream(workdir, MVC_STREAMS[2])
    buf = ctypes.create_string_buffer(data, len(data) + 64)
    dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
    from api_helpers import first_frame, free_decoder
    f, out = first_frame(lib, dec, data, buf), Edge264Frame()
    assert lib.edge264_get_second_view(dec, ctypes.byref(f), ctypes.byref(out)) == 0
    assert out.FrameId == f.FrameId_mvc and not out.samples_mvc[0] and _frame_bytes(out) == _frame_bytes(f, True)
    mono = Edge264Frame.from_buffer_copy(bytes(f)); mono.return_arg = ctypes.c_void_p(f.return_arg & 255)
    assert lib.edge264_get_second_view(dec, ctypes.byref(mono), ctypes.byref(out)) == errno.ENOENT
    lib.edge264_return_frame(dec, f.return_arg)
    assert lib.edge264_get_second_view(dec, ctypes.byref(f), ctypes.byref(out)) == errno.EINVAL
    assert lib.edge264_get_second_view(dec, None, ctypes.byref(out)) == errno.EINVAL
    free_decoder(lib, dec)
    plain = open(make_stream(workdir, "mvc_api_plain", 6, 4, "-n 3 -s 2013 --gop I"), "rb").read()
    assert all(f[-1] is None for f in decode(plain, "outputs")[0])


def _area(a, tw, th):
    ov = lambda s, t: np.maximum(0, np.minimum((np.arange(t)[:, None] + 1) * s, (np.arange(s)[None, :] + 1) * t)
                                 - np.maximum(np.arange(t)[:, None] * s, np.arange(s)[None, :] * t)).astype(np.int64)
    n, d = ov(a.shape[0], th) @ a.astype(np.int64) @ ov(a.shape[1], tw).T, a.size
    return ((2 * n + d) // (2 * d)).astype(np.uint8)


def check_outputs(frames, resized_to):
    """Second views of decode_bytes(errors, motion, resized, picstats, second_view) against numpy over their samples."""
    n = 0
    for fr in frames:
        sv = fr[-1]
        _, w, h, i420, _, _, p, st = sv
        raw = np.frombuffer(i420, np.uint8)
        planes = [raw[:w * h].reshape(h, w)] + [raw[w * h + i * (w * h // 4):][:w * h // 4].reshape(h // 2, w // 2) for i in (0, 1)]
        tw, th = resized_to
        assert np.array_equal(p["y"], _area(planes[0], tw, th)) and np.array_equal(p["cbcr"], np.stack([_area(c, tw // 2, th // 2) for c in planes[1:]], axis=2))
        for k, (P, m) in enumerate(zip(planes, (16, 8, 8))):
            assert np.array_equal(st["hist"][k], np.bincount(P.ravel(), minlength=256))
            if P.shape[0] % m == 0 and P.shape[1] % m == 0:
                v = P.astype(np.uint32).reshape(P.shape[0] // m, m, P.shape[1] // m, m)
                assert np.array_equal(st["sum"][k], v.sum(axis=(1, 3))) and np.array_equal(st["sum_sq"][k], (v * v).sum(axis=(1, 3)))
        n += 1
    return n


OUTPUTS = dict(errors=True, motion=True, resized=(pkg.PACKED_NV12, 40, 26), picstats=True)


def test_second_view_outputs(workdir):
    """The second view's resized output and statistics equal numpy over samples_mvc, and its motion export names the base
    view's FrameId for inter-view blocks: every reference FrameId of a second view is one of its own view or the base
    view of its access unit."""
    for s in (MVC_STREAMS[2], MVC_STREAMS[5]):
        frames, _ = decode(stream(workdir, s), "outputs", **OUTPUTS)
        assert check_outputs(frames, (40, 26)) == len(frames)
        second_ids = {f[-1][0] for f in frames}
        inter_view = 0
        for f in frames:
            m = f[-1][5]
            ids = set(np.unique(m["ref_frame_id"])) - {-1}
            assert ids <= second_ids | {f[0]}, (f[0], ids)
            inter_view += int((m["ref_frame_id"] == f[0]).sum())
            assert f[0] not in set(np.unique(f[5]["ref_frame_id"]))   # the base view never predicts from itself
        assert inter_view > 0


def test_second_view_motion_rebuilds_inter_view_blocks(workdir):
    """Anchor second views predict from the base view only: every inter block of theirs names the base FrameId."""
    frames, _ = decode(stream(workdir, MVC_STREAMS[0]), "outputs", motion=True)
    for f in frames:
        m = f[-1][4]
        inter = m["ref_frame_id"][0][m["ref_frame_id"][0] >= 0]
        assert inter.size and set(np.unique(inter)) == {f[0]}


def test_damaged_stereo_error_maps(workdir):
    """A truncated second-view slice marks its own view; a lost base slice marks the base view and, through inter-view
    prediction, the second view of its access unit."""
    data = stream(workdir, MVC_STREAMS[2])
    nals = _nals(data)
    sv = [k for k, (s, e) in enumerate(nals) if data[s] & 31 == 20]
    base = [k for k, (s, e) in enumerate(nals) if data[s] & 31 in (1, 5)]
    def without(k, cut=False):
        s, e = nals[k]
        return data[:s + (e - s) // 2] + data[e:] if cut else data[:s - 3] + data[e:]
    # a truncated NAL unit 20 of the third access unit
    frames, _ = decode(without(sv[2], cut=True), "outputs", errors=True)
    assert any(f[-1][4] for f in frames) and all(not f[4] for f in frames[:1])
    # the base slice of the second access unit lost: its second view predicts from a concealed picture
    frames, _ = decode(without(base[1]), "outputs", errors=True)
    hit = [f for f in frames if f[4]]
    assert hit and any(f[-1][4] and max(f[-1][4]) > 0 for f in hit)


def test_record_contract_on_second_view_slices(workdir):
    from test_record_fuzz import _check_records
    for s in MVC_STREAMS:
        for t in (0, 3):
            code, why = _check_records(make_stream(workdir, *s), t)
            assert code == 0, (s[0], t, why)


# ---- GPU ----
@pytest.mark.gpu
@pytest.mark.parametrize("threads", [0, 3])
def test_device_equals_restatement(workdir, threads):
    """Both views and every optional output of the second view, on the device and on the restatement."""
    inputs = [(s[0], stream(workdir, s)) for s in MVC_STREAMS] + [(n, stored(n)) for n in STORED]
    for name, data in inputs:
        g, gc = decode(data, "gpu", threads, **OUTPUTS)
        p, pc = decode(data, "outputs", threads, **OUTPUTS)
        assert gc == pc and len(g) == len(p), name
        for a, b in zip(g, p):
            for x, y in ((a, b), (a[-1], b[-1])) if b[-1] else ((a, b),):
                assert x[:5] == y[:5], (name, x[0])
                for k in y[5]:
                    assert np.array_equal(x[5][k], y[5][k]), (name, x[0], k)
                assert all(np.array_equal(x[6][k], y[6][k]) for k in ("y", "cbcr")) and all(np.array_equal(x[7][k], y[7][k]) for k in ("hist", "sum", "sum_sq"))


@pytest.mark.gpu
def test_device_equals_goldens(workdir):
    for s in MVC_STREAMS + [MVC_1080P]:
        frames, codes = decode(stream(workdir, s), "gpu")
        g = gold()["streams"][s[0]]
        assert summary(frames) == g["frames"] and codes == g["codes"], s[0]
    for n in STORED:
        frames, codes = decode(stored(n), "gpu")
        assert summary(frames) == gold()["stored"][n]["frames"]


@pytest.mark.gpu
def test_device_modes(workdir):
    for s in (MVC_STREAMS[2], MVC_STREAMS[8]):
        data = stream(workdir, s)
        for kw in (dict(luma_only=True), dict(loop_filter=pkg.LOOP_FILTER_REF), dict(skip=pkg.SKIP_NONREF), dict(skip=pkg.SKIP_NONKEY)):
            assert decode(data, "gpu", 0, **kw) == decode(data, "port", 0, **kw), (s[0], kw)


_DEVICE_SUB = r"""
import sys, os, ctypes, json, hashlib
sys.path.insert(0, os.path.join(sys.argv[1], "tests")); sys.path.insert(0, sys.argv[1])
import torch, edge264_b200 as pkg
from api_helpers import new_decoder, free_decoder, loop, _cudart, _ALLOC, _FREE
data = open(sys.argv[2], "rb").read()
def grab(f, mvc):
    out = bytearray()
    for pl in range(3):
        w = f.width_C if pl else f.width_Y; h = f.height_C if pl else f.height_Y; st = f.stride_C if pl else f.stride_Y
        p = ctypes.cast((f.samples_mvc if mvc else f.samples)[pl], ctypes.c_void_p).value
        t = torch.as_tensor(pkg._DeviceBytes(p, st * (h - 1) + w), device="cuda").cpu().numpy()
        for y in range(h): out += bytes(t[y * st:y * st + w])
    return hashlib.md5(bytes(out)).hexdigest()
lib, res, cbs = pkg.load(), [], (None, None)
if sys.argv[3] == "alloc_cb":   # device memory from the application's allocator
    rt = _cudart()
    rt.cudaMalloc.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_size_t]; rt.cudaFree.argtypes = [ctypes.c_void_p]
    def alloc(samples, size, mbs, mbs_size, err, arg):
        p = ctypes.c_void_p(); rt.cudaMalloc(ctypes.byref(p), size + 64); samples[0] = p.value
    def release(samples, mbs, arg):
        rt.cudaFree(samples)
    cbs = (_ALLOC(alloc), _FREE(release))
dec = new_decoder(lib, alloc=cbs)
loop(lib, dec, data, lambda f: res.append([f.FrameId, grab(f, 0), f.FrameId_mvc, grab(f, 1)]))
free_decoder(lib, dec)
print(json.dumps(res))
"""


@pytest.mark.gpu
def test_device_memory_frames(workdir):
    """E264B_OUTPUT=device, and a device alloc_cb: both views of every pair are correct in device memory."""
    import sys
    for s in (MVC_STREAMS[2], MVC_STREAMS[7]):
        for how, env in (("output_device", dict(os.environ, E264B_OUTPUT="device")), ("alloc_cb", dict(os.environ))):
            r = subprocess.run([sys.executable, "-c", _DEVICE_SUB, ROOT, make_stream(workdir, *s), how], capture_output=True, text=True, env=env, timeout=600)
            assert r.returncode == 0, r.stderr[-2000:]
            assert json.loads(r.stdout.strip().splitlines()[-1]) == gold()["streams"][s[0]]["frames"], (s[0], how)


@pytest.mark.gpu
def test_decoders_in_flight_mixing_stereo_and_mono(workdir):
    """8 decoders at once, stereo and single-view streams, 0 to 2 workers each: every output equals the restatement's."""
    from concurrent.futures import ThreadPoolExecutor
    mono = open(make_stream(workdir, "mvc_eos_mono", 9, 7, "-n 6 -s 2012 --gop IPB --deblock 0"), "rb").read()
    jobs = [stream(workdir, s) for s in MVC_STREAMS[:4]] + [mono, mono, stored("supp-nals.264"), stored("nal-ref-idc-0.264")]
    want = [summary(decode(d)[0]) for d in jobs]
    for r in range(2):
        with ThreadPoolExecutor(8) as ex:
            got = list(ex.map(lambda ij: summary(decode(ij[1], "gpu", (ij[0] + r) % 3)[0]), enumerate(jobs)))
        assert got == want


@pytest.mark.gpu
def test_access_unit_costs_its_two_pictures(workdir):
    """Launches and copies (e264b_stats) per NAL unit, synchronous decoding: the base view's NAL units cost what they cost
    in the stream without its second view, prefix NAL units and subset SPSs cost nothing, and each second-view picture
    copies back what its base view picture does (one frame, no error map on these clean streams)."""
    from test_skip import stats_per_nal
    for s in (MVC_STREAMS[0], MVC_STREAMS[2], MVC_STREAMS[4]):
        data = stream(workdir, s)
        st, _ = stats_per_nal(data, pkg.SKIP_NONE)
        mono, _ = stats_per_nal(strip_mvc(data), pkg.SKIP_NONE)
        types = [data[a] & 31 for a, _ in _nals(data)]
        assert len(st) == len(types) + 1 and len(mono) == len(types) - types.count(14) - types.count(15) - types.count(20) + 1   # the last call: end of stream
        assert [c for c, t in zip(st, types) if t not in (14, 15, 20)] + st[-1:] == mono, s[0]
        assert all(c == (0, 0, 0) for c, t in zip(st, types) if t in (14, 15))
        base = [c for c, t in zip(st, types) if t in (1, 5) and c[0]]
        second = [c for c, t in zip(st, types) if t == 20 and c[0]]
        assert len(second) == len(base) == int(s[3].split()[1]), s[0]
        assert all(b[2] == c[2] for b, c in zip(base, second)) and sum(c[0] for c in st) == sum(c[0] for c in mono) + sum(c[0] for c in second)


@pytest.mark.gpu
def test_replay_of_stereo_stream_equals_live_decode(workdir, monkeypatch):
    """The kernel-only replay of a stereo stream's pictures leaves every frame slot as the live decode did."""
    from test_in_flight import _core
    from bench import ReplayStats
    from api_helpers import new_decoder, free_decoder, loop
    monkeypatch.setenv("E264B_KEEP", "1")
    lib, core = pkg.load(), _core()
    core.e264b_replay.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ReplayStats)]
    for s in (MVC_STREAMS[2], MVC_STREAMS[5]):
        data = stream(workdir, s)
        dec = new_decoder(lib, n_threads=2)
        frames = []
        loop(lib, dec, data, lambda f: frames.append((_frame_bytes(f), _frame_bytes(f, True))))
        ctx = core.e264b_of_decoder(dec)
        assert core.e264b_kept_count(ctx) == 2 * len(frames) == 2 * int(s[3].split()[1])
        hashes = [core.e264b_slot_hash(ctx, k) for k in range(core.e264b_slot_count(ctx))]
        st = ReplayStats()
        assert core.e264b_replay((ctypes.c_void_p * 1)(ctx), 1, 2, 1, ctypes.byref(st)) == 0 and core.e264b_error_flag(ctx) == 0
        assert [core.e264b_slot_hash(ctx, k) for k in range(core.e264b_slot_count(ctx))] == hashes, s[0]
        assert [(_md5(a), _md5(b)) for a, b in frames] == [(f[1], f[3]) for f in gold()["streams"][s[0]]["frames"]]
        free_decoder(lib, dec)
