"""Skipped pictures (include/edge264_skip.h): EDGE264_SKIP_NONREF leaves out every picture with nal_ref_idc 0,
EDGE264_SKIP_NONKEY every picture that is neither IDR nor begun by an I slice.  Their headers run, so the decoded picture
buffer evolves as in a full decode; their slice data is never parsed and they cost the device nothing.  The oracle is the
decoder's own full decode (pinned to the reference decoder elsewhere, and here for the --i-period streams through
tests/golden/skip.json): a skip mode outputs the full decode's frames with the skipped pictures removed.

CPU tests run the product's host sources over the plain-C restatement with error maps and the motion export
(tests/native/port_outputs_backend.c, built by tests/checkers.py); the GPU tests compare the device with it."""
import ctypes, errno, functools, hashlib, json, os
import pytest
from conftest import ROOT, STREAMS, DPB_STREAMS, make_stream, md5_frames, have
from test_mb_errors import _nals, _slice_head
from api_helpers import lib_of, _damaged
from checkers import port_outputs_lib
import edge264_b200 as pkg
import checkers

NONE, NONREF, NONKEY = pkg.SKIP_NONE, pkg.SKIP_NONREF, pkg.SKIP_NONKEY

# open GOPs: a non-IDR I picture every few pictures, P and B pictures after it predicting across it
I_STREAMS = [
    ("iperiod_ipb",        6, 4, "-n 40 -s 1301 --gop IPB --i-period 6 --refs 3 --idr 40 --deblock 0 --wp 2 --temporal"),
    ("iperiod_ipb_cavlc",  5, 4, "-n 30 -s 1302 --gop IPB --i-period 7 --refs 2 --deblock 2 --slices 2 --cavlc --wp 1"),
    ("iperiod_bref",       4, 4, "-n 40 -s 1303 --gop IPB --i-period 8 --bref --refs 3 --idr 21 --deblock 0 --wp 2"),
    ("iperiod_ip",         5, 3, "-n 30 -s 1304 --gop IP --i-period 5 --refs 3 --nonref-p --deblock 0"),
]
ALL = STREAMS + DPB_STREAMS + I_STREAMS


@functools.lru_cache(None)
def gold():
    """Read on first use, so that tests/make_skip_golden.py can import the stream list without the file."""
    return json.load(open(os.path.join(ROOT, "tests", "golden", "skip.json")))


def pictures(data):
    """Decoding-order pictures of one of the generator's streams (a picture starts with the slice of first_mb_in_slice 0):
    per picture the indices of its NAL units, its nal_unit_type and nal_ref_idc, and the slice_type % 5 of its slices."""
    pics = []
    for k, (s, e) in enumerate(_nals(data)):
        if data[s] & 31 not in (1, 5):
            continue
        ref, typ, first, st = _slice_head(data[s:e])
        if first == 0:
            pics.append({"nals": [], "type": typ, "ref": ref, "slices": []})
        pics[-1]["nals"].append(k); pics[-1]["slices"].append(st)
    return pics


def kept(p, mode):
    return mode == NONE or (mode == NONREF and p["ref"] > 0) or (mode == NONKEY and (p["type"] == 5 or p["slices"][0] == 2))


def decode(data, backend="port", n_threads=0, skip=NONE, motion=False, before=None, after=None):
    """The README loop with a skip mode; before(k, lib, dec) / after(k, lib, dec) run around the decode_NAL of NAL unit k.
    Per frame (FrameId, i420 bytes, error map or None, motion export or None); per NAL unit its return code."""
    lib = lib_of(backend)
    buf = ctypes.create_string_buffer(data, len(data) + 64)
    base = ctypes.addressof(buf); end = base + len(data)
    dec = lib.edge264_alloc(n_threads, None, None, 0, None, None, None)
    assert dec
    if motion:
        assert lib.edge264_enable_motion(dec) == 0
    assert lib.edge264_set_skip(dec, skip) == 0
    nal, k = base + 3 + (1 if data[2] == 0 else 0), 0
    frames, codes, f = [], [], pkg.Edge264Frame()
    while True:
        sc = lib.edge264_find_start_code(nal, end, 0) if nal < end else end
        before and before(k, lib, dec)
        n0 = len(frames)
        res = lib.edge264_decode_NAL(dec, nal, sc, None, None)
        while lib.edge264_get_frame(dec, ctypes.byref(f), 0) == 0:
            frames.append((f.FrameId, pkg._frame_bytes(f), pkg._frame_errors(f), pkg.frame_motion(lib, dec, f) if motion else None))
        if res == errno.ENOBUFS:
            assert len(frames) > n0
            continue
        after and after(k, lib, dec)
        codes.append(res)
        if nal >= end:
            break
        nal = sc + 3 if sc + 3 < end else end
        k += 1
    d = ctypes.c_void_p(dec)
    lib.edge264_free(ctypes.byref(d))
    return frames, codes


def stream(workdir, name, w, h, args):
    return open(make_stream(workdir, name, w, h, args), "rb").read()


def check_subset(full, part, label, exact=True):
    """part is an in-order subsequence of full with the same FrameIds, samples and maps.  exact=False: a frame with an error
    map the full decode's frame lacks may predict from a filled skipped picture (rule 3); only its FrameId is checked."""
    by_id = {f[0]: f for f in full}
    ids = [f[0] for f in full]
    pos = [ids.index(f[0]) if f[0] in by_id else -1 for f in part]
    assert -1 not in pos and pos == sorted(pos) and len(set(pos)) == len(pos), (label, [f[0] for f in part])
    for f in part:
        g = by_id[f[0]]
        if not exact and f[2] is not None and g[2] is None:
            continue
        assert f[1] == g[1], "%s: frame %d differs from the full decode" % (label, f[0])
        assert f[2] == g[2], "%s: frame %d has another error map than in the full decode" % (label, f[0])


def intra_only(pics, frames, mode):
    """FrameIds of the output pictures whose slices are all I (FrameIds grow in decoding order)"""
    ids = sorted(f[0] for f in frames)
    chosen = [p for p in pics if kept(p, mode)]
    assert len(ids) == len(chosen)
    return {i for i, p in zip(ids, chosen) if all(st == 2 for st in p["slices"])}


# ---- 1. the output of a skip mode is the full decode without the skipped pictures ----
@pytest.mark.parametrize("name,w,h,args", ALL, ids=[s[0] for s in ALL])
def test_skip_output_is_a_subsequence_of_the_full_decode(workdir, name, w, h, args):
    data = stream(workdir, name, w, h, args)
    pics = pictures(data)
    full, fcodes = decode(data)
    assert len(full) == len(pics)
    for mode in (NONREF, NONKEY):
        for t in (0, 3):
            label = "%s mode %d, %d workers" % (name, mode, t)
            part, codes = decode(data, n_threads=t, skip=mode, motion=mode == NONKEY)
            assert len(part) == sum(kept(p, mode) for p in pics), label
            check_subset(full, part, label)
            if t == 0:
                assert codes == fcodes, label   # the skipped pictures' slices answer 0 like the decoded ones do
            if mode == NONKEY:
                intra = intra_only(pics, part, mode)
                for f in part:
                    if f[0] in intra:
                        assert (f[3]["mb_type"] < 4).all(), "%s: frame %d has inter macroblocks" % (label, f[0])


# ---- 2. the --i-period streams' full decode against the reference ----
@pytest.mark.parametrize("name,w,h,args", I_STREAMS, ids=[s[0] for s in I_STREAMS])
def test_i_period_streams_match_golden(workdir, name, w, h, args):
    g = gold()[name]
    assert g["args"] == f"-W {w} -H {h} {args}"
    data = stream(workdir, name, w, h, args)
    assert (len(data), hashlib.md5(data).hexdigest()) == (g["bytes"], g["stream_md5"])
    pics = pictures(data)
    assert sum(p["type"] == 1 and p["slices"][0] == 2 for p in pics) >= 2, "no non-IDR I picture"
    assert md5_frames(checkers.decode_bytes(data, "port")[0]) == g["md5"]
    if have("ref"):
        assert md5_frames(checkers.decode_bytes(data, "ref")[0]) == g["md5"]


def test_i_period_pictures_predict_across_the_i_picture(workdir):
    """open GOP: some P or B picture after a non-IDR I picture refers to a picture decoded before it"""
    name, w, h, args = I_STREAMS[0]
    data = stream(workdir, name, w, h, args)
    frames, _ = decode(data, motion=True)
    order = sorted(f[0] for f in frames)
    pics = pictures(data)
    i_ids = [order[k] for k, p in enumerate(pics) if p["type"] == 1 and p["slices"][0] == 2]
    across = 0
    for f in frames:
        last_i = max((i for i in i_ids if i < f[0]), default=None)
        if last_i is not None:
            refs = f[3]["ref_frame_id"]
            across += int(((refs >= 0) & (refs < last_i)).any())
    assert across > 0


# ---- 3. mode switches and skipped reference pictures that are predicted from ----
def switch_at(k_switch, mode):
    def before(k, lib, dec):
        if k == k_switch:
            assert lib.edge264_set_skip(dec, mode) == 0
    return before


def idr_switch_case(workdir):
    name, w, h, args = next(s for s in DPB_STREAMS if s[0] == "dpb_ipb_spatial")
    data = stream(workdir, name, w, h, args)
    idrs = [p for p in pictures(data) if p["type"] == 5]
    assert len(idrs) >= 2
    return data, idrs[1]["nals"][0]


def test_switch_to_full_decode_at_an_idr(workdir):
    data, k = idr_switch_case(workdir)
    full, _ = decode(data)
    part, _ = decode(data, skip=NONKEY, before=switch_at(k, NONE))
    check_subset(full, part, "NONKEY -> NONE")
    # every frame from the IDR on is output, as in the full decode
    idr_id = sorted(f[0] for f in full)[len([p for p in pictures(data) if p["nals"][0] < k])]
    after = [f[0] for f in full if f[0] >= idr_id]
    assert len(after) >= 5 and [f[0] for f in part if f[0] >= idr_id] == after
    assert len([f for f in part if f[0] < idr_id]) < len([f for f in full if f[0] < idr_id])


def rule3_cases(workdir):
    """(label, stream, mode, before hook): pictures that predict from a skipped reference picture"""
    out = []
    # a switch NONKEY -> NONE in the middle of an open GOP: the next P picture predicts from skipped P pictures
    name, w, h, args = I_STREAMS[0]
    data = stream(workdir, name, w, h, args)
    pics = pictures(data)
    k = next(p["nals"][0] for p in pics[3:] if p["type"] == 1 and p["slices"][0] == 0)
    out.append(("switch at a P picture", data, NONKEY, switch_at(k, NONE)))
    # NONREF -> NONKEY -> NONE on a stream with reference B pictures
    name, w, h, args = I_STREAMS[2]
    data = stream(workdir, name, w, h, args)
    pics = pictures(data)
    ks = [p["nals"][0] for p in pics if p["type"] == 1 and p["slices"][0] == 1]
    hooks = {ks[2]: NONKEY, ks[8]: NONE}
    out.append(("switches at B pictures", data, NONREF, lambda k, lib, dec: k in hooks and lib.edge264_set_skip(dec, hooks[k])))
    # mixed-slice pictures begun by an I slice: their P and B slices predict from skipped pictures
    for name, w, h, args in DPB_STREAMS:
        if name.startswith("mixed_slices"):
            out.append((name + " I slice first", i_slice_first(stream(workdir, name, w, h, args))[0], NONKEY, None))
    return out


def i_slice_first(data):
    """The stream with, in every P or B picture that has an I slice, one such slice moved to the front of the picture
    (slices of a picture may come in any order to this decoder), and the number of pictures moved."""
    nals = _nals(data)
    order = list(range(len(nals)))
    moved = 0
    for p in pictures(data):
        if p["slices"][0] != 2 and 2 in p["slices"]:
            i = p["nals"][p["slices"].index(2)]
            order.remove(i)
            order.insert(order.index(p["nals"][0]), i)
            moved += 1
    return b"".join(b"\x00\x00\x00\x01" + data[s:e] for s, e in (nals[i] for i in order)), moved


def test_reordered_mixed_slices_decode_like_the_original(workdir):
    for name, w, h, args in DPB_STREAMS:
        if name.startswith("mixed_slices"):
            data = stream(workdir, name, w, h, args)
            moved, n = i_slice_first(data)
            assert n >= 2
            a, b = decode(data)[0], decode(moved)[0]
            assert [(f[0], f[1]) for f in a] == [(f[0], f[1]) for f in b], name


def test_pictures_predicting_from_skipped_ones_are_marked(workdir):
    for label, data, mode, hook in rule3_cases(workdir):
        full, _ = decode(data)
        for t in (0, 3):
            part, codes = decode(data, n_threads=t, skip=mode, before=hook)
            check_subset(full, part, label, exact=False)
            marked = [f for f in part if f[2] is not None and [g for g in full if g[0] == f[0]][0][2] is None]
            assert marked, "%s: no frame marks the macroblocks predicted from a skipped picture" % label
            assert all(100 in f[2] for f in marked), label
            if t == 0:
                ref = part
            else:
                assert [f[:3] for f in part] == [f[:3] for f in ref], "%s: differs with %d workers" % (label, t)


# ---- 4. the slice data of a skipped picture is not parsed ----
def damaged_b(workdir):
    """(stream, damaged stream, index of the damaged NAL unit): slice data of one non-reference B picture cut short or
    overwritten, in the first way the full decode answers EBADMSG for"""
    name, w, h, args = next(s for s in STREAMS if s[0] == "b_default")
    data = stream(workdir, name, w, h, args)
    nals = _nals(data)
    pics = pictures(data)
    k = next(p["nals"][0] for p in pics[4:] if p["ref"] == 0 and p["slices"] == [1])
    s, e = nals[k]
    for frac in (0.5, 0.3, 0.7, 0.85):
        cut = s + max(8, int((e - s) * frac))
        for dmg in (data[:cut] + data[e:], data[:cut] + bytes([0xff, 0x5a] * ((e - cut) // 2)) + data[cut + (e - cut) // 2 * 2:]):
            codes = decode(dmg)[1]
            if codes[k] == errno.EBADMSG:
                return data, dmg, k
    pytest.fail("no damage made the full decode answer EBADMSG")


def test_skipped_slice_data_is_not_parsed(workdir):
    data, dmg, k = damaged_b(workdir)
    clean, _ = decode(data, skip=NONREF)
    for t in (0, 3):
        frames, codes = decode(dmg, n_threads=t, skip=NONREF)
        assert codes[k] == 0
        assert [f[:3] for f in frames] == [f[:3] for f in clean], t


def test_damaged_streams_keep_the_record_contract(workdir, monkeypatch):
    lib = port_outputs_lib()
    monkeypatch.setenv("E264_CHECK_RECORDS", "1")
    for name, seed, data in _damaged(workdir):
        for mode in (NONREF, NONKEY):
            for t in (0, 3):
                decode(data, n_threads=t, skip=mode)
                assert lib.e264_test_record_violations() == 0, "%s seed %d mode %d (%d workers): %s" % (name, seed, mode, t, lib.e264_test_last_violation())


# ---- 6. API ----
def test_api_errors():
    lib = port_outputs_lib()
    assert lib.edge264_set_skip(None, NONREF) == errno.EINVAL
    dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
    for mode in (3, -1, 100):
        assert lib.edge264_set_skip(dec, mode) == errno.EINVAL
    for mode in (NONE, NONREF, NONKEY):
        assert lib.edge264_set_skip(dec, mode) == 0
    d = ctypes.c_void_p(dec)
    lib.edge264_free(ctypes.byref(d))
    assert hasattr(checkers.load("port"), "edge264_set_skip")


def test_mode_set_mid_picture_applies_from_the_next_picture(workdir):
    name, w, h, args = next(s for s in STREAMS if s[0] == "b_scaling_mv")   # two slices per picture
    data = stream(workdir, name, w, h, args)
    pics = pictures(data)
    nonref = [p for p in pics if p["ref"] == 0]
    assert len(nonref) >= 2 and len(nonref[0]["nals"]) == 2
    k = nonref[0]["nals"][1]                      # between the two slices of the first non-reference picture
    full, _ = decode(data)
    part, _ = decode(data, before=switch_at(k, NONREF))
    order = sorted(f[0] for f in full)
    first_nonref = order[pics.index(nonref[0])]
    assert first_nonref in [f[0] for f in part]   # already started: decoded
    later = [order[i] for i, p in enumerate(pics) if p["ref"] == 0 and p["nals"][0] > k]
    assert later and not set(later) & {f[0] for f in part}
    check_subset(full, part, "mid-picture switch")


def test_reference_library_has_no_skip(workdir):
    if not have("ref"):
        pytest.skip("oracle/_ref not built")
    lib = checkers.load("ref")
    assert not hasattr(lib, "edge264_set_skip")
    data = stream(workdir, *STREAMS[6])
    with pytest.raises(RuntimeError, match="ENOTSUP"):
        pkg.decode_bytes(data, lib, skip=NONREF)
    assert pkg.decode_bytes(data, lib, skip=NONE)[0]


# ---- GPU: the device against the port ----
def _gpu_inputs(workdir):
    for name, w, h, args in ALL:
        yield name, stream(workdir, name, w, h, args), NONREF, None
        yield name, stream(workdir, name, w, h, args), NONKEY, None
    for label, data, mode, hook in rule3_cases(workdir):
        yield label, data, mode, hook
    yield "damaged B", damaged_b(workdir)[1], NONREF, None
    for name, seed, data in _damaged(workdir):
        yield "%s/%d" % (name, seed), data, NONREF, None
        yield "%s/%d" % (name, seed), data, NONKEY, None


@pytest.mark.gpu
def test_device_matches_port(workdir):
    for label, data, mode, hook in _gpu_inputs(workdir):
        for t in (0, 3):
            g, gc = decode(data, "gpu", t, mode, before=hook)
            p, pc = decode(data, "port", t, mode, before=hook)
            assert [f[0] for f in g] == [f[0] for f in p], (label, mode, t)
            for a, b in zip(g, p):
                assert a[1] == b[1], "%s mode %d (%d workers) frame %d: samples differ" % (label, mode, t, a[0])
                assert a[2] == b[2], "%s mode %d (%d workers) frame %d: maps differ" % (label, mode, t, a[0])
            if t == 0:
                assert gc == pc, label


@pytest.mark.gpu
def test_device_nonkey_motion_matches_port(workdir):
    for name, w, h, args in I_STREAMS:
        data = stream(workdir, name, w, h, args)
        g, _ = decode(data, "gpu", skip=NONKEY, motion=True)
        p, _ = decode(data, "port", skip=NONKEY, motion=True)
        assert [f[0] for f in g] == [f[0] for f in p]
        for a, b in zip(g, p):
            assert all((a[3][k] == b[3][k]).all() for k in a[3]), (name, a[0])


# ---- 5. device cost ----
def stats_per_nal(data, skip, hook=None):
    """launches, H2D and D2H bytes each NAL unit's decode_NAL caused, synchronous decoding"""
    per = []
    s = [ctypes.c_uint64() for _ in range(3)]
    def after(k, lib, dec):
        lib.e264b_stats(lib.e264b_of_decoder(dec), *[ctypes.byref(x) for x in s])
        per.append(tuple(x.value for x in s))
    lib = pkg.load()
    lib.e264b_of_decoder.restype = ctypes.c_void_p; lib.e264b_of_decoder.argtypes = [ctypes.c_void_p]
    lib.e264b_stats.argtypes = [ctypes.c_void_p] + [ctypes.POINTER(ctypes.c_uint64)] * 3
    frames, _ = decode(data, "gpu", 0, skip, before=hook, after=after)
    deltas = [tuple(b - a for a, b in zip(per[i - 1] if i else (0, 0, 0), per[i])) for i in range(len(per))]
    return deltas, frames


@pytest.mark.gpu
def test_skipped_pictures_cost_the_device_nothing(workdir):
    for name, w, h, args in [s for s in STREAMS if s[0] in ("b_default", "b_scaling_mv", "bref_spatial")] + I_STREAMS:
        data = stream(workdir, name, w, h, args)
        pics = pictures(data)
        full, _ = stats_per_nal(data, NONE)
        for mode in (NONREF, NONKEY):
            part, frames = stats_per_nal(data, mode)
            want = [sum(full[k][i] for p in pics if kept(p, mode) for k in p["nals"]) for i in range(3)]
            got = [sum(d[i] for d in part) for i in range(3)]
            assert got == want, (name, mode, got, want)
            for p in pics:
                if not kept(p, mode):
                    assert all(part[k] == (0, 0, 0) for k in p["nals"]), (name, mode)
