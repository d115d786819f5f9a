"""Low-latency output (include/edge264_latency.h): edge264_set_output_latency(dec, N) caps the output reorder depth at N
and makes edge264_get_frame wait for a due frame whose picture is closed.  The mode is defined by a twin stream: the same
bits with VUI bitstream_restriction stating max_num_reorder_frames = min(N, the value in force) and
max_dec_frame_buffering unchanged.  tools/gen264 --no-vui writes a stream whose depths are inferred from the level (the
camera case), and --no-vui --reorder N its twin.

The oracle is the compiled reference decoder decoding the twins: tests/golden/latency.json holds, for every pair below,
the return code of each edge264_decode_NAL and the frames each following edge264_get_frame loop returned
(tests/make_latency_golden.py records it).  CPU tests run the product's host sources over the plain-C restatement
(oracle/liboracle_dec.so, and the restatement with every optional output); the GPU tests compare the device with the
goldens and with the restatement, and count its launches and copies."""
import ctypes, errno, functools, hashlib, json, os, random
from concurrent.futures import ThreadPoolExecutor
import pytest
from conftest import ROOT, make_stream, have
from checkers import load, port_outputs_lib, Edge264Frame, _frame_bytes
from api_helpers import _damaged
from test_mb_errors import _nals
import edge264_b200 as pkg

GOLDEN = os.path.join(ROOT, "tests", "golden", "latency.json")

# (name, width_mbs, height_mbs, generator arguments): streams without VUI, decoded with the mode at each depth of DEPTHS
PAIRS = [
    ("lat_i_cabac",      6, 4, "-n 5 -s 3001 --gop I --deblock 0 --t8x8 50"),
    ("lat_ip_cavlc",     7, 5, "-n 12 -s 3002 --gop IP --refs 3 --cavlc --deblock 2"),
    ("lat_ipb_cabac",    9, 7, "-n 14 -s 3003 --gop IPB --wp 2 --temporal --deblock 0"),
    ("lat_ipb_cavlc",    8, 6, "-n 14 -s 3004 --gop IPB --refs 2 --cavlc --slices 3 --mixed-slices --wp 1"),
    ("lat_bref",         4, 4, "-n 30 -s 3005 --gop IPB --bref --refs 3 --idr 11 --deblock 0 --wp 1"),
    ("lat_dpb_ip",       4, 3, "-n 40 -s 3006 --gop IP --refs 4 --dpb --idr 17 --deblock 0"),
    ("lat_dpb_ipb",      5, 4, "-n 40 -s 3007 --gop IPB --refs 4 --dpb --idr 23 --wp 2"),
    ("lat_mmco5",        4, 3, "-n 30 -s 3008 --gop IP --refs 3 --dpb --mmco5 --idr 13 --cavlc"),
    ("lat_crop_iperiod", 6, 5, "-n 20 -s 3009 --gop IPB --i-period 5 --refs 3 --crop-left 4 --crop-top 2 --crop-bottom 6"),
    ("lat_poc2_nonref",  4, 4, "-n 20 -s 3010 --gop IP --nonref-p --extra-nals --refs 3 --idr 9 --poc-type 2"),
]
DEPTHS = (0, 1, 2)
# frame_num gaps: a stream with the NAL units of some reference pictures removed (the same units of its twin)
GAP = ("lat_gap", 5, 4, "-n 24 -s 3011 --gop IP --refs 3 --idr 30 --deblock 0")
GAP_DROP = (7, 8, 15)
# the streams' own VUI (max_num_reorder_frames 1 for IPB, 0 for IP): below it the twin, at or above it the default decode
VUI = [("lat_vui_ipb", 9, 7, "-n 14 -s 3012 --gop IPB --refs 2 --wp 1"), ("lat_vui_ip", 7, 5, "-n 12 -s 3013 --gop IP --refs 2")]
# stereo: the subset SPS has no VUI either; pairs leave as the reference pairs them
MVC = [("lat_mvc_ipb", 9, 7, "-n 14 -s 3014 --gop IPB --deblock 0 --t8x8 50 --mvc 3"),
       ("lat_mvc_dpb", 5, 4, "-n 30 -s 3015 --gop IP --refs 4 --dpb --idr 17 --wp 1 --mvc 4")]
MVC_DEPTHS = (0, 1)
# 1920x1088 at level 5.1 (an inferred depth of 16): decoded on the GPU only
FULL = [("lat_1080p_ip", 120, 68, "-n 8 -s 3016 --gop IP --level 51 --t8x8 50 --density 40"),
        ("lat_1080p_ipb", 120, 68, "-n 8 -s 3017 --gop IPB --level 51 --refs 2 --t8x8 50 --density 40")]
FULL_DEPTHS = {"lat_1080p_ip": 0, "lat_1080p_ipb": 1}
HOLDS = (1, 3)
FLUSH_AT = (9, 20)


@functools.lru_cache(None)
def gold():
    """Read on first use, so that tests/make_latency_golden.py can import this module without the file."""
    return json.load(open(GOLDEN))


def _md5(b):
    return hashlib.md5(b).hexdigest()


def original(workdir, s):
    name, w, h, args = s
    return open(make_stream(workdir, name, w, h, args + " --no-vui"), "rb").read()


def twin(workdir, s, n, vui=False):
    """The twin of stream s for depth n; vui=True: of the stream with its own VUI (VUI, MVC-less streams of VUI)."""
    name, w, h, args = s
    return open(make_stream(workdir, "%s_r%d" % (name, n), w, h, args + ("" if vui else " --no-vui") + " --reorder %d" % n), "rb").read()


def drop(data, ks):
    """the stream without its NAL units ks (indices in decoding order)"""
    return b"".join(b"\x00\x00\x00\x01" + data[a:b] for k, (a, b) in enumerate(_nals(data)) if k not in ks)


def cases(workdir, full=False):
    """name -> (stream decoded with the mode, its twin, depth) of every pair the goldens hold"""
    out = {}
    for s in PAIRS + MVC:
        for n in (MVC_DEPTHS if s in MVC else DEPTHS):
            out["%s/%d" % (s[0], n)] = (original(workdir, s), twin(workdir, s, n), n)
    for n in DEPTHS:
        out["%s/%d" % (GAP[0], n)] = (drop(original(workdir, GAP), GAP_DROP), drop(twin(workdir, GAP, n), GAP_DROP), n)
    out["lat_vui_ipb/0"] = (open(make_stream(workdir, *VUI[0]), "rb").read(), twin(workdir, VUI[0], 0, vui=True), 0)
    if full:
        for s in FULL:
            out["%s/%d" % (s[0], FULL_DEPTHS[s[0]])] = (original(workdir, s), twin(workdir, s, FULL_DEPTHS[s[0]]), FULL_DEPTHS[s[0]])
    return out


def observe(data, lib, n_threads=0, latency=-1, hold=0, flush_at=None, hooks=None, **modes):
    """The README loop over the C API: per decode_NAL call [NAL index, return code, indices of the frames its get_frame
    loop returned], and per frame [FrameId, md5, FrameId_mvc, md5_mvc].  hold > 0: every frame is borrowed and handed back
    `hold` frames later; flush_at: edge264_flush after that NAL unit; hooks {k: depth}: edge264_set_output_latency before
    NAL unit k; modes: skip=, luma_only=, loop_filter= as in edge264_b200.decode_bytes."""
    buf = ctypes.create_string_buffer(data, len(data) + 64)
    base = ctypes.addressof(buf); end = base + len(data)
    dec = lib.edge264_alloc(n_threads, None, None, 0, None, None, None)
    assert dec
    if latency != -1:
        assert lib.edge264_set_output_latency(dec, latency) == 0
    if modes.get("skip"):
        assert lib.edge264_set_skip(dec, modes["skip"]) == 0
    if modes.get("luma_only"):
        assert lib.edge264_enable_luma_only(dec) == 0
    if modes.get("loop_filter"):
        assert lib.edge264_set_loop_filter(dec, modes["loop_filter"]) == 0
    nal = base + 3 + (1 if data[2] == 0 else 0)
    held, frames, calls, f, k = [], [], [], Edge264Frame(), 0

    def give_back():
        fr = held.pop(0)
        lib.edge264_return_frame(dec, fr.return_arg)
    while True:
        sc = lib.edge264_find_start_code(nal, end, 0) if nal < end else end
        if hooks and k in hooks:
            lib.edge264_set_output_latency(dec, hooks[k])
        res = lib.edge264_decode_NAL(dec, nal, sc, None, None)
        got = []
        while lib.edge264_get_frame(dec, ctypes.byref(f), 1 if hold else 0) == 0:
            mvc = bool(f.samples_mvc[0])
            frames.append([f.FrameId, _md5(_frame_bytes(f)), f.FrameId_mvc if mvc else None, _md5(_frame_bytes(f, True)) if mvc else None])
            got.append(len(frames) - 1)
            if hold:
                held.append(Edge264Frame.from_buffer_copy(bytes(f)))
                while len(held) > hold:
                    give_back()
        calls.append([k, res, got])
        if res == errno.ENOBUFS:
            if not got:
                if not held:
                    break
                give_back()
            continue
        if flush_at is not None and k == flush_at:
            while held:
                give_back()
            lib.edge264_flush(dec)
        if res not in (0, errno.ENOTSUP, errno.EBADMSG) or nal >= end:
            break
        nal = sc + 3 if sc + 3 < end else end
        k += 1
    while held:
        give_back()
    d = ctypes.c_void_p(dec)
    lib.edge264_free(ctypes.byref(d))
    return {"calls": calls, "frames": frames}


def api_cases(workdir):
    """name -> (stream, depth, hold, flush_at) of the API observations: borrowed frames, flush mid-stream, End of sequence"""
    ipb, dpb = original(workdir, PAIRS[2]), original(workdir, PAIRS[6])
    mono = original(workdir, PAIRS[1])
    out = {"hold%d/%s" % (h, s[0]): (d, n, h, None) for s, d, n in ((PAIRS[2], ipb, 0), (PAIRS[6], dpb, 1)) for h in HOLDS}
    out.update({"flush%d" % at: (dpb, 1, 1, at) for at in FLUSH_AT})
    out["eos"] = (ipb + b"\x00\x00\x00\x01\x0a" + mono, 0, 0, None)
    return out


def api_twin(workdir, name):
    """the twin of an API case's stream"""
    ipb, dpb, mono = twin(workdir, PAIRS[2], 0), twin(workdir, PAIRS[6], 1), twin(workdir, PAIRS[1], 0)
    if name == "eos":
        return ipb + b"\x00\x00\x00\x01\x0a" + mono
    return ipb if PAIRS[2][0] in name else dpb


def frame_nal(obs):
    """per frame, the NAL index after which it was returned"""
    out = {}
    for k, _, got in obs["calls"]:
        for i in got:
            out[i] = k
    return [out[i] for i in range(len(obs["frames"]))]


def codes(obs):
    return [c for _, c, _ in obs["calls"]]


def final_codes(obs):
    """the return code of every NAL unit: a frame still being parsed when a picture needs its buffer, or at the end of the
    stream, makes a call answer ENOBUFS first with workers, as it does without the mode"""
    return [c for c in codes(obs) if c != errno.ENOBUFS]


def ids(obs):
    """obs without the samples: the frames of pictures predicted from the non-existing frames of a frame_num gap have
    samples the reference leaves undefined (never-written buffers) and this decoder clears"""
    return {"calls": obs["calls"], "frames": [[f[0], f[2]] for f in obs["frames"]]}


def views(obs):
    """per view, the frames in output order"""
    return [[f[0:2] for f in obs["frames"]], [f[2:4] for f in obs["frames"] if f[2] is not None]]


def check_threaded(data, obs, g):
    """With workers: the frames, FrameIds and return codes of the golden, every frame no later than the get_frame loop after
    the first slice of the next picture that follows the NAL unit after which the reference returned it.  A frame still
    being parsed at the end of the stream makes that call answer ENOBUFS first, as it does without the mode.
    Stereo streams: the reference counts a picture towards its view's depth by the frame buffer it takes, which depends on
    which frames the application has fetched (tests/test_mvc.py); with workers a due frame may still be parsed when the
    next picture starts, so each view's frames and the return codes are the golden's, but pairs may be formed otherwise."""
    assert final_codes(obs) == final_codes(g)
    if any(f[2] is not None for f in g["frames"]):
        assert sorted(views(obs)[0]) == sorted(views(g)[0]) and sorted(views(obs)[1]) == sorted(views(g)[1])
        return
    assert obs["frames"] == g["frames"]
    nals = _nals(data)
    slices = [k for k, (a, _) in enumerate(nals) if data[a] & 31 in (1, 5, 20)] + [len(nals)]
    for i, (want, got) in enumerate(zip(frame_nal(g), frame_nal(obs))):
        bound = next((k for k in slices if k > want), len(nals))
        assert want <= got <= bound, "frame %d: returned after NAL %d, the reference after NAL %d" % (i, got, want)


# ---- CPU: the twin streams ----
def test_twins_differ_from_their_stream_in_the_sps_only(workdir):
    """--no-vui and --reorder N change the sequence parameter sets and nothing else; without --no-vui, --reorder leaves a
    stream that already states N unchanged"""
    for s in (PAIRS[3], MVC[0]):
        a, b = original(workdir, s), twin(workdir, s, 0)
        na, nb = _nals(a), _nals(b)
        assert len(na) == len(nb)
        diff = {a[x] & 31 for (x, y), (u, v) in zip(na, nb) if a[x:y] != b[u:v]}
        assert diff == ({7, 15} if s in MVC else {7})
    assert twin(workdir, VUI[0], 1, vui=True) == open(make_stream(workdir, *VUI[0]), "rb").read()


CPU_NAMES = ["%s/%d" % (s[0], n) for s in PAIRS for n in DEPTHS] + ["%s/%d" % (GAP[0], n) for n in DEPTHS] + ["lat_vui_ipb/0"] + \
            ["%s/%d" % (s[0], n) for s in MVC for n in MVC_DEPTHS]


@pytest.mark.parametrize("name", CPU_NAMES)
def test_port_equals_the_reference_on_the_twin(workdir, name):
    """Without workers the calls, frames and return codes are the golden's exactly; with 1 and 3 workers the frames and
    codes are, and every frame comes out no later than the loop after the next picture's first slice."""
    data, tw, n = cases(workdir)[name]
    g = gold()["pairs"][name]
    assert g["twin_md5"] == _md5(tw), "tools/gen264 no longer writes the twin of the golden"
    port = load("port")
    low, want = observe(data, port, 0, n), {"calls": g["calls"], "frames": g["frames"]}
    assert low == observe(tw, port, 0)   # the twin decoded without the mode
    assert (ids(low) == ids(want)) if name.startswith(GAP[0]) else (low == want)
    for t in (1, 3):
        obs = observe(data, port, t, n)
        check_threaded(data, obs, g if not name.startswith(GAP[0]) else dict(g, frames=low["frames"]))


def test_default_mode_holds_frames_back(workdir):
    """Without the mode a stream without VUI holds frames back (its level's depth is 16 here; the decoder's frame slots, four
    beyond the references, bound it first); at depth 0 each frame of an IP stream leaves after the NAL unit that completes
    its picture"""
    s = PAIRS[5]
    data, port = original(workdir, s), load("port")
    default, low = observe(data, port), observe(data, port, 0, 0)
    assert default["frames"] == low["frames"]
    pics = [k for k, (a, _) in enumerate(_nals(data)) if data[a] & 31 in (1, 5)]
    assert frame_nal(low) == pics
    held = [pics.index(max(k for k in pics if k <= at)) - i for i, at in enumerate(frame_nal(default)) if at < len(_nals(data))]
    assert max(held) >= 4


@pytest.mark.parametrize("s", VUI, ids=[s[0] for s in VUI])
def test_streams_with_vui(workdir, s):
    """at or above the stream's own max_num_reorder_frames the decode is the default decode, call by call"""
    data, port = open(make_stream(workdir, *s), "rb").read(), load("port")
    default = observe(data, port)
    for n in (1, 2, 16) if "ipb" in s[0] else (0, 1, 16):
        assert observe(data, port, 0, n) == default, n


def test_mode_switches(workdir):
    """-1 set before every NAL unit is the decoder without the call; a switch applies from the next picture's first slice;
    the frames of any sequence of switches are the default decode's, and before the first switch so is every call"""
    port = load("port")
    for s in (PAIRS[2], PAIRS[6]):
        data = original(workdir, s)
        default = observe(data, port)
        n_nals = len(_nals(data))
        assert observe(data, port, hooks={k: -1 for k in range(n_nals + 1)}) == default
        assert observe(data, port, hooks={0: 1}) == observe(data, port, 0, 1)
        for t in (0, 3):
            got = observe(data, port, t, hooks={9: 0, 20: -1, 30: 2})
            assert sorted(got["frames"]) == sorted(default["frames"]) and final_codes(got) == final_codes(default)
            if t == 0:
                assert got["calls"][:9] == default["calls"][:9]
    # set between two slices of a picture: the picture keeps the depth read at its first slice
    from test_skip import pictures
    data = original(workdir, PAIRS[3])
    pics = pictures(data)
    assert len(pics[4]["nals"]) > 1
    assert observe(data, port, hooks={pics[4]["nals"][1]: 0}) == observe(data, port, hooks={pics[5]["nals"][0]: 0}) != observe(data, port)


def test_optional_outputs_are_unchanged(workdir):
    """error maps, motion export, statistics, packed and resized output: byte for byte the default decode's (IP and IPB
    streams at a depth that keeps POC order, so the frames come out in the same order)"""
    lib = port_outputs_lib()
    for s, n in ((PAIRS[5], 0), (PAIRS[3], 1), (PAIRS[8], 1)):
        data = original(workdir, s)
        for kw in ({"errors": True, "motion": True, "picstats": True}, {"packed": (pkg.PACKED_NV12, 1)}, {"resized": (pkg.PACKED_I420, 30, 22)}):
            for t in (0, 3):
                a, b = pkg.decode_bytes(data, lib, t, **kw), pkg.decode_bytes(data, lib, t, output_latency=n, **kw)
                assert repr(a) == repr(b), (s[0], sorted(kw), t)


COMBOS = [{"skip": pkg.SKIP_NONREF}, {"skip": pkg.SKIP_NONKEY}, {"luma_only": True}, {"loop_filter": pkg.LOOP_FILTER_REF},
          {"loop_filter": pkg.LOOP_FILTER_NONE, "luma_only": True}]


@pytest.mark.parametrize("kw", COMBOS, ids=["-".join("%s%s" % i for i in sorted(k.items())) for k in COMBOS])
def test_combinations_equal_the_twins(workdir, kw):
    """with skip, luma-only and loop filter modes the mode's decode is the twin's decode in those modes, call by call"""
    lib = port_outputs_lib()
    for s, n in ((PAIRS[2], 0), (PAIRS[4], 1), (MVC[0], 0)):
        data, tw = original(workdir, s), twin(workdir, s, n)
        assert observe(data, lib, 0, n, **kw) == observe(tw, lib, 0, **kw), s[0]
        check_threaded(data, observe(data, lib, 3, n, **kw), observe(tw, lib, 0, **kw))


@pytest.mark.parametrize("name", ["hold1/lat_ipb_cabac", "hold3/lat_ipb_cabac", "hold1/lat_dpb_ipb", "hold3/lat_dpb_ipb", "flush9", "flush20", "eos"])
def test_api_observations(workdir, name):
    """borrowed frames handed back later, edge264_flush mid-stream and End of sequence: the reference's calls on the twin"""
    data, n, hold, at = api_cases(workdir)[name]
    g = gold()["api"][name]
    assert observe(data, load("port"), 0, n, hold, at) == g
    assert observe(api_twin(workdir, name), load("port"), 0, -1, hold, at) == g


def test_damaged_streams(workdir, monkeypatch):
    """The damaged streams of test_robustness.py at depth 0: every submitted picture keeps the record contract.  Without
    workers the return codes, FrameIds, samples and error maps are the default decode's.  With workers the return codes
    are; a slice that continues a picture whose slices already covered every macroblock starts a new picture if a worker
    has closed the first one by then (as without workers), and joins it otherwise (as without the mode)."""
    lib = port_outputs_lib()
    monkeypatch.setenv("E264_CHECK_RECORDS", "1")
    before, n = lib.e264_test_record_violations(), 0
    by_id = lambda fr: sorted(fr, key=lambda f: f[0])
    for name, seed, data in _damaged(workdir, 10):
        full = pkg.decode_bytes(data, lib, 0, errors=True)
        got = pkg.decode_bytes(data, lib, 0, errors=True, output_latency=0)
        assert got[1] == full[1] and by_id(got[0]) == by_id(full[0]), "%s seed %d" % (name, seed)
        assert pkg.decode_bytes(data, lib, 3, errors=True, output_latency=0)[1] == pkg.decode_bytes(data, lib, 3, errors=True)[1]
        n += 1
    assert n == 30
    assert lib.e264_test_record_violations() == before, lib.e264_test_last_violation()


def test_api_contract(workdir):
    lib = port_outputs_lib()
    assert lib.edge264_set_output_latency(None, 0) == errno.EINVAL
    dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
    for v in (-2, 17, 100, -100):
        assert lib.edge264_set_output_latency(dec, v) == errno.EINVAL
    for v in (-1, 0, 16, 5, -1):
        assert lib.edge264_set_output_latency(dec, v) == 0
    d = ctypes.c_void_p(dec)
    lib.edge264_free(ctypes.byref(d))
    if have("ref"):
        ref = load("ref")
        assert not hasattr(ref, "edge264_set_output_latency")
        with pytest.raises(RuntimeError, match="ENOTSUP"):
            pkg.decode_bytes(original(workdir, PAIRS[1]), ref, output_latency=0)


# ---- GPU ----
GPU_NAMES = ["%s/%d" % (s[0], n) for s in PAIRS for n in (0, 1)] + ["%s/0" % GAP[0], "lat_vui_ipb/0"] + \
            ["%s/%d" % (s[0], n) for s in MVC for n in MVC_DEPTHS] + ["%s/%d" % (s[0], n) for s, n in ((FULL[0], 0), (FULL[1], 1))]


@pytest.mark.gpu
@pytest.mark.parametrize("name", GPU_NAMES)
def test_device_equals_the_goldens(workdir, name):
    """Without workers every call returns the frames the reference returns after the same NAL unit: no get_frame answers
    ENOMSG for a frame the reference has finished, the wait for the device is inside the call.  With 3 workers the bound
    of the CPU tests holds; colour and luma-only equal the restatement."""
    data, tw, n = cases(workdir, full=True)[name]
    g = gold()["pairs"][name]
    assert g["twin_md5"] == _md5(tw)
    lib, want = pkg.load(), {"calls": g["calls"], "frames": g["frames"]}
    low = observe(data, lib, 0, n)
    if name.startswith(GAP[0]):   # samples predicted from a frame_num gap's frames: those of the restatement
        assert ids(low) == ids(want) and low == observe(data, load("port"), 0, n)
        want["frames"] = low["frames"]
    assert low == want
    check_threaded(data, observe(data, lib, 3, n), want)
    if "1080p" not in name:
        port = load("port")
        assert observe(data, lib, 0, n, luma_only=True) == observe(data, port, 0, n, luma_only=True)


@pytest.mark.gpu
def test_many_decoders_in_flight(workdir):
    """8 host threads decode the pairs in mixed modes (default, depth 0, depth 1; 0 or 2 workers) at once, twice, in
    shuffled orders; each output equals that decoder's output alone"""
    lib = pkg.load()
    data = {s[0]: original(workdir, s) for s in PAIRS + FULL[:1]}
    jobs = [(nm, m, t) for nm in data for m in (-1, 0, 1) for t in (0, 2)]
    alone = {j: pkg.decode_bytes(data[j[0]], lib, j[2], output_latency=j[1]) for j in jobs}
    for r in range(2):
        random.Random(r).shuffle(jobs)
        with ThreadPoolExecutor(8) as ex:
            got = list(ex.map(lambda j: pkg.decode_bytes(data[j[0]], lib, j[2], output_latency=j[1]), jobs))
        for j, g in zip(jobs, got):
            assert g == alone[j], j


@pytest.mark.gpu
def test_launch_and_copy_counts(workdir):
    """e264b_stats after every NAL unit: the mode launches and copies what the default decode does, NAL unit by NAL unit"""
    from test_skip import stats_per_nal
    for s in (PAIRS[2], PAIRS[6], FULL[0]):
        data = original(workdir, s)
        full, ffull = stats_per_nal(data, pkg.SKIP_NONE)
        for n in (0, 1):
            low, flow = stats_per_nal(data, pkg.SKIP_NONE, lambda k, lib, dec: k == 0 and lib.edge264_set_output_latency(dec, n))
            assert low == full and sorted(f[0] for f in flow) == sorted(f[0] for f in ffull), (s[0], n)
