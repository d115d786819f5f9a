"""Streams at the standard's limits, stream -> parser -> records -> kernels, against the reference decoder's output.

tools/gen264 keeps its default streams far inside the standard; its options --qp-walk, --levels big, --cqp-offset,
--wp-range full and --pcm-extreme write mb_qp_delta over -26..25 with QP_Y wrapping modulo 52, levels up to the 8-bit
bound -32768..32767 (CAVLC level_prefix 15, 16 and above, long CABAC suffixes), fixed chroma QP offsets of up to +-12,
explicit weights and offsets over -128..127 at logWD 0..7, and PCM macroblocks with 0/255 steps, ramps, checkers and
random bits as intra and inter sources.  tests/golden/limits.json (written by tests/make_limits_golden.py from the compiled
reference) pins each stream's bytes and the reference's frames.  The CPU half checks the generator, the port, the
reference when it is built, the record contract, and that the limits are actually reached (the port's E264_COVERAGE
counters); the GPU half checks the device against the same digests without the reference."""
import functools, hashlib, json, os, re, subprocess
import pytest
from conftest import ROOT, make_stream, md5_frames, have
from checkers import decode_bytes



@functools.lru_cache(None)
def gold():
    """Read on first use, so that tests/make_limits_golden.py can import the stream lists without the file."""
    return json.load(open(os.path.join(ROOT, "tests", "golden", "limits.json")))


# (name, width_mbs, height_mbs, generator arguments): CAVLC and CABAC, 4x4 and 8x8 transforms, scaling lists, several
# slices, deblocking idc 0 and 2 (with the generator's filter offsets of -12..12), P and B pictures, reference B
# pictures, spatial and temporal direct
LIMITS = [
    ("lim_qp_cabac",      6, 4, "-n 6 -s 301 --gop IPB --qp-walk --levels big --cqp-offset -12,12 --deblock 0 --t8x8 50"),
    ("lim_qp_cavlc",      7, 5, "-n 6 -s 302 --gop IP --qp-walk --levels big --cqp-offset 12,-12 --deblock 2 --slices 2 --cavlc"),
    # high QPs with scaling lists: the 4x4 saturation and the 8x8 int16 wrap the reference computes (DESIGN §5)
    ("lim_levels_i_cabac", 5, 4, "-n 3 -s 303 --gop I --levels big --t8x8 50 --scaling 3 --qp 40 --deblock 0 --density 60"),
    ("lim_levels_i_cavlc", 5, 4, "-n 3 -s 304 --gop I --levels big --t8x8 0 --scaling 2 --qp 45 --deblock 0 --density 60 --cavlc"),
    ("lim_cqp_low_cavlc", 4, 3, "-n 6 -s 305 --gop IP --qp-walk --cqp-offset -12,-7 --deblock 0 --cavlc"),
    ("lim_wp_p",          8, 6, "-n 8 -s 306 --gop IP --wp-range full --wp 1 --refs 4 --deblock 0"),
    ("lim_wp_b_spatial",  8, 6, "-n 10 -s 307 --gop IPB --wp-range full --wp 1 --refs 3 --bref --deblock 0"),
    ("lim_wp_b_temporal_cavlc", 9, 7, "-n 10 -s 308 --gop IPB --wp-range full --wp 1 --refs 2 --temporal --slices 3 --deblock 2 --cavlc"),
    ("lim_pcm_intra",     6, 5, "-n 3 -s 309 --gop I --pcm 300 --pcm-extreme --t8x8 50 --deblock 0"),
    ("lim_pcm_ipb",       9, 7, "-n 9 -s 310 --gop IPB --pcm 200 --pcm-extreme --wp-range full --wp 1 --mvrange 40 --deblock 0"),
    ("lim_all_cabac",     13, 9, "-n 7 -s 311 --gop IPB --qp-walk --levels big --cqp-offset 5,-12 --wp-range full --wp 1 --pcm 80 --pcm-extreme --scaling 3 --t8x8 50 --slices 3 --deblock 0"),
    ("lim_all_cavlc",     4, 3, "-n 10 -s 312 --gop IPB --qp-walk --levels big --cqp-offset -3,9 --wp-range full --wp 1 --pcm 120 --pcm-extreme --t8x8 50 --deblock 2 --temporal --cavlc"),
]
# 1920x1088 on the GPU only, against the reference's summary line (frame count and digest of all frames)
FULL_LIMITS = [
    ("lim_1080p_qp_levels", 120, 68, "-n 3 -s 321 --gop IPB --qp-walk --levels big --cqp-offset -12,12 --t8x8 50 --deblock 0"),
    ("lim_1080p_wp_pcm",    120, 68, "-n 4 -s 322 --gop IPB --wp-range full --wp 1 --pcm 60 --pcm-extreme --t8x8 50 --deblock 0"),
]
IDS = [s[0] for s in LIMITS]


@pytest.mark.parametrize("name,w,h,args", LIMITS + FULL_LIMITS, ids=IDS + [s[0] for s in FULL_LIMITS])
def test_generator_writes_the_recorded_stream(workdir, name, w, h, args):
    g = gold()[name]
    assert g["args"] == f"-W {w} -H {h} {args}"
    data = open(make_stream(workdir, name, w, h, args), "rb").read()
    assert (len(data), hashlib.md5(data).hexdigest()) == (g["bytes"], g["stream_md5"])


@pytest.mark.parametrize("name,w,h,args", LIMITS, ids=IDS)
def test_port_matches_golden(workdir, name, w, h, args):
    data = open(make_stream(workdir, name, w, h, args), "rb").read()
    port, _ = decode_bytes(data, "port")
    assert md5_frames(port) == gold()[name]["md5"], "the port differs from the reference's recorded frames"


@pytest.mark.skipif(not have("ref"), reason="oracle/_ref (the compiled reference decoder) is not built")
@pytest.mark.parametrize("name,w,h,args", LIMITS, ids=IDS)
def test_reference_matches_golden_and_port(workdir, name, w, h, args):
    data = open(make_stream(workdir, name, w, h, args), "rb").read()
    ref, _ = decode_bytes(data, "ref")
    port, _ = decode_bytes(data, "port")
    assert md5_frames(ref) == gold()[name]["md5"]
    assert [(f[0], f[1], f[2]) for f in ref] == [(f[0], f[1], f[2]) for f in port]   # FrameId, cropped size


def _oracle_decode(path, **env):
    return subprocess.run([os.path.join(ROOT, "oracle", "oracle_decode"), path, "-q"], capture_output=True, text=True,
                          env=dict(os.environ, **env), timeout=300)


@pytest.mark.parametrize("name,w,h,args", LIMITS, ids=IDS)
def test_records_keep_the_contract(workdir, name, w, h, args):
    r = _oracle_decode(make_stream(workdir, name, w, h, args), E264_CHECK_RECORDS="1")
    assert r.returncode == 0, r.stderr[-500:]


def _limits(workdir, name, w, h, args):
    r = _oracle_decode(make_stream(workdir, name, w, h, args), E264_COVERAGE="1")
    m = re.search(r"^limits (.*)$", r.stderr, re.M)
    assert r.returncode == 0 and m, r.stderr[-500:]
    f = m.group(1).split()
    return dict(zip(f[0::2], map(int, f[1::2])))


@pytest.fixture(scope="module")
def reach(workdir):
    return {s[0]: _limits(workdir, *s) for s in LIMITS}


def _bits(mask):
    return {q for q in range(64) if mask >> q & 1}


def test_limits_are_reached(reach):
    """Counted by the port on the records the parser produced from the streams above (oracle/port_recon.c)."""
    total = {k: sum(c[k] for c in reach.values()) for k in next(iter(reach.values()))}
    mask = {k: 0 for k in ("qp_y_mask", "qp_cb_mask", "qp_cr_mask")}
    for c in reach.values():
        for k in mask:
            mask[k] |= c[k]
    assert _bits(mask["qp_y_mask"]) == set(range(52)), "QP_Y values never decoded: %s" % sorted(set(range(52)) - _bits(mask["qp_y_mask"]))
    assert {0, 39} <= _bits(mask["qp_cb_mask"]) and {0, 39} <= _bits(mask["qp_cr_mask"])
    for k in ("qp_wrap_up", "qp_wrap_down", "uni_w_-128", "uni_w_127", "offset_-128", "offset_127",
              "luma_log2_wd_0", "luma_log2_wd_7", "chroma_log2_wd_0", "chroma_log2_wd_7", "bi_sum_-128", "bi_sum_128",
              "bi_sum_127_wd7", "sat_4x4", "wrap_8x8", "plane_luma_0", "plane_luma_255", "plane_chroma_0",
              "plane_chroma_255", "index_clip_0", "index_clip_51", "bi_sat16", "dc_only_wrap16"):
        assert total[k] > 0, "never reached: " + k
    for cabac, cavlc in (("lim_qp_cabac", "lim_qp_cavlc"), ("lim_levels_i_cabac", "lim_levels_i_cavlc")):
        for name in (cabac, cavlc):   # levels of 4096 and more, and at -32768 or 32767, through each entropy coder
            assert reach[name]["level_4096"] > 0 and reach[name]["level_bound"] > 0, name


@pytest.mark.gpu
@pytest.mark.parametrize("threads", [0, 2])
@pytest.mark.parametrize("name,w,h,args", LIMITS, ids=IDS)
def test_device_matches_golden_and_port(workdir, name, w, h, args, threads):
    data = open(make_stream(workdir, name, w, h, args), "rb").read()
    gpu, codes = decode_bytes(data, "gpu", threads)
    assert md5_frames(gpu) == gold()[name]["md5"]
    port, pcodes = decode_bytes(data, "port", threads)
    assert md5_frames(port) == gold()[name]["md5"] and codes == pcodes
    assert [(f[0], f[1], f[2]) for f in gpu] == [(f[0], f[1], f[2]) for f in port]


@pytest.mark.gpu
@pytest.mark.parametrize("name,w,h,args", FULL_LIMITS, ids=[s[0] for s in FULL_LIMITS])
def test_device_full_size_against_reference(workdir, name, w, h, args):
    path = make_stream(workdir, name, w, h, args)
    out = subprocess.run([os.path.join(ROOT, "tools", "b200_decode"), path, "-q"], capture_output=True, text=True, timeout=600)
    assert out.stdout.strip().splitlines()[-1] == gold()[name]["ref_summary"]
