"""The packed output (include/edge264_packed.h): every output frame cropped, as I420 or NV12, box-downscaled by 1, 2, 4
or 8 (e264_pack_kernel on the GPU).  The oracle of every case is a few lines of numpy over the frame's own full-size
samples, which other tests pin bit for bit to the reference decoder.  CPU tests run the product's host sources over the
plain-C restatement (tests/native/port_outputs_backend.c), bound into a library built here; GPU tests run the product
library."""
import ctypes, errno, os, pickle, subprocess, sys
import numpy as np
import pytest
from conftest import ROOT, STREAMS, DPB_STREAMS, make_stream
from test_robustness import CASES as DAMAGED_CASES
from api_helpers import lib_of, new_decoder, free_decoder, first_frame, loop, with_alloc_cb, _libc, _cudart, _damaged
from checkers import port_outputs_lib
import edge264_b200 as pkg
import checkers

CSRC = os.path.join(ROOT, "edge264_b200", "csrc")
I420, NV12 = pkg.PACKED_I420, pkg.PACKED_NV12
MODES = [(f, k) for f in (I420, NV12) for k in range(4)]
MODE_IDS = ["%s-k%d" % ("nv12" if f else "i420", k) for f, k in MODES]


def gen(workdir, name, w, h, args):
    return open(make_stream(workdir, name, w, h, args), "rb").read()


# ---- the definition, in numpy ----
def box(p, k):
    n = 1 << k
    h, w = p.shape
    yy = np.minimum(np.arange(-(-h // n) * n), h - 1)
    xx = np.minimum(np.arange(-(-w // n) * n), w - 1)
    s = p[yy][:, xx].astype(np.uint32).reshape(len(yy) // n, n, len(xx) // n, n).sum(axis=(1, 3))
    return ((s + (n * n >> 1)) >> (2 * k)).astype(np.uint8)


def want(w, h, i420, fmt, k):
    raw = np.frombuffer(i420, np.uint8)
    y = box(raw[:w * h].reshape(h, w), k)
    cb = box(raw[w * h:w * h * 5 // 4].reshape(h // 2, w // 2), k)
    cr = box(raw[w * h * 5 // 4:].reshape(h // 2, w // 2), k)
    assert cb.shape == (-(-y.shape[0] // 2), -(-y.shape[1] // 2))
    return {"y": y, "cbcr": np.stack([cb, cr], axis=2)} if fmt == NV12 else {"y": y, "cb": cb, "cr": cr}


def check(frames, fmt, k, label=""):
    for f in frames:
        got, exp = f[-1], want(f[1], f[2], f[3], fmt, k)
        assert got["format"] == fmt and got["log2_scale"] == k
        for name in exp:
            assert got[name].shape == exp[name].shape, "%s frame %d %s: %s, expected %s" % (label, f[0], name, got[name].shape, exp[name].shape)
            bad = np.argwhere(got[name] != exp[name])
            assert not len(bad), "%s frame %d %s: %d samples differ, first at %s" % (label, f[0], name, len(bad), bad[0])


def same_packed(a, b):
    """the same picture, wherever it lives"""
    return a.keys() == b.keys() and all(np.array_equal(a[n], b[n]) for n in a if n != "on_device")


def layout_bytes(w, h, fmt, k):
    """size of the packed buffer of a w x h cropped picture: strides rounded up to 64, planes and the whole to 256"""
    up = lambda v, a: (v + a - 1) // a * a
    n = 1 << k
    W, H, WC, HC = -(-w // n), -(-h // n), -(-(w // 2) // n), -(-(h // 2) // n)
    luma = up(up(W, 64) * H, 256)
    return luma + (up(up(2 * WC, 64) * HC, 256) if fmt == NV12 else 2 * up(up(WC, 64) * HC, 256))


# ---- 1. every format and scale on I/P/B streams ----
BASIC = [s for s in STREAMS if s[0] in ("i_cabac_8x8_dbk", "i_cavlc_slices", "p_refs_wp", "p_cavlc", "b_default", "b_cavlc_all")]
# ---- 2. sizes and cropping rectangles that stress the edges ----
EDGES = [s for s in STREAMS if s[0] in ("ragged_1x1_intra", "ragged_1xN_intra", "wide_33x2")] + [
    ("pk_9x1", 9, 1, "-n 3 -s 601 --gop I --deblock 0"),
    next(s for s in DPB_STREAMS if s[0] == "crop_rect"),                      # left 10: an odd chroma column offset
    ("pk_crop_odd_top", 5, 4, "-n 4 -s 602 --gop IPB --crop-left 6 --crop-right 2 --crop-top 10 --crop-bottom 6 --deblock 0"),
] + [("pk_crop_%d" % c, 3, 2, "-n 3 -s %d --gop IP --crop-right %d --crop-bottom %d --deblock 0" % (610 + c, c, 16 - c)) for c in range(2, 16, 2)]
P1080 = ("pk_1080p", 120, 68, "-n 2 -s 620 --gop IP --crop-bottom 8 --density 20 --deblock 0")


def run_modes(workdir, stream, backend, modes=MODES):
    name, w, h, args = stream
    data = gen(workdir, name, w, h, args)
    plain, codes = pkg.decode_bytes(data, lib_of(backend))
    for fmt, k in modes:
        frames, c = pkg.decode_bytes(data, lib_of(backend), packed=(fmt, k))
        assert c == codes and [f[:4] for f in frames] == plain
        check(frames, fmt, k, "%s %s k=%d" % (name, "nv12" if fmt else "i420", k))
        if (fmt, k) == (I420, 0):   # the copy: the bytes decode_bytes already returns
            for f in frames:
                p = f[-1]
                assert p["y"].tobytes() + p["cb"].tobytes() + p["cr"].tobytes() == f[3]
    return plain


@pytest.mark.parametrize("stream", BASIC, ids=[s[0] for s in BASIC])
def test_every_format_and_scale(workdir, stream):
    run_modes(workdir, stream, "port")


@pytest.mark.parametrize("stream", EDGES, ids=[s[0] for s in EDGES])
def test_edges_and_cropping(workdir, stream):
    plain = run_modes(workdir, stream, "port")
    if stream[0].startswith("pk_crop_") and stream[0][8:].isdigit():
        c = int(stream[0][8:])
        assert (plain[0][1], plain[0][2]) == (48 - c, 16 + c)     # 2..14 mod 16, each of them 2 mod 4 in one direction or the other


def test_1080p_with_bottom_crop(workdir):
    plain = run_modes(workdir, P1080, "port", [(NV12, 0), (NV12, 2), (I420, 3)])
    assert (plain[0][1], plain[0][2]) == (1920, 1080)


def test_oracle_is_not_a_cascade():
    """The definition rounds once: a cascade of 2x2 averages gives another answer on this block."""
    p = np.array([[1, 1, 0, 0], [0, 0, 0, 0], [1, 1, 0, 0], [0, 0, 0, 0]], np.uint8)
    assert box(p, 2)[0, 0] == 0 and box(box(p, 1), 1)[0, 0] == 1


# ---- 3. API contract ----
def test_api_errors(workdir):
    data = gen(workdir, *BASIC[0])
    buf = ctypes.create_string_buffer(data, len(data) + 64)
    lib = port_outputs_lib()
    assert lib.edge264_enable_packed(None, NV12, 0) == errno.EINVAL
    dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
    for fmt, k in ((2, 0), (-1, 0), (NV12, 4), (I420, -1)):
        assert lib.edge264_enable_packed(dec, fmt, k) == errno.EINVAL
    f = first_frame(lib, dec, data, buf)
    assert lib.edge264_get_packed(dec, ctypes.byref(f), ctypes.byref(pkg.Edge264Packed())) == errno.ENOENT
    assert lib.edge264_enable_packed(dec, NV12, 1) == errno.EBUSY
    d = ctypes.c_void_p(dec); lib.edge264_free(ctypes.byref(d))
    # enabled: a frame the application does not hold, NULL arguments
    dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
    assert lib.edge264_enable_packed(dec, NV12, 1) == 0
    f = first_frame(lib, dec, data, buf)
    p = pkg.Edge264Packed()
    assert lib.edge264_get_packed(dec, ctypes.byref(f), ctypes.byref(p)) == 0 and p.planes[2] is None and p.stride[2] == 0
    assert lib.edge264_get_packed(dec, ctypes.byref(f), None) == errno.EINVAL and lib.edge264_get_packed(None, ctypes.byref(f), ctypes.byref(p)) == errno.EINVAL
    stale = pkg.Edge264Frame()
    assert lib.edge264_get_packed(dec, ctypes.byref(stale), ctypes.byref(p)) == errno.EINVAL
    lib.edge264_return_frame(dec, f.return_arg)
    assert lib.edge264_get_packed(dec, ctypes.byref(f), ctypes.byref(p)) == errno.EINVAL
    d = ctypes.c_void_p(dec); lib.edge264_free(ctypes.byref(d))
    # a backend without it: oracle/port_backend.c
    plain = checkers.load("port")
    dec = plain.edge264_alloc(0, None, None, 0, None, None, None)
    assert plain.edge264_enable_packed(dec, NV12, 0) == errno.ENOTSUP
    d = ctypes.c_void_p(dec); plain.edge264_free(ctypes.byref(d))
    with pytest.raises(RuntimeError, match="ENOTSUP"):
        pkg.decode_bytes(data, plain, packed=(NV12, 0))


def test_ctypes_layout_and_layout_arithmetic(tmp_path):
    """The ctypes mirror matches the header; the size arithmetic of records.h matches the header's words (layout_bytes)."""
    src = tmp_path / "layout.c"
    fields = ("planes", "stride", "width", "height", "width_C", "height_C", "format", "log2_scale", "on_device")
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include <stdlib.h>\n#include "edge264_packed.h"\n#include "records.h"\n'
                   'int main(int c, char **v) { if (c == 1) { printf("%zu' + " %zu" * len(fields) + ' %d %d\\n", sizeof(Edge264Packed), '
                   + ", ".join("offsetof(Edge264Packed, %s)" % n for n in fields) + ", EDGE264_PACKED_I420, EDGE264_PACKED_NV12); return 0; }\n"
                   "E264PackedDesc k = {atoi(v[1]), atoi(v[2]), 0, 0, atoi(v[3]), atoi(v[4])}; E264PackedLayout l = e264_packed_layout(&k);\n"
                   'printf("%d %d %d %d %d\\n", l.bytes, l.width, l.height, l.width_C, l.height_C); return 0; }\n')
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-I", CSRC, str(src), "-o", exe], check=True)
    got = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    P = pkg.Edge264Packed
    assert got == [ctypes.sizeof(P)] + [getattr(P, n).offset for n in fields] + [I420, NV12]
    for w, h in ((16, 16), (38, 22), (1920, 1080), (2, 2), (7680, 4320)):
        for fmt, k in MODES:
            out = [int(x) for x in subprocess.run([exe, str(fmt), str(k), str(w), str(h)], capture_output=True, text=True, check=True).stdout.split()]
            n = 1 << k
            assert out == [layout_bytes(w, h, fmt, k), -(-w // n), -(-h // n), -(-(w // 2) // n), -(-(h // 2) // n)]
            assert out[3] == -(-out[1] // 2) and out[4] == -(-out[2] // 2)


# ---- 4. lifetime ----
BREF = ("pk_bref", 6, 5, "-n 30 -s 631 --gop IPB --bref --refs 3 --idr 17")


def test_borrowed_frames_keep_their_packed_picture(workdir):
    data = gen(workdir, *BREF)
    lib = port_outputs_lib()
    plain = {f[0]: f[-1] for f in pkg.decode_bytes(data, lib, packed=(NV12, 1))[0]}
    dec, held = new_decoder(lib, packed=(NV12, 1)), []
    loop(lib, dec, data, held.append, borrow=1)
    got = {f.FrameId: pkg.frame_packed(lib, dec, f) for f in held}     # read after everything is decoded
    for f in held:
        lib.edge264_return_frame(dec, f.return_arg)
    assert lib.edge264_get_packed(dec, ctypes.byref(held[0]), ctypes.byref(pkg.Edge264Packed())) == errno.EINVAL
    free_decoder(lib, dec)
    assert plain.keys() == got.keys() and len(plain) == 30 and all(same_packed(plain[i], got[i]) for i in plain)


def test_buffers_are_reused_when_not_borrowed(workdir):
    data = gen(workdir, *BREF)
    lib = port_outputs_lib()
    dec, ptrs = new_decoder(lib, packed=(I420, 2)), set()
    def see(f):
        p = pkg.Edge264Packed()
        assert lib.edge264_get_packed(dec, ctypes.byref(f), ctypes.byref(p)) == 0
        ptrs.add(p.planes[0])
    assert loop(lib, dec, data, see) == 30
    free_decoder(lib, dec)
    assert len(ptrs) < 30


def test_packed_output_survives_flush(workdir):
    data = gen(workdir, *BREF)
    lib = port_outputs_lib()
    fresh = [f[-1] for f in pkg.decode_bytes(data, lib, packed=(NV12, 2))[0]]
    dec, got = new_decoder(lib, packed=(NV12, 2)), []
    loop(lib, dec, data, lambda f: None, stop_after=12)
    lib.edge264_flush(dec)
    loop(lib, dec, data, lambda f: got.append(pkg.frame_packed(lib, dec, f)))
    free_decoder(lib, dec)
    assert len(got) == len(fresh) == 30 and all(same_packed(a, b) for a, b in zip(got, fresh))


def test_size_change_follows_each_frames_sps(workdir):
    a = gen(workdir, "pk_size_a", 5, 4, "-n 5 -s 641 --gop IPB --crop-right 6 --deblock 0")
    b = gen(workdir, "pk_size_b", 3, 6, "-n 5 -s 642 --gop IP --crop-left 2 --crop-bottom 10 --deblock 0")
    for fmt, k in ((NV12, 0), (I420, 1), (NV12, 3)):
        frames, _ = pkg.decode_bytes(a + b + a, port_outputs_lib(), packed=(fmt, k))
        assert [(f[1], f[2]) for f in frames] == [(74, 64)] * 5 + [(46, 86)] * 5 + [(74, 64)] * 5
        check(frames, fmt, k, "size change")


# ---- 5. alloc_cb ----
def test_alloc_cb_gets_one_more_call_per_buffer(workdir):
    name, w, h, args = BREF
    data = gen(workdir, name, w, h, args)
    lib = port_outputs_lib()
    malloc, free = _libc()
    ref = pkg.decode_bytes(data, lib, motion=True, packed=(NV12, 1))[0]
    _, off = with_alloc_cb(lib, data, malloc, free)
    on, calls = with_alloc_cb(lib, data, malloc, free, packed=(NV12, 1))
    both, calls2 = with_alloc_cb(lib, data, malloc, free, packed=(NV12, 1), motion=True)
    size = layout_bytes(16 * w, 16 * h, NV12, 1)
    assert all(m for _, m in off)                                         # sample buffers come with an mbs request
    assert calls == [c for s in off for c in (s, (size, 0))]              # then the packed buffer, mbs_size 0
    assert calls2 == [c for s in off for c in (s, (162 * w * h, 0), (size, 0))]
    for got in (on, both):
        assert [g[0] for g in got] == [f[0] for f in ref] and all(same_packed(g[3], f[-1]) for g, f in zip(got, ref))
    assert all(g[4].keys() == f[-2].keys() and all(np.array_equal(g[4][n], f[-2][n]) for n in g[4]) for g, f in zip(both, ref))


# ---- 6. parse-ahead threads ----
def test_packed_output_is_the_same_for_every_thread_count(workdir):
    data = gen(workdir, *BREF)
    runs = [pkg.decode_bytes(data, port_outputs_lib(), t, packed=(NV12, 1))[0] for t in (0, 1, 3)]
    check(runs[0], NV12, 1)
    for r in runs[1:]:
        assert [f[:4] for f in r] == [f[:4] for f in runs[0]] and all(same_packed(a[-1], b[-1]) for a, b in zip(r, runs[0]))


# ---- 7. damaged streams ----
def test_damaged_streams(workdir, monkeypatch):
    """The packed picture is a function of the samples, whatever they are; samples, error maps and return codes are those
    of a decoder without it, and the record contract holds."""
    lib = port_outputs_lib()
    monkeypatch.setenv("E264_CHECK_RECORDS", "1")
    n = 0
    for name, seed, data in _damaged(workdir, 8):
        fmt, k = MODES[(n * 3 + 1) % 8]
        on, codes_on = pkg.decode_bytes(data, lib, errors=True, packed=(fmt, k))
        off, codes_off = pkg.decode_bytes(data, lib, errors=True)
        assert lib.e264_test_record_violations() == 0, "%s seed %d: %s" % (name, seed, lib.e264_test_last_violation())
        assert codes_on == codes_off and [f[:5] for f in on] == off, "%s seed %d" % (name, seed)
        check(on, fmt, k, "%s seed %d" % (name, seed))
        n += 1
    assert n == 8 * len(DAMAGED_CASES)


# ---- 8. not enabled: nothing changes ----
def test_not_enabled_is_a_decoder_without_the_feature(workdir):
    malloc, free = _libc()
    for s in (BREF, next(s for s in DPB_STREAMS if s[0] == "crop_rect")):
        data = gen(workdir, *s)
        new, old = port_outputs_lib(), checkers.load("port")     # the second library's backend has no packed output at all
        assert pkg.decode_bytes(data, new, errors=True) == pkg.decode_bytes(data, old, errors=True)
        a, calls_new = with_alloc_cb(new, data, malloc, free)
        b, calls_old = with_alloc_cb(old, data, malloc, free)
        assert a == b and calls_new == calls_old and all(m for _, m in calls_new)


def test_libraries_export_the_packed_api():
    for path in (checkers._LIBS["gpu"], checkers._LIBS["port"]):
        lib = ctypes.CDLL(path)
        assert hasattr(lib, "edge264_enable_packed") and hasattr(lib, "edge264_get_packed"), path
    assert hasattr(ctypes.CDLL(checkers._LIBS["gpu"]), "e264b_submit_outputs")


# ---- 9. the device against numpy ----
GPU_WIDTHS = [("pk_w%d" % w, w, 2, "-n 3 -s %d --gop IPB --crop-left %d --crop-right %d --deblock 0" % (650 + w, 2 * (w % 4), 2 * (w % 5))) for w in (63, 64, 65, 127, 129)]


@pytest.mark.gpu
@pytest.mark.parametrize("stream", BASIC + EDGES + [P1080] + GPU_WIDTHS, ids=[s[0] for s in BASIC + EDGES + [P1080] + GPU_WIDTHS])
def test_device_every_format_and_scale(workdir, stream):
    run_modes(workdir, stream, "gpu")


@pytest.mark.gpu
@pytest.mark.parametrize("name,w,h", [("pk_2160p", 240, 135), ("pk_4320p", 480, 270)])
def test_device_large_pictures(workdir, name, w, h):
    run_modes(workdir, (name, w, h, "-n 1 -s 660 --gop I --density 10 --deblock 0"), "gpu", [(NV12, 0), (I420, 0), (NV12, 3), (I420, 3)])


# ---- 10. the packed picture where the samples are: device memory ----
# the samples are device memory too: only the packed picture is read (through torch)
_SUB = """
import sys, ctypes, errno, pickle
sys.path.insert(0, sys.argv[3])
import edge264_b200 as pkg
lib = pkg.load()
data = open(sys.argv[1], 'rb').read()
buf = ctypes.create_string_buffer(data, len(data) + 64); base = ctypes.addressof(buf); end = base + len(data)
dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
assert lib.edge264_enable_packed(dec, int(sys.argv[4]), int(sys.argv[5])) == 0
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
    data = gen(workdir, *next(s for s in DPB_STREAMS if s[0] == "crop_rect"))
    lib = pkg.load()
    cudart = _cudart()
    cudart.cudaMalloc.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_size_t]
    cudart.cudaFree.argtypes = [ctypes.c_void_p]
    def dmalloc(n):
        p = ctypes.c_void_p()
        assert cudart.cudaMalloc(ctypes.byref(p), n) == 0
        return p.value
    for fmt, k in ((NV12, 0), (I420, 1), (NV12, 2)):
        host = pkg.decode_bytes(data, lib, packed=(fmt, k))[0]
        check(host, fmt, k, "host mirrors")
        assert all(f[-1]["on_device"] == 0 for f in host)
        got, _ = with_alloc_cb(lib, data, dmalloc, cudart.cudaFree, packed=(fmt, k))
        assert [g[0] for g in got] == [f[0] for f in host] and all(g[3]["on_device"] == 1 and same_packed(g[3], f[-1]) for g, f in zip(got, host))
        src, out = os.path.join(workdir, "pk_dev.264"), os.path.join(workdir, "pk_dev.pkl")
        open(src, "wb").write(data)
        subprocess.run([sys.executable, "-c", _SUB, src, out, ROOT, str(fmt), str(k)], check=True, env=dict(os.environ, E264B_OUTPUT="device"), timeout=300)
        dev = pickle.load(open(out, "rb"))
        assert [f[0] for f in dev] == [f[0] for f in host] and all(a[1]["on_device"] == 1 and same_packed(a[1], b[-1]) for a, b in zip(dev, host))


# ---- 11. the device against the restatement ----
@pytest.mark.gpu
def test_device_matches_restatement_on_damaged_streams_and_with_threads(workdir):
    n = 0
    for name, seed, data in _damaged(workdir, 6):
        fmt, k = MODES[(n * 3 + 2) % 8]
        g, gc = pkg.decode_bytes(data, pkg.load(), errors=True, packed=(fmt, k))
        p, pc = pkg.decode_bytes(data, port_outputs_lib(), errors=True, packed=(fmt, k))
        assert gc == pc and [f[:5] for f in g] == [f[:5] for f in p], (name, seed)
        assert all(same_packed(a[-1], b[-1]) for a, b in zip(g, p)), (name, seed)
        n += 1
    data = gen(workdir, *BREF)
    for t in (1, 3):
        for fmt, k in ((NV12, 1), (I420, 3)):
            g = pkg.decode_bytes(data, pkg.load(), t, motion=True, packed=(fmt, k))[0]
            p = pkg.decode_bytes(data, port_outputs_lib(), t, motion=True, packed=(fmt, k))[0]
            assert [f[:4] for f in g] == [f[:4] for f in p] and all(same_packed(a[-1], b[-1]) for a, b in zip(g, p))
            assert all(np.array_equal(a[-2][m], b[-2][m]) for a, b in zip(g, p) for m in b[-2])


# ---- 12. launches and copies ----
def _stats(data, packed, touch=True):
    lib = pkg.load()
    lib.e264b_of_decoder.restype = ctypes.c_void_p; lib.e264b_of_decoder.argtypes = [ctypes.c_void_p]
    lib.e264b_stats.argtypes = [ctypes.c_void_p] + [ctypes.POINTER(ctypes.c_uint64)] * 3
    dec = new_decoder(lib, packed=packed)
    if packed is None and touch:      # refused calls leave the decoder as it was
        assert lib.edge264_enable_packed(dec, 7, 0) == errno.EINVAL
    frames = []
    loop(lib, dec, data, lambda f: frames.append(pkg._frame_bytes(f)))
    s = [ctypes.c_uint64() for _ in range(3)]
    lib.e264b_stats(lib.e264b_of_decoder(dec), *[ctypes.byref(x) for x in s])
    free_decoder(lib, dec)
    return [x.value for x in s], frames


@pytest.mark.gpu
def test_one_launch_and_the_packed_bytes_per_picture(workdir):
    name, w, h, args = "pk_stats", 20, 12, "-n 12 -s 671 --gop IPB --refs 2 --crop-right 6"
    data = gen(workdir, name, w, h, args)
    never, s_never = _stats(data, None, touch=False)
    off, s_off = _stats(data, None)
    assert off == never and s_off == s_never and len(s_off) == 12
    for fmt, k in MODES:
        on, s_on = _stats(data, (fmt, k))
        assert s_on == s_off
        assert on == [off[0] + 12, off[1], off[2] + 12 * layout_bytes(16 * w - 6, 16 * h, fmt, k)], (fmt, k)
