"""The resized output (include/edge264_packed.h, edge264_enable_resized): every output frame cropped, as I420 or NV12,
resampled to any size by exact area averaging (e264_resize_kernel on the GPU).  The oracle is a few lines of numpy over
the frame's own full-size samples, which other tests pin bit for bit to the reference decoder: the integer overlap
matrices A_v (t_h x s_h) and A_h (t_w x s_w), N = A_v P A_h^T, out = (2 N + D) // 2D.  CPU tests run the product's host
sources over the plain-C restatement (tests/native/port_outputs_backend.c), bound into a library built here; GPU tests
compare the product library with it byte for byte."""
import ctypes, errno, os, pickle, random, subprocess, sys
import numpy as np
import pytest
from conftest import ROOT, DPB_STREAMS
from test_packed_output import BASIC, EDGES, P1080, GPU_WIDTHS, BREF, gen, same_packed, layout_bytes
from api_helpers import lib_of, new_decoder, free_decoder, first_frame, loop, with_alloc_cb, _libc, _cudart, _damaged
from checkers import port_outputs_lib
import edge264_b200 as pkg
import checkers

CSRC = os.path.join(ROOT, "edge264_b200", "csrc")
I420, NV12 = pkg.PACKED_I420, pkg.PACKED_NV12


# ---- the definition, in numpy ----
def overlap(s, t):
    """A (t x s): A[x][i] = max(0, min((x + 1) s, (i + 1) t) - max(x s, i t))"""
    x, i = np.arange(t)[:, None], np.arange(s)[None, :]
    return np.maximum(0, np.minimum((x + 1) * s, (i + 1) * t) - np.maximum(x * s, i * t)).astype(np.int64)


def area(p, tw, th):
    """(2 A_v P A_h^T + D) // 2D.  The products go through float64, exact here (integers below 255 D < 2^37), so that
    they take BLAS's time rather than numpy's integer loops; the rounding is int64."""
    sh, sw = p.shape
    d = sw * sh
    n = overlap(sh, th).astype(np.float64) @ p.astype(np.float64) @ overlap(sw, tw).T.astype(np.float64)
    return ((2 * n.astype(np.int64) + d) // (2 * d)).astype(np.uint8)


def target(w, h, tw, th):
    """the size of a w x h cropped picture resized to tw x th, a 0 side following the aspect ratio"""
    side = lambda a, b, tb: min(16384, max(2, 2 * ((a * tb + b) // (2 * b))))
    return (tw or side(w, h, th)), (th or side(h, w, tw))


def want(w, h, i420, fmt, tw, th):
    tw, th = target(w, h, tw, th)
    raw = np.frombuffer(i420, np.uint8)
    y = area(raw[:w * h].reshape(h, w), tw, th)
    cb = area(raw[w * h:w * h * 5 // 4].reshape(h // 2, w // 2), tw // 2, th // 2)
    cr = area(raw[w * h * 5 // 4:].reshape(h // 2, w // 2), tw // 2, th // 2)
    return {"y": y, "cbcr": np.stack([cb, cr], axis=2)} if fmt == NV12 else {"y": y, "cb": cb, "cr": cr}


def check(frames, fmt, tw, th, label=""):
    for f in frames:
        got, exp = f[-1], want(f[1], f[2], f[3], fmt, tw, th)
        assert got["format"] == fmt and got["log2_scale"] == -1
        for name in exp:
            assert got[name].shape == exp[name].shape, "%s frame %d %s: %s, expected %s" % (label, f[0], name, got[name].shape, exp[name].shape)
            bad = np.argwhere(got[name] != exp[name])
            assert not len(bad), "%s frame %d %s: %d samples differ, first at %s" % (label, f[0], name, len(bad), bad[0])


def targets_of(w, h):
    """1280x720 and 640x360 (ratios 1.5 and 3 from 1080p), a square, the smallest, the identity, 3:1 by 2:1, one side 0"""
    return [(1280, 720), (640, 360), (224, 224), (2, 2), (w, h), (2 * max(1, round(w / 6)), 2 * max(1, round(h / 4))), (224, 0), (0, 360)]


def run_targets(workdir, stream, backend, fmts=(I420, NV12), targets=None):
    name, w, h, args = stream
    data = gen(workdir, name, w, h, args)
    plain, codes = pkg.decode_bytes(data, lib_of(backend))
    for fmt in fmts:
        for tw, th in targets or targets_of(plain[0][1], plain[0][2]):
            frames, c = pkg.decode_bytes(data, lib_of(backend), resized=(fmt, tw, th))
            assert c == codes and [f[:4] for f in frames] == plain
            check(frames, fmt, tw, th, "%s %s %dx%d" % (name, "nv12" if fmt else "i420", tw, th))
            if (fmt, tw, th) == (I420, plain[0][1], plain[0][2]):   # the identity: the bytes decode_bytes already returns
                for f in frames:
                    p = f[-1]
                    assert p["y"].tobytes() + p["cb"].tobytes() + p["cr"].tobytes() == f[3]
    return plain


# ---- 1. targets on I/P/B streams, edges, cropping ----
@pytest.mark.parametrize("stream", BASIC, ids=[s[0] for s in BASIC])
def test_every_target(workdir, stream):
    run_targets(workdir, stream, "port")


def test_1080p_targets(workdir):
    plain = run_targets(workdir, P1080, "port", targets=[(1280, 720), (640, 360), (224, 224), (640, 540), (224, 0), (0, 360)])
    assert (plain[0][1], plain[0][2]) == (1920, 1080)


@pytest.mark.parametrize("stream", EDGES, ids=[s[0] for s in EDGES])
def test_enlarging_edges_and_cropping(workdir, stream):
    run_targets(workdir, stream, "port", targets=[(224, 224), (2, 2), (38, 0), (0, 10)])


POW2 = BASIC[:1] + BASIC[-1:] + [next(s for s in EDGES if s[0] == "wide_33x2")]


def power_of_two_ratios(workdir, stream, backend):
    """Wherever the cropped size is 2^k times the target, the resized output is edge264_enable_packed(format, k)."""
    name, w, h, args = stream
    data = gen(workdir, name, w, h, args)
    lib, n = lib_of(backend), 0
    W, H = pkg.decode_bytes(data, lib)[0][0][1:3]
    for fmt in (I420, NV12):
        for k in range(4):
            if (W >> k) % 2 or (H >> k) % 2 or (W >> k) << k != W or (H >> k) << k != H:
                continue
            a = pkg.decode_bytes(data, lib, resized=(fmt, W >> k, H >> k))[0]
            b = pkg.decode_bytes(data, lib, packed=(fmt, k))[0]
            assert all(x[-1]["log2_scale"] == -1 and y[-1]["log2_scale"] == k for x, y in zip(a, b))
            assert all(all(np.array_equal(x[-1][m], y[-1][m]) for m in y[-1] if m not in ("log2_scale", "on_device")) for x, y in zip(a, b))
            n += 1
    assert n >= 4


@pytest.mark.parametrize("stream", POW2, ids=[s[0] for s in POW2])
def test_power_of_two_ratio_is_the_packed_output(workdir, stream):
    power_of_two_ratios(workdir, stream, "port")


def test_oracle_is_not_a_cascade():
    """The definition rounds once: rounding after the horizontal pass, then after the vertical one, differs here."""
    p = np.array([[0, 1, 1], [1, 2, 1], [1, 2, 2]], np.uint8)
    h = (2 * (p.astype(np.int64) @ overlap(3, 2).T) + 3) // 6
    assert area(p, 2, 2)[0, 0] == 1 and (2 * (overlap(3, 2) @ h) + 3)[0, 0] // 6 == 0


def test_rounding_helper_against_python_integers(tmp_path):
    """e264_rs_round (resize_math.cuh, compiled for the host) is floor((2N + D) / 2D) exactly: N at kD - D/2 and kD
    +- 1 around every rounding boundary, at 0 and 255 D, for D from 1 to 16368 x 16880."""
    src = tmp_path / "rs.c"
    src.write_text('#include <stdio.h>\n#include "resize_math.cuh"\nint main(void) { long long n, d;\n'
                   'while (scanf("%lld %lld", &n, &d) == 2) printf("%d\\n", e264_rs_round(n, d, e264_rs_inv(d))); return 0; }\n')
    exe = str(tmp_path / "rs")
    subprocess.run(["gcc", "-O2", "-march=x86-64-v3", "-I", CSRC, str(src), "-o", exe], check=True)
    rng = random.Random(5)
    ds = [1, 2, 3, 4, 5, 7, 1 << 20, 1920 * 1080, 960 * 540, 16368 * 16880, 16368 * 16880 - 1, 8184 * 8440, 16384 * 16384 // 2]
    ds += [rng.randrange(2, 16368 * 16880) for _ in range(40)] + [rng.randrange(1, 16368) * rng.randrange(1, 16880) for _ in range(40)]
    cases = []
    for d in ds:
        for k in range(256):
            for n in (k * d - (d + 1) // 2, k * d - d // 2, k * d - d // 2 - 1, k * d + 1, k * d - 1, k * d, k * d + d // 2, k * d + (d - 1) // 2):
                if 0 <= n <= 255 * d:
                    cases.append((n, d))
        cases += [(0, d), (255 * d, d)] + [(rng.randrange(0, 255 * d + 1), d) for _ in range(50)]
    out = subprocess.run([exe], input="".join("%d %d\n" % c for c in cases), capture_output=True, text=True, check=True).stdout.split()
    assert len(out) == len(cases)
    bad = [(n, d, int(o)) for (n, d), o in zip(cases, out) if int(o) != (2 * n + d) // (2 * d)]
    assert not bad, bad[:5]


# ---- 2. API contract ----
def test_api_errors_and_replacement(workdir):
    data = gen(workdir, *BASIC[0])
    buf = ctypes.create_string_buffer(data, len(data) + 64)
    lib = port_outputs_lib()
    assert lib.edge264_enable_resized(None, NV12, 64, 64) == errno.EINVAL
    dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
    for args in ((2, 64, 64), (-1, 64, 64), (NV12, 63, 64), (I420, 64, 35), (NV12, 0, 0), (NV12, 16386, 64), (I420, 64, 16386), (NV12, -2, 64), (NV12, 64, -2)):
        assert lib.edge264_enable_resized(dec, *args) == errno.EINVAL, args
    assert lib.edge264_enable_resized(dec, NV12, 16384, 0) == 0 and lib.edge264_enable_resized(dec, I420, 2, 16384) == 0
    f = first_frame(lib, dec, data, buf)
    assert lib.edge264_enable_resized(dec, NV12, 64, 64) == errno.EBUSY
    p = pkg.Edge264Packed()
    assert lib.edge264_get_packed(dec, ctypes.byref(f), ctypes.byref(p)) == 0
    assert (p.width, p.height, p.width_C, p.height_C, p.format, p.log2_scale) == (2, 16384, 1, 8192, I420, -1)
    free_decoder(lib, dec)
    # neither mode: ENOENT
    dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
    f = first_frame(lib, dec, data, buf)
    assert lib.edge264_get_packed(dec, ctypes.byref(f), ctypes.byref(p)) == errno.ENOENT
    free_decoder(lib, dec)
    # each replaces the other
    w, h = pkg.decode_bytes(data, lib)[0][0][1:3]
    for first, second, want_scale in (("packed", "resized", -1), ("resized", "packed", 1)):
        dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
        for mode in (first, second):
            assert (lib.edge264_enable_packed(dec, NV12, 1) if mode == "packed" else lib.edge264_enable_resized(dec, NV12, 38, 22)) == 0
        f = first_frame(lib, dec, data, buf)
        assert lib.edge264_get_packed(dec, ctypes.byref(f), ctypes.byref(p)) == 0 and p.log2_scale == want_scale
        assert (p.width, p.height) == ((38, 22) if want_scale < 0 else (w // 2, h // 2)) and p.planes[2] is None and p.stride[2] == 0
        assert p.stride[0] == (p.width + 63) // 64 * 64 and p.planes[1] - p.planes[0] == (p.stride[0] * p.height + 255) // 256 * 256
        free_decoder(lib, dec)
    # a backend without packed output: oracle/port_backend.c
    plain = checkers.load("port")
    dec = plain.edge264_alloc(0, None, None, 0, None, None, None)
    assert plain.edge264_enable_resized(dec, NV12, 64, 64) == errno.ENOTSUP
    free_decoder(plain, dec)
    with pytest.raises(RuntimeError, match="ENOTSUP"):
        pkg.decode_bytes(data, plain, resized=(NV12, 64, 64))


def resized_bytes(tw, th, fmt):
    """size of the resized buffer: the packed layout of a picture the size of the target at scale 1"""
    return layout_bytes(tw, th, fmt, 0)


# ---- 3. size changes, lifetime ----
def test_size_change(workdir):
    a = gen(workdir, "pk_size_a", 5, 4, "-n 5 -s 641 --gop IPB --crop-right 6 --deblock 0")
    b = gen(workdir, "pk_size_b", 3, 6, "-n 5 -s 642 --gop IP --crop-left 2 --crop-bottom 10 --deblock 0")
    for fmt, tw, th, shapes in ((NV12, 64, 48, [(64, 48)] * 3), (I420, 40, 0, [(40, 34), (40, 74), (40, 34)]), (NV12, 0, 30, [(34, 30), (16, 30), (34, 30)])):
        frames, _ = pkg.decode_bytes(a + b + a, port_outputs_lib(), resized=(fmt, tw, th))
        assert [(f[1], f[2]) for f in frames] == [(74, 64)] * 5 + [(46, 86)] * 5 + [(74, 64)] * 5
        assert [(f[-1]["y"].shape[1], f[-1]["y"].shape[0]) for f in frames] == [s for s in shapes for _ in range(5)]
        check(frames, fmt, tw, th, "size change")


def test_borrowed_frames_and_flush(workdir):
    data = gen(workdir, *BREF)
    lib = port_outputs_lib()
    fresh = pkg.decode_bytes(data, lib, resized=(NV12, 30, 22))[0]
    check(fresh, NV12, 30, 22)
    plain = {f[0]: f[-1] for f in fresh}
    dec, held = new_decoder(lib, resized=(NV12, 30, 22)), []
    loop(lib, dec, data, held.append, borrow=1)
    got = {f.FrameId: pkg.frame_packed(lib, dec, f) for f in held}     # read after everything is decoded
    for f in held:
        lib.edge264_return_frame(dec, f.return_arg)
    assert lib.edge264_get_packed(dec, ctypes.byref(held[0]), ctypes.byref(pkg.Edge264Packed())) == errno.EINVAL
    free_decoder(lib, dec)
    assert plain.keys() == got.keys() and len(plain) == 30 and all(same_packed(plain[i], got[i]) for i in plain)
    dec, got = new_decoder(lib, resized=(NV12, 30, 22)), []
    loop(lib, dec, data, lambda f: None, stop_after=12)
    lib.edge264_flush(dec)
    loop(lib, dec, data, lambda f: got.append(pkg.frame_packed(lib, dec, f)))
    free_decoder(lib, dec)
    assert len(got) == 30 and all(same_packed(a, b[-1]) for a, b in zip(got, fresh))


# ---- 4. alloc_cb ----
def test_alloc_cb_gets_one_more_call_per_buffer(workdir):
    name, w, h, args = BREF
    data = gen(workdir, name, w, h, args)
    lib = port_outputs_lib()
    malloc, free = _libc()
    ref = pkg.decode_bytes(data, lib, motion=True, resized=(I420, 50, 0))[0]
    _, off = with_alloc_cb(lib, data, malloc, free)
    on, calls = with_alloc_cb(lib, data, malloc, free, resized=(I420, 50, 0))
    both, calls2 = with_alloc_cb(lib, data, malloc, free, resized=(I420, 50, 0), motion=True)
    size = resized_bytes(50, 42, I420)                                    # 96x80 at the aspect ratio: 50 x 2 floor((80 * 50 + 96) / 192)
    assert ref[0][-1]["y"].shape == (42, 50)
    assert calls == [c for s in off for c in (s, (size, 0))]
    assert calls2 == [c for s in off for c in (s, (162 * w * h, 0), (size, 0))]
    for got in (on, both):
        assert [g[0] for g in got] == [f[0] for f in ref] and all(same_packed(g[3], f[-1]) for g, f in zip(got, ref))
    assert all(all(np.array_equal(g[4][n], f[-2][n]) for n in g[4]) for g, f in zip(both, ref))


# ---- 5. threads, damaged streams, off ----
def test_resized_output_is_the_same_for_every_thread_count(workdir):
    data = gen(workdir, *BREF)
    runs = [pkg.decode_bytes(data, port_outputs_lib(), t, resized=(NV12, 38, 26))[0] for t in (0, 1, 3)]
    check(runs[0], NV12, 38, 26)
    for r in runs[1:]:
        assert [f[:4] for f in r] == [f[:4] for f in runs[0]] and all(same_packed(a[-1], b[-1]) for a, b in zip(r, runs[0]))


DAMAGED_TARGETS = [(I420, 22, 14), (NV12, 224, 224), (NV12, 0, 10), (I420, 6, 0)]


def test_damaged_streams(workdir, monkeypatch):
    """The resized picture is a function of the samples, whatever they are; samples, error maps and return codes are
    those of a decoder without it, and the record contract holds."""
    lib = port_outputs_lib()
    monkeypatch.setenv("E264_CHECK_RECORDS", "1")
    for n, (name, seed, data) in enumerate(_damaged(workdir, 4)):
        fmt, tw, th = DAMAGED_TARGETS[n % 4]
        on, codes_on = pkg.decode_bytes(data, lib, errors=True, resized=(fmt, tw, th))
        off, codes_off = pkg.decode_bytes(data, lib, errors=True)
        assert lib.e264_test_record_violations() == 0, "%s seed %d: %s" % (name, seed, lib.e264_test_last_violation())
        assert codes_on == codes_off and [f[:5] for f in on] == off, "%s seed %d" % (name, seed)
        check(on, fmt, tw, th, "%s seed %d" % (name, seed))


def test_not_enabled_is_a_decoder_without_the_feature(workdir):
    malloc, free = _libc()
    for s in (BREF, next(s for s in DPB_STREAMS if s[0] == "crop_rect")):
        data = gen(workdir, *s)
        new, old = port_outputs_lib(), checkers.load("port")
        assert pkg.decode_bytes(data, new, errors=True) == pkg.decode_bytes(data, old, errors=True)
        a, calls_new = with_alloc_cb(new, data, malloc, free)
        b, calls_old = with_alloc_cb(old, data, malloc, free)
        assert a == b and calls_new == calls_old


def test_libraries_export_the_resized_api():
    for path in (checkers._LIBS["gpu"], checkers._LIBS["port"]):
        assert hasattr(ctypes.CDLL(path), "edge264_enable_resized"), path


# ---- 6. the device against the restatement ----
def same_as_restatement(data, fmt, tw, th, n_threads=0, label=""):
    g, gc = pkg.decode_bytes(data, pkg.load(), n_threads, errors=True, resized=(fmt, tw, th))
    p, pc = pkg.decode_bytes(data, port_outputs_lib(), n_threads, errors=True, resized=(fmt, tw, th))
    assert gc == pc and [f[:5] for f in g] == [f[:5] for f in p], label
    for a, b in zip(g, p):
        assert a[-1]["format"] == b[-1]["format"] == fmt and a[-1]["log2_scale"] == b[-1]["log2_scale"] == -1, label
        for m in ("y", "cb", "cr", "cbcr"):
            if m in b[-1]:
                assert a[-1][m].shape == b[-1][m].shape, (label, m)
                bad = np.argwhere(a[-1][m] != b[-1][m])
                assert not len(bad), "%s frame %d %s: %d samples differ, first at %s" % (label, a[0], m, len(bad), bad[0])
    return g


@pytest.mark.gpu
@pytest.mark.parametrize("stream", BASIC + EDGES + [P1080] + GPU_WIDTHS, ids=[s[0] for s in BASIC + EDGES + [P1080] + GPU_WIDTHS])
def test_device_every_target(workdir, stream):
    name, w, h, args = stream
    data = gen(workdir, name, w, h, args)
    W, H = pkg.decode_bytes(data, pkg.load())[0][0][1:3]
    for i, (tw, th) in enumerate(targets_of(W, H)):
        fmt = (I420, NV12)[i % 2]
        check(same_as_restatement(data, fmt, tw, th, label="%s %dx%d" % (name, tw, th)), fmt, tw, th, "%s %dx%d" % (name, tw, th))


@pytest.mark.gpu
@pytest.mark.parametrize("name,w,h,crop,targets", [("rs_2160p", 240, 135, "", [(1280, 720), (224, 224)]), ("rs_4320p", 480, 270, "", [(1920, 1080), (2, 2)]),
                                                   ("rs_16x16", 1, 1, "", [(2048, 2048)]), ("rs_wide", 1023, 1, "", [(2, 2), (2, 16384)]),
                                                   ("rs_2x2", 1, 1, " --crop-right 14 --crop-bottom 14", [(16384, 2), (2, 16384), (16384, 6)])])
def test_device_large_and_extreme_ratios(workdir, name, w, h, crop, targets):
    """4K and 8K pictures; enlarging 16x16 to 2048x2048; 16368 -> 2 and 2 -> 16384, with a different ratio on each axis"""
    data = gen(workdir, name, w, h, "-n 1 -s 660 --gop I --density 10 --deblock 0" + crop)
    for i, (tw, th) in enumerate(targets):
        same_as_restatement(data, (NV12, I420)[i % 2], tw, th, label="%s %dx%d" % (name, tw, th))


@pytest.mark.gpu
@pytest.mark.parametrize("stream", POW2, ids=[s[0] for s in POW2])
def test_device_power_of_two_ratio_is_the_packed_output(workdir, stream):
    power_of_two_ratios(workdir, stream, "gpu")


# the samples are device memory too: only the resized picture is read (through torch)
_SUB = """
import sys, ctypes, errno, pickle
sys.path.insert(0, sys.argv[3])
import edge264_b200 as pkg
lib = pkg.load()
data = open(sys.argv[1], 'rb').read()
buf = ctypes.create_string_buffer(data, len(data) + 64); base = ctypes.addressof(buf); end = base + len(data)
dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
assert lib.edge264_enable_resized(dec, int(sys.argv[4]), int(sys.argv[5]), int(sys.argv[6])) == 0
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
    for fmt, tw, th in ((NV12, 40, 30), (I420, 0, 24)):
        host = pkg.decode_bytes(data, lib, resized=(fmt, tw, th))[0]
        check(host, fmt, tw, th, "host mirrors")
        assert all(f[-1]["on_device"] == 0 for f in host)
        got, _ = with_alloc_cb(lib, data, dmalloc, cudart.cudaFree, resized=(fmt, tw, th))
        assert [g[0] for g in got] == [f[0] for f in host] and all(g[3]["on_device"] == 1 and same_packed(g[3], f[-1]) for g, f in zip(got, host))
        src, out = os.path.join(workdir, "rs_dev.264"), os.path.join(workdir, "rs_dev.pkl")
        open(src, "wb").write(data)
        subprocess.run([sys.executable, "-c", _SUB, src, out, ROOT, str(fmt), str(tw), str(th)], check=True, env=dict(os.environ, E264B_OUTPUT="device"), timeout=300)
        dev = pickle.load(open(out, "rb"))
        assert [f[0] for f in dev] == [f[0] for f in host] and all(a[1]["on_device"] == 1 and same_packed(a[1], b[-1]) for a, b in zip(dev, host))


@pytest.mark.gpu
def test_device_matches_restatement_on_damaged_streams_and_with_threads(workdir):
    for n, (name, seed, data) in enumerate(_damaged(workdir, 4)):
        fmt, tw, th = DAMAGED_TARGETS[(n + 1) % 4]
        same_as_restatement(data, fmt, tw, th, label="%s seed %d" % (name, seed))
    data = gen(workdir, *BREF)
    for t in (1, 3):
        for fmt, tw, th in ((NV12, 38, 26), (I420, 0, 100)):
            g = pkg.decode_bytes(data, pkg.load(), t, motion=True, resized=(fmt, tw, th))[0]
            p = pkg.decode_bytes(data, port_outputs_lib(), t, motion=True, resized=(fmt, tw, th))[0]
            assert [f[:4] for f in g] == [f[:4] for f in p] and all(same_packed(a[-1], b[-1]) for a, b in zip(g, p))
            assert all(np.array_equal(a[-2][m], b[-2][m]) for a, b in zip(g, p) for m in b[-2])


# ---- 7. launches and copies ----
def _stats(data, resized):
    lib = pkg.load()
    lib.e264b_of_decoder.restype = ctypes.c_void_p; lib.e264b_of_decoder.argtypes = [ctypes.c_void_p]
    lib.e264b_stats.argtypes = [ctypes.c_void_p] + [ctypes.POINTER(ctypes.c_uint64)] * 3
    dec = new_decoder(lib, resized=resized)
    frames = []
    loop(lib, dec, data, lambda f: frames.append(pkg._frame_bytes(f)))
    s = [ctypes.c_uint64() for _ in range(3)]
    lib.e264b_stats(lib.e264b_of_decoder(dec), *[ctypes.byref(x) for x in s])
    free_decoder(lib, dec)
    return [x.value for x in s], frames


@pytest.mark.gpu
def test_one_launch_and_the_resized_bytes_per_picture(workdir):
    data = gen(workdir, "rs_stats", 20, 12, "-n 12 -s 671 --gop IPB --refs 2 --crop-right 6")
    off, s_off = _stats(data, None)
    assert len(s_off) == 12
    for fmt, tw, th in ((NV12, 224, 224), (I420, 1280, 720), (NV12, 0, 64)):
        on, s_on = _stats(data, (fmt, tw, th))
        tw, th = target(16 * 20 - 6, 16 * 12, tw, th)
        assert s_on == s_off
        assert on == [off[0] + 12, off[1], off[2] + 12 * resized_bytes(tw, th, fmt)], (fmt, tw, th)
