"""Picture statistics (include/edge264_picstats.h): each output frame's histograms over the cropped planes, and the sums and
sums of squares of every coded macroblock (e264_picstats_kernel on the GPU).  The oracle is numpy over the frame's coded
planes, read through Edge264Frame.samples[], frame_crop_offsets and the strides with ctypes (not through the cropped bytes
decode_bytes returns), which other tests pin bit for bit to the reference decoder.  CPU tests run the product's host
sources over the plain-C restatement (tests/native/port_outputs_backend.c), bound into a library built here; GPU tests
compare the product library with it byte for byte."""
import ctypes, errno, os, pickle, subprocess, sys, threading
import numpy as np
import pytest
from conftest import ROOT, STREAMS, DPB_STREAMS, make_stream
from test_limits import LIMITS
from test_packed_output import BREF, P1080
from test_luma_only import STORED
from api_helpers import new_decoder, free_decoder, first_frame, loop, with_alloc_cb, _libc, _ALLOC, _FREE, _cudart, _damaged
from checkers import port_outputs_lib
import edge264_b200 as pkg
import checkers
sys.path.insert(0, os.path.join(ROOT, "tools"))
from picstats_cost import constant_stream   # noqa: E402

CSRC = os.path.join(ROOT, "edge264_b200", "csrc")


def _data(workdir, s):
    return open(make_stream(workdir, *s) if isinstance(s, tuple) else s, "rb").read()


def _id(s):
    return s[0] if isinstance(s, tuple) else os.path.basename(s)


# ---- the definition, in numpy ----
def coded_planes(f):
    """The coded Y, Cb, Cr planes of a frame in host memory, from samples[], frame_crop_offsets and the strides."""
    top, right, bottom, left = f.frame_crop_offsets
    w, h = f.width_Y + left + right, f.height_Y + top + bottom
    y0 = ctypes.cast(f.samples[0], ctypes.c_void_p).value - top * f.stride_Y - left
    c0 = ctypes.cast(f.samples[1], ctypes.c_void_p).value - (top >> 1) * f.stride_C - (left >> 1)
    assert ctypes.cast(f.samples[2], ctypes.c_void_p).value - ctypes.cast(f.samples[1], ctypes.c_void_p).value == f.stride_C >> 1
    Y = np.frombuffer(ctypes.string_at(y0, (h - 1) * f.stride_Y + w), np.uint8)
    C = np.frombuffer(ctypes.string_at(c0, (h // 2 - 1) * f.stride_C + (f.stride_C >> 1) + w // 2), np.uint8)
    rows = lambda a, base, n, width, stride: np.stack([a[base + j * stride:base + j * stride + width] for j in range(n)])
    return rows(Y, 0, h, w, f.stride_Y), rows(C, 0, h // 2, w // 2, f.stride_C), rows(C, f.stride_C >> 1, h // 2, w // 2, f.stride_C)


def oracle(f):
    top, right, bottom, left = f.frame_crop_offsets
    out = {"hist": np.zeros((3, 256), np.uint32)}
    sums, sqs = [], []
    for p, P in enumerate(coded_planes(f)):
        n, s = (8, 1) if p else (16, 0)
        H, W = P.shape[0] // n, P.shape[1] // n
        v = P.astype(np.int64)
        sums.append(v.reshape(H, n, W, n).sum(axis=(1, 3)))
        sqs.append((v * v).reshape(H, n, W, n).sum(axis=(1, 3)))
        crop = P[top >> s:P.shape[0] - (bottom >> s), left >> s:P.shape[1] - (right >> s)]
        assert crop.shape == ((f.height_C, f.width_C) if p else (f.height_Y, f.width_Y))
        out["hist"][p] = np.bincount(crop.ravel(), minlength=256)
    out["sum"], out["sum_sq"] = np.stack(sums).astype(np.uint32), np.stack(sqs).astype(np.uint32)
    return out


def same_stats(a, b):
    return all(np.array_equal(a[k], b[k]) for k in ("hist", "sum", "sum_sq"))


def check(got, f, want, label):
    """got: frame_picstats of frame f; want: the oracle; and the header's two invariants"""
    for k in ("hist", "sum", "sum_sq"):
        assert got[k].shape == want[k].shape and got[k].dtype == np.uint32, "%s frame %d %s: %s" % (label, f.FrameId, k, got[k].shape)
        bad = np.argwhere(got[k] != want[k])
        assert not len(bad), "%s frame %d %s: %d values differ, first at %s" % (label, f.FrameId, k, len(bad), bad[0])
    assert [int(got["hist"][p].sum()) for p in range(3)] == [f.width_Y * f.height_Y] + [f.width_C * f.height_C] * 2, label
    if not any(f.frame_crop_offsets):
        assert int((np.arange(256) * got["hist"][0].astype(np.int64)).sum()) == int(got["sum"][0].astype(np.int64).sum()), label


def run(lib, data, label="", with_oracle=True, **kw):
    """Decode with the statistics on; every frame checked against the oracle (host memory).  Returns
    [(FrameId, stats)]."""
    dec, out = new_decoder(lib, picstats=True, **kw), []
    def see(f):
        got = pkg.frame_picstats(lib, dec, f)
        if with_oracle:
            check(got, f, oracle(f), label)
        out.append((f.FrameId, got))
    loop(lib, dec, data, see)
    free_decoder(lib, dec)
    return out


def same_runs(a, b, label=""):
    assert [x[0] for x in a] == [x[0] for x in b], label
    for x, y in zip(a, b):
        for k in ("hist", "sum", "sum_sq"):
            bad = np.argwhere(x[1][k] != y[1][k])
            assert not len(bad), "%s frame %d %s: %d values differ, first at %s" % (label, x[0], k, len(bad), bad[0])


GENERATED = STREAMS + DPB_STREAMS
ALL = GENERATED + LIMITS + STORED
IDS = [_id(s) for s in ALL]


# ---- 1. CPU: the restatement against numpy ----
@pytest.mark.parametrize("stream", ALL, ids=IDS)
def test_port_matches_the_definition_with_every_thread_count(workdir, stream):
    data, lib = _data(workdir, stream), port_outputs_lib()
    runs = [sorted(run(lib, data, "%s t%d" % (_id(stream), t), n_threads=t), key=lambda x: x[0]) for t in (0, 1, 3)]   # by FrameId: the
    assert runs[0]                                                                                                         # output order may differ
    same_runs(runs[0], runs[1], _id(stream)); same_runs(runs[0], runs[2], _id(stream))


def test_streams_cover_cropping_and_shapes(workdir):
    """crop_rect crops all four sides, inside macroblocks; zero-cropping.264, wide_256x2 and ragged_1x1_intra are there."""
    ids = set(IDS)
    assert {"crop_rect", "wide_256x2", "ragged_1x1_intra", "zero-cropping.264"} <= ids and len(STORED) >= 7
    lib, seen = port_outputs_lib(), []
    dec = new_decoder(lib, picstats=True)
    loop(lib, dec, _data(workdir, next(s for s in DPB_STREAMS if s[0] == "crop_rect")), lambda f: seen.append(tuple(f.frame_crop_offsets)))
    free_decoder(lib, dec)
    assert set(seen) == {(8, 6, 4, 10)}


def test_every_other_output_is_unchanged(workdir):
    """Samples, FrameIds, return codes, error maps, motion export, packed and resized output equal a decode without it."""
    lib = port_outputs_lib()
    for s in (BREF, next(x for x in DPB_STREAMS if x[0] == "crop_rect"), next(x for x in STREAMS if x[0] == "b_explicit")):
        data = _data(workdir, s)
        for t in (0, 3):
            for kw in ({"packed": (pkg.PACKED_NV12, 1)}, {"resized": (pkg.PACKED_I420, 40, 26)}, {}):
                off, codes_off = pkg.decode_bytes(data, lib, t, errors=True, motion=True, **kw)
                on, codes_on = pkg.decode_bytes(data, lib, t, errors=True, motion=True, picstats=True, **kw)
                assert codes_on == codes_off and len(on) == len(off), s[0]
                for a, b in zip(on, off):
                    assert len(a) == len(b) + 1 and a[:5] == b[:5], (s[0], kw)
                    assert all(x.keys() == y.keys() and all(np.array_equal(x[k], y[k]) for k in x) for x, y in zip(a[5:-1], b[5:])), (s[0], kw)
                    assert a[-1].keys() == {"hist", "sum", "sum_sq", "on_device"}


@pytest.mark.parametrize("stream", GENERATED, ids=[s[0] for s in GENERATED])
def test_luma_only(workdir, stream):
    """Luma statistics equal the full decode's; chroma is a plane of 128."""
    data, lib, s = _data(workdir, stream), port_outputs_lib(), stream[0]
    full, luma = run(lib, data, s), run(lib, data, s + " luma", luma_only=True)
    assert [x[0] for x in full] == [x[0] for x in luma]
    dec = new_decoder(lib, picstats=True, luma_only=True)
    sizes = []
    loop(lib, dec, data, lambda f: sizes.append(f.width_C * f.height_C))
    free_decoder(lib, dec)
    for (i, a), (_, b), n in zip(full, luma, sizes):
        assert np.array_equal(a["hist"][0], b["hist"][0]) and np.array_equal(a["sum"][0], b["sum"][0]) and np.array_equal(a["sum_sq"][0], b["sum_sq"][0]), (s, i)
        want = np.zeros(256, np.uint32); want[128] = n
        assert all(np.array_equal(b["hist"][p], want) for p in (1, 2)), (s, i)
        assert (b["sum"][1:] == 8192).all() and (b["sum_sq"][1:] == 1048576).all(), (s, i)


@pytest.mark.parametrize("skip", [pkg.SKIP_NONREF, pkg.SKIP_NONKEY], ids=["nonref", "nonkey"])
def test_skip_modes(workdir, skip):
    """Each output frame's statistics are those of the same FrameId in the full decode."""
    lib, n = port_outputs_lib(), 0
    for s in GENERATED:
        data = _data(workdir, s)
        full = dict((i, st) for i, st in run(lib, data, s[0]))
        for i, st in run(lib, data, s[0] + " skip", skip=skip):
            assert same_stats(st, full[i]), (s[0], i)
            n += 1
    assert n


# ---- 2. lifetimes and buffers ----
def test_borrowed_frames_and_flush(workdir):
    data = _data(workdir, BREF)
    lib = port_outputs_lib()
    order = run(lib, data, "bref")
    fresh = dict(order)
    dec, held = new_decoder(lib, picstats=True), []
    loop(lib, dec, data, held.append, borrow=1)
    got = {f.FrameId: pkg.frame_picstats(lib, dec, f) for f in held}   # read after everything is decoded
    for f in held:
        lib.edge264_return_frame(dec, f.return_arg)
    assert lib.edge264_get_picstats(dec, ctypes.byref(held[0]), ctypes.byref(pkg.Edge264PicStats())) == errno.EINVAL
    free_decoder(lib, dec)
    assert got.keys() == fresh.keys() and len(got) == 30 and all(same_stats(got[i], fresh[i]) for i in got)
    dec, after = new_decoder(lib, picstats=True), []
    loop(lib, dec, data, lambda f: None, stop_after=12)
    lib.edge264_flush(dec)
    loop(lib, dec, data, lambda f: after.append((f.FrameId, pkg.frame_picstats(lib, dec, f))))
    free_decoder(lib, dec)
    assert len(after) == 30 and all(same_stats(a[1], b[1]) for a, b in zip(after, order))   # FrameIds go on counting after a flush


def test_size_change(workdir):
    a = _data(workdir, ("pk_size_a", 5, 4, "-n 5 -s 641 --gop IPB --crop-right 6 --deblock 0"))
    b = _data(workdir, ("pk_size_b", 3, 6, "-n 5 -s 642 --gop IP --crop-left 2 --crop-bottom 10 --deblock 0"))
    got = run(port_outputs_lib(), a + b + a, "size change")
    assert [st["sum"].shape for _, st in got] == [(3, 4, 5)] * 5 + [(3, 6, 3)] * 5 + [(3, 4, 5)] * 5


def test_alloc_cb_gets_one_more_call_per_buffer(workdir):
    name, w, h, args = BREF
    data = _data(workdir, BREF)
    lib = port_outputs_lib()
    malloc, free = _libc()
    ref = run(lib, data, "bref")
    _, off = with_alloc_cb(lib, data, malloc, free, picstats=False)
    on, calls = with_alloc_cb(lib, data, malloc, free, picstats=True)
    both, calls2 = with_alloc_cb(lib, data, malloc, free, picstats=True, motion=True)
    size = 3072 + 24 * w * h
    assert all(m for _, m in off)
    assert calls == [c for s in off for c in (s, (size, 0))]
    assert calls2 == [c for s in off for c in (s, (162 * w * h, 0), (size, 0))]
    for got in (on, both):
        same_runs([(g[0], g[5]) for g in got], ref, "alloc_cb")


def test_alloc_cb_order_with_packed_output(workdir):
    """The statistics' buffer is asked for after the packed one."""
    name, w, h, args = BREF
    data = _data(workdir, BREF)
    lib = port_outputs_lib()
    malloc, free = _libc()
    live, calls = set(), []
    def alloc(samples, size, mbs, mbs_size, err, arg):
        p = malloc(size); live.add(p); calls.append((size, mbs_size)); samples[0] = p
    def release(samples, mbs, arg):
        live.remove(samples); free(samples)
    cbs = (_ALLOC(alloc), _FREE(release))
    dec = new_decoder(lib, picstats=True, alloc=cbs)
    assert lib.edge264_enable_packed(dec, pkg.PACKED_NV12, 3) == 0
    loop(lib, dec, data, lambda f: None)
    free_decoder(lib, dec)
    assert not live and len(calls) % 3 == 0 and calls[2::3] == [(3072 + 24 * w * h, 0)] * (len(calls) // 3)
    assert all(m == 0 for _, m in calls[1::3]) and all(m for _, m in calls[0::3])


# ---- 3. damaged streams ----
def test_damaged_streams(workdir, monkeypatch):
    """The statistics are a function of the samples, whatever they are; samples, error maps and return codes are those of
    a decoder without them, and the record contract holds."""
    lib = port_outputs_lib()
    monkeypatch.setenv("E264_CHECK_RECORDS", "1")
    n = 0
    for name, seed, data in _damaged(workdir, 8):
        on, codes_on = pkg.decode_bytes(data, lib, errors=True, picstats=True)
        off, codes_off = pkg.decode_bytes(data, lib, errors=True)
        assert lib.e264_test_record_violations() == 0, "%s seed %d: %s" % (name, seed, lib.e264_test_last_violation())
        assert codes_on == codes_off and [f[:5] for f in on] == off, "%s seed %d" % (name, seed)
        run(lib, data, "%s seed %d" % (name, seed))
        n += 1
    assert n >= 16


# ---- 4. API ----
def test_api_codes(workdir):
    data = _data(workdir, STREAMS[0])
    buf = ctypes.create_string_buffer(data, len(data) + 64)
    lib = port_outputs_lib()
    assert lib.edge264_enable_picstats(None) == errno.EINVAL
    dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
    f = first_frame(lib, dec, data, buf)
    s = pkg.Edge264PicStats()
    assert lib.edge264_get_picstats(dec, ctypes.byref(f), ctypes.byref(s)) == errno.ENOENT
    assert lib.edge264_enable_picstats(dec) == errno.EBUSY
    free_decoder(lib, dec)
    dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
    assert lib.edge264_enable_picstats(dec) == 0 and lib.edge264_enable_picstats(dec) == 0
    f = first_frame(lib, dec, data, buf)
    assert lib.edge264_get_picstats(dec, ctypes.byref(f), ctypes.byref(s)) == 0 and (s.width_mbs, s.height_mbs, s.on_device) == (6, 5, 0)
    assert lib.edge264_get_picstats(dec, ctypes.byref(f), None) == errno.EINVAL and lib.edge264_get_picstats(None, ctypes.byref(f), ctypes.byref(s)) == errno.EINVAL
    assert lib.edge264_get_picstats(dec, ctypes.byref(pkg.Edge264Frame()), ctypes.byref(s)) == errno.EINVAL
    lib.edge264_return_frame(dec, f.return_arg)
    assert lib.edge264_get_picstats(dec, ctypes.byref(f), ctypes.byref(s)) == errno.EINVAL   # no longer held
    free_decoder(lib, dec)
    # a backend without submit_outputs
    plain = checkers.load("port")
    dec = plain.edge264_alloc(0, None, None, 0, None, None, None)
    assert plain.edge264_enable_picstats(dec) == errno.ENOTSUP
    free_decoder(plain, dec)
    with pytest.raises(RuntimeError, match="ENOTSUP"):
        pkg.decode_bytes(data, plain, picstats=True)


def test_ctypes_layout_and_offsets(tmp_path):
    """The ctypes mirror matches the header; records.h's offsets are the header's words."""
    src = tmp_path / "layout.c"
    fields = ("hist", "sum", "sum_sq", "width_mbs", "height_mbs", "on_device")
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "edge264_picstats.h"\n#include "records.h"\n'
                   'int main(void) { printf("%zu' + " %zu" * len(fields) + ' %d %d %zu %zu\\n", sizeof(Edge264PicStats), '
                   + ", ".join("offsetof(Edge264PicStats, %s)" % n for n in fields)
                   + ", E264_PICSTATS_HIST, E264_PICSTATS_SUM, E264_PICSTATS_SUM_SQ(8160), E264_PICSTATS_BYTES(8160)); return 0; }\n")
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-I", CSRC, str(src), "-o", exe], check=True)
    got = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    P = pkg.Edge264PicStats
    assert got == [ctypes.sizeof(P)] + [getattr(P, n).offset for n in fields] + [0, 3072, 3072 + 12 * 8160, 3072 + 24 * 8160]


def test_not_enabled_is_a_decoder_without_the_feature(workdir):
    malloc, free = _libc()
    for s in (BREF, next(x for x in DPB_STREAMS if x[0] == "crop_rect")):
        data = _data(workdir, s)
        new, old = port_outputs_lib(), checkers.load("port")
        assert pkg.decode_bytes(data, new, errors=True) == pkg.decode_bytes(data, old, errors=True)
        a, calls_new = with_alloc_cb(new, data, malloc, free, picstats=False)
        b, calls_old = with_alloc_cb(old, data, malloc, free, picstats=False)
        assert a == b and calls_new == calls_old


# ---- 5. the device against the restatement ----
CONSTANT = [(20, 12, 4, 200), (120, 68, 8, 16)]   # width_mbs, height_mbs, crop_bottom, value
LARGE = [("ps_1088p", 120, 68, "-n 2 -s 682 --gop IP --density 20 --deblock 0"), P1080,
         ("pk_2160p", 240, 135, "-n 1 -s 660 --gop I --density 10 --deblock 0"), ("pk_4320p", 480, 270, "-n 1 -s 660 --gop I --density 10 --deblock 0")]


def same_as_restatement(data, label, n_threads=0, **kw):
    g = run(pkg.load(), data, label + " gpu", n_threads=n_threads, **kw)
    p = run(port_outputs_lib(), data, label + " port", n_threads=n_threads, **kw)
    same_runs(g, p, label)
    for _, st in g:
        assert st["on_device"] == 0
    return g


@pytest.mark.gpu
@pytest.mark.parametrize("stream", ALL, ids=IDS)
def test_device_matches_restatement(workdir, stream):
    data = _data(workdir, stream)
    for t in (0, 3):
        same_as_restatement(data, "%s t%d" % (_id(stream), t), t)
    same_as_restatement(data, _id(stream) + " luma", luma_only=True)


def test_constant_stream_decodes_to_constant_planes():
    lib = port_outputs_lib()
    for w, h, crop, v in CONSTANT:
        for luma_only in (False, True):
            frames, codes = pkg.decode_bytes(constant_stream(w, h, 3, v, crop), lib, luma_only=luma_only, picstats=True)
            n = 16 * w * (16 * h - crop)
            assert len(frames) == 3 and all(f[3] == bytes([v]) * n + bytes([128 if luma_only else v]) * (n // 2) for f in frames)
            for f in frames:
                assert f[-1]["hist"][0][v] == n and (f[-1]["sum"][0] == 256 * v).all() and (f[-1]["sum_sq"][0] == 256 * v * v).all()


@pytest.mark.gpu
def test_device_constant_picture():
    """Every sample of a plane is the same value, the histogram's worst case; luma-only too (chroma 128)."""
    for w, h, crop, v in CONSTANT:
        data = constant_stream(w, h, 4, v, crop)
        for kw in ({}, {"luma_only": True}):
            for _, st in same_as_restatement(data, "constant %dx%d %s" % (w, h, kw), **kw):
                assert all(np.count_nonzero(st["hist"][p]) == 1 for p in range(3)), kw


@pytest.mark.gpu
@pytest.mark.parametrize("stream", LARGE, ids=[s[0] for s in LARGE])
def test_device_full_size(workdir, stream):
    same_as_restatement(_data(workdir, stream), stream[0])


@pytest.mark.gpu
def test_device_damaged_streams(workdir):
    for name, seed, data in _damaged(workdir, 6):
        same_as_restatement(data, "%s seed %d" % (name, seed))
        same_as_restatement(data, "%s seed %d luma" % (name, seed), luma_only=True)


@pytest.mark.gpu
def test_device_decoders_in_parallel(workdir):
    """Decoders on 8 host threads at once, every other one luma-only, match the restatement."""
    streams = [s for s in GENERATED if s[0] in ("crop_rect", "b_explicit", "pb_intra_heavy", "wide_33x2", "bref_spatial", "p_refs_wp", "ps_update", "b_cavlc_all")]
    datas = [_data(workdir, s) for s in streams]
    want = [run(port_outputs_lib(), d, s[0], luma_only=bool(i % 2)) for i, (s, d) in enumerate(zip(streams, datas))]
    got, errs = [None] * len(datas), []
    def work(i):
        try:
            got[i] = run(pkg.load(), datas[i], streams[i][0], with_oracle=False, luma_only=bool(i % 2))
        except Exception as e:   # reported below
            errs.append(e)
    th = [threading.Thread(target=work, args=(i,)) for i in range(len(datas))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs
    for s, a, b in zip(streams, got, want):
        same_runs(a, b, s[0])


# the samples are device memory too: only the statistics are read (through torch)
_SUB = """
import sys, ctypes, errno, pickle
sys.path.insert(0, sys.argv[3])
import edge264_b200 as pkg
lib = pkg.load()
data = open(sys.argv[1], 'rb').read()
buf = ctypes.create_string_buffer(data, len(data) + 64); base = ctypes.addressof(buf); end = base + len(data)
dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
assert lib.edge264_enable_picstats(dec) == 0
nal, out, f = base + 3 + (1 if data[2] == 0 else 0), [], pkg.Edge264Frame()
while True:
    sc = lib.edge264_find_start_code(nal, end, 0) if nal < end else end
    res = lib.edge264_decode_NAL(dec, nal, sc, None, None)
    while lib.edge264_get_frame(dec, ctypes.byref(f), 0) == 0:
        out.append((f.FrameId, pkg.frame_picstats(lib, dec, f)))
    if res == errno.ENOBUFS:
        continue
    if nal >= end:
        break
    nal = sc + 3 if sc + 3 < end else end
pickle.dump(out, open(sys.argv[2], 'wb'))
"""


@pytest.mark.gpu
def test_device_memory_output(workdir):
    data = _data(workdir, next(s for s in DPB_STREAMS if s[0] == "crop_rect"))
    host = run(pkg.load(), data, "host")
    cudart = _cudart()
    cudart.cudaMalloc.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_size_t]
    cudart.cudaFree.argtypes = [ctypes.c_void_p]
    def dmalloc(n):
        p = ctypes.c_void_p()
        assert cudart.cudaMalloc(ctypes.byref(p), n) == 0
        return p.value
    got = [(g[0], g[5]) for g in with_alloc_cb(pkg.load(), data, dmalloc, cudart.cudaFree, picstats=True)[0]]
    assert all(st["on_device"] == 1 for _, st in got)
    same_runs(got, host, "alloc_cb device memory")
    src, out = os.path.join(workdir, "ps_dev.264"), os.path.join(workdir, "ps_dev.pkl")
    open(src, "wb").write(data)
    subprocess.run([sys.executable, "-c", _SUB, src, out, ROOT], check=True, env=dict(os.environ, E264B_OUTPUT="device"), timeout=300)
    dev = pickle.load(open(out, "rb"))
    assert all(st["on_device"] == 1 for _, st in dev)
    same_runs(dev, host, "E264B_OUTPUT=device")


def _stats(data, picstats):
    lib = pkg.load()
    lib.e264b_of_decoder.restype = ctypes.c_void_p; lib.e264b_of_decoder.argtypes = [ctypes.c_void_p]
    lib.e264b_stats.argtypes = [ctypes.c_void_p] + [ctypes.POINTER(ctypes.c_uint64)] * 3
    dec = new_decoder(lib, picstats=picstats)
    frames = []
    loop(lib, dec, data, lambda f: frames.append(pkg._frame_bytes(f)))
    s = [ctypes.c_uint64() for _ in range(3)]
    lib.e264b_stats(lib.e264b_of_decoder(dec), *[ctypes.byref(x) for x in s])
    free_decoder(lib, dec)
    return [x.value for x in s], frames


@pytest.mark.gpu
def test_one_launch_and_the_statistics_bytes_per_picture(workdir):
    w, h = 20, 12
    data = _data(workdir, ("ps_stats", w, h, "-n 12 -s 671 --gop IPB --refs 2 --crop-right 6"))
    off, s_off = _stats(data, False)
    again, _ = _stats(data, False)
    on, s_on = _stats(data, True)
    assert len(s_off) == 12 and s_on == s_off and again == off
    assert on == [off[0] + 12, off[1], off[2] + 12 * (3072 + 24 * w * h)]
