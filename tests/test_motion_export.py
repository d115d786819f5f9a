"""The motion export (include/edge264_motion.h): per output frame, the vectors of every 4x4 block, the FrameId each 8x8
block predicts from, the macroblock types and QP_Y, derived from the reconstruction records (e264_motion_kernel on the
GPU).  CPU tests run the product's host sources over the plain-C restatement of the reconstruction and of the export
(tests/native/port_outputs_backend.c), bound into a library built here; the values are checked against the decoded pixels,
which are bit-exact with the reference decoder.  The GPU tests compare the device's export with that restatement."""
import ctypes, errno, json, os, subprocess, sys
import numpy as np
import pytest
from conftest import ROOT, make_stream
from api_helpers import lib_of, _ALLOC, _FREE, _cudart, _damaged
from checkers import port_outputs_lib
import edge264_b200 as pkg
import checkers


def decode(data, backend="port", n_threads=0, motion=True):
    """(FrameId, width, height, i420 bytes, error map, motion dict) per frame, and the return codes."""
    return pkg.decode_bytes(data, lib_of(backend), n_threads, errors=True, motion=motion)


def same_motion(a, b):
    return a.keys() == b.keys() and all(np.array_equal(a[k], b[k]) for k in a)


def gen(workdir, name, w, h, args):
    return open(make_stream(workdir, name, w, h, args), "rb").read()


# ---- 1. the values against the pixels ----
# no inter residual, no deblocking, default weights: an inter 4x4 block whose vectors are full-sample is a plain copy (or
# the rounded average of two) of samples of the pictures its FrameIds name
PIXEL_STREAMS = [
    ("mv_ip", 20, 12, "-n 10 -s 401 --gop IP --refs 3 --density 0 --deblock 1 --wp 0 --intra-pct 5 --mvrange 8"),
    ("mv_ipb", 20, 12, "-n 12 -s 402 --gop IPB --refs 3 --density 0 --deblock 1 --wp 0 --intra-pct 5 --mvrange 8"),
    ("mv_ip_slices", 16, 10, "-n 10 -s 403 --gop IP --refs 3 --density 0 --deblock 1 --wp 0 --slices 3 --cavlc --mvrange 12"),
    ("mv_ipb_slices", 16, 10, "-n 12 -s 404 --gop IPB --refs 3 --density 0 --deblock 1 --wp 0 --slices 3 --mvrange 12"),
]


def planes(f):
    w, h, raw = f[1], f[2], np.frombuffer(f[3], np.uint8)
    y = raw[:w * h].reshape(h, w)
    cb = raw[w * h:w * h * 5 // 4].reshape(h // 2, w // 2)
    cr = raw[w * h * 5 // 4:].reshape(h // 2, w // 2)
    return y, cb, cr


def predict(stack, idx, by, bx, mvx, mvy, n):
    """n x n blocks at (by, bx) (block units) of the pictures stack[idx], moved by whole-sample (mvx, mvy), border clamped."""
    d = np.arange(n)
    yy = np.clip(by[:, None, None] * n + d[None, :, None] + mvy[:, None, None], 0, stack.shape[1] - 1)
    xx = np.clip(bx[:, None, None] * n + d[None, None, :] + mvx[:, None, None], 0, stack.shape[2] - 1)
    return stack[idx[:, None, None], yy, xx].astype(np.int32)


def check_against_pixels(frames):
    """Returns (luma blocks, bi-predicted luma blocks, chroma blocks) checked."""
    ids = [f[0] for f in frames]
    pos = {fid: k for k, fid in enumerate(ids)}
    pl = [planes(f) for f in frames]
    stacks = [np.stack([p[c] for p in pl]) for c in range(3)]
    n_luma = n_bi = n_chroma = 0
    for k, f in enumerate(frames):
        m = f[5]
        mv, rid = m["mv"].astype(np.int32), m["ref_frame_id"]
        inter = np.kron(m["mb_type"] >= 4, np.ones((4, 4), bool))
        used = np.stack([np.kron(rid[l] >= 0, np.ones((2, 2), bool)) for l in range(2)])
        assert not (used & ~inter).any() and (used[0] | used[1] | ~inter).all()
        assert not mv[~used].any(), "a vector where the list is unused"
        for l in range(2):
            assert all(i in pos for i in np.unique(rid[l][rid[l] >= 0])), "a FrameId no output frame has"
        rid4 = np.stack([np.kron(rid[l], np.ones((2, 2), np.int32)) for l in range(2)])
        for comp, unit in ((0, 4), (1, 8)):
            exact = ((mv[..., 0] % unit == 0) & (mv[..., 1] % unit == 0)) | ~used
            by, bx = np.nonzero(inter & exact[0] & exact[1])
            n = 4 if comp == 0 else 2
            preds = []
            for l in range(2):
                u = used[l, by, bx]
                idx = np.array([pos.get(i, 0) for i in rid4[l, by, bx]], np.int64)
                planes_ = [stacks[0]] if comp == 0 else [stacks[1], stacks[2]]
                preds.append((u, [predict(s, idx, by, bx, mv[l, by, bx, 0] // unit, mv[l, by, bx, 1] // unit, n) for s in planes_]))
            (u0, p0), (u1, p1) = preds
            for c in range(len(p0)):
                pred = np.where((u0 & u1)[:, None, None], (p0[c] + p1[c] + 1) >> 1, np.where(u0[:, None, None], p0[c], p1[c]))
                plane = pl[k][0] if comp == 0 else pl[k][1 + c]
                d = np.arange(n)
                got = plane[by[:, None, None] * n + d[None, :, None], bx[:, None, None] * n + d[None, None, :]]
                bad = np.nonzero((pred != got).any(axis=(1, 2)))[0]
                assert not len(bad), "frame %d plane %d: %d of %d blocks differ, first at 4x4 block (%d, %d)" % (
                    f[0], comp + c, len(bad), len(by), bx[bad[0]], by[bad[0]])
            if comp == 0:
                n_luma += len(by); n_bi += int((u0 & u1).sum())
            else:
                n_chroma += len(by)
    return n_luma, n_bi, n_chroma


@pytest.mark.parametrize("name,w,h,args", PIXEL_STREAMS, ids=[s[0] for s in PIXEL_STREAMS])
def test_vectors_and_frame_ids_rebuild_the_pixels(workdir, name, w, h, args):
    frames, _ = decode(gen(workdir, name, w, h, args))
    n_luma, n_bi, n_chroma = check_against_pixels(frames)
    print("%s: %d luma blocks (%d bi-predicted), %d chroma blocks rebuilt" % (name, n_luma, n_bi, n_chroma))
    assert n_luma >= 2000 and n_chroma >= 500
    if "IPB" in args:
        assert n_bi >= 100


def test_pixel_check_sees_a_wrong_frame_id(workdir):
    """The check is not vacuous: naming the previous picture in place of the right one is caught."""
    name, w, h, args = PIXEL_STREAMS[0]
    frames, _ = decode(gen(workdir, name, w, h, args))
    ids = sorted(f[0] for f in frames)
    k = next(k for k, f in enumerate(frames) if (f[5]["ref_frame_id"][0] == ids[0]).any() and f[0] > ids[1])
    m = dict(frames[k][5]); r = m["ref_frame_id"].copy(); r[r == ids[0]] = ids[1]; m["ref_frame_id"] = r
    with pytest.raises(AssertionError):
        check_against_pixels(frames[:k] + [frames[k][:5] + (m,)] + frames[k + 1:])


# ---- 2. types, intra, skip, QP ----
def test_intra_and_skip_macroblocks(workdir):
    frames, _ = decode(gen(workdir, "mv_types", 12, 8, "-n 12 -s 411 --gop IPB --refs 2 --intra-pct 30 --skip-pct 40 --pcm 20 --t8x8 50"))
    seen = set()
    for f in frames:
        m = f[5]
        t = m["mb_type"]
        seen |= set(np.unique(t).tolist())
        intra = np.kron(t <= 3, np.ones((4, 4), bool))
        assert not m["mv"][:, intra].any()
        assert (m["ref_frame_id"][:, np.kron(t <= 3, np.ones((2, 2), bool))] == -1).all()
        assert (m["mb_qp"][t == 3] == 0).all()
        # skipped macroblocks predict from list 0 only in P pictures, from at least one list always
        skip = np.kron(t == 5, np.ones((2, 2), bool))
        assert ((m["ref_frame_id"][0] >= 0) | (m["ref_frame_id"][1] >= 0))[skip].all()
    assert seen == {0, 1, 2, 3, 4, 5}, seen


@pytest.mark.parametrize("qp", [4, 20, 36, 48])
def test_mb_qp_follows_the_stream_qp(workdir, qp):
    """gen264 keeps every macroblock's QP_Y in [qp - 8, qp + 10]; I_PCM reports 0."""
    frames, _ = decode(gen(workdir, "mv_qp%d" % qp, 8, 6, "-n 6 -s %d --gop IPB --qp %d --pcm 10" % (420 + qp, qp)))
    vals = np.concatenate([f[5]["mb_qp"][f[5]["mb_type"] != 3] for f in frames])
    assert vals.min() >= max(qp - 8, 0) and vals.max() <= min(qp + 10, 51)
    assert abs(float(np.median(vals)) - qp) <= 3


# ---- 3. output order and lifetime ----
BREF = ("mv_bref", 6, 5, "-n 30 -s 431 --gop IPB --bref --refs 3 --idr 17")


def _borrowed(lib, data):
    """Every frame borrowed and held until the end of the stream; the exports read after everything is decoded."""
    buf = ctypes.create_string_buffer(data, len(data) + 64)
    base = ctypes.addressof(buf); end = base + len(data)
    dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
    assert lib.edge264_enable_motion(dec) == 0
    held, nal = [], base + 3 + (1 if data[2] == 0 else 0)
    while True:
        sc = lib.edge264_find_start_code(nal, end, 0) if nal < end else end
        before = len(held)
        res = lib.edge264_decode_NAL(dec, nal, sc, None, None)
        while True:
            f = pkg.Edge264Frame()
            if lib.edge264_get_frame(dec, ctypes.byref(f), 1):
                break
            held.append(f)
        if res == errno.ENOBUFS and len(held) > before:
            continue
        if nal >= end:
            break
        nal = sc + 3 if sc + 3 < end else end
    out = {f.FrameId: pkg.frame_motion(lib, dec, f) for f in held}
    for f in held:
        lib.edge264_return_frame(dec, f.return_arg)
    assert lib.edge264_get_motion(dec, ctypes.byref(held[0]), ctypes.byref(pkg.Edge264Motion())) == errno.EINVAL
    d = ctypes.c_void_p(dec)
    lib.edge264_free(ctypes.byref(d))
    return out


def test_borrowed_frames_keep_their_export(workdir):
    data = gen(workdir, *BREF)
    plain = {f[0]: f[5] for f in decode(data)[0]}
    borrowed = _borrowed(port_outputs_lib(), data)
    assert plain.keys() == borrowed.keys() and len(plain) == 30
    assert all(same_motion(plain[k], borrowed[k]) for k in plain)


def test_export_survives_flush(workdir):
    """Half the stream, edge264_flush, then the whole stream again on the same decoder: the second pass equals a fresh one,
    FrameIds apart (the numbering goes on across a flush, in the export's reference FrameIds as in the frames')."""
    data = gen(workdir, *BREF)
    fresh = [(f[0], f[5]) for f in decode(data)[0]]
    lib = port_outputs_lib()
    buf = ctypes.create_string_buffer(data, len(data) + 64)
    base = ctypes.addressof(buf); end = base + len(data)
    dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
    assert lib.edge264_enable_motion(dec) == 0
    f, got = pkg.Edge264Frame(), []
    for half in (True, False):
        nal, count = base + 3 + (1 if data[2] == 0 else 0), 0
        while True:
            sc = lib.edge264_find_start_code(nal, end, 0) if nal < end else end
            res = lib.edge264_decode_NAL(dec, nal, sc, None, None)
            while lib.edge264_get_frame(dec, ctypes.byref(f), 0) == 0:
                count += 1
                if not half:
                    got.append((f.FrameId, pkg.frame_motion(lib, dec, f)))
            if res == errno.ENOBUFS:
                continue
            if nal >= end or (half and count >= 12):
                break
            nal = sc + 3 if sc + 3 < end else end
        if half:
            lib.edge264_flush(dec)
    d = ctypes.c_void_p(dec)
    lib.edge264_free(ctypes.byref(d))
    shift = got[0][0] - fresh[0][0]
    assert shift > 0 and [g[0] for g in got] == [f[0] + shift for f in fresh]
    for (_, g), (_, fr) in zip(got, fresh):
        r = fr["ref_frame_id"]
        assert same_motion(g, dict(fr, ref_frame_id=np.where(r >= 0, r + shift, r)))


def test_export_is_the_same_for_every_thread_count(workdir):
    data = gen(workdir, *BREF)
    runs = [decode(data, n_threads=t)[0] for t in (0, 1, 3)]
    for r in runs[1:]:
        assert [f[0] for f in r] == [f[0] for f in runs[0]]
        assert all(same_motion(a[5], b[5]) for a, b in zip(r, runs[0]))


# ---- 4. damaged streams ----
def test_damaged_streams_with_the_export(workdir, monkeypatch):
    """The record contract holds with the export on; samples and error maps are those of a decoder without it, and every
    FrameId the export names is one the decoder gave a picture."""
    lib = port_outputs_lib()
    monkeypatch.setenv("E264_CHECK_RECORDS", "1")
    n = 0
    for name, seed, data in _damaged(workdir):
        on, codes_on = decode(data)
        off, codes_off = decode(data, motion=False)
        assert lib.e264_test_record_violations() == 0, "%s seed %d: %s" % (name, seed, lib.e264_test_last_violation())
        assert codes_on == codes_off and [f[:5] for f in on] == [f[:5] for f in off], "%s seed %d" % (name, seed)
        top = max([f[0] for f in on], default=-1)
        for f in on:
            m = f[5]
            assert m["mb_type"].max() <= 5
            r = m["ref_frame_id"]
            assert ((r == -1) | ((r >= 0) & (r <= top + 64))).all()
        n += 1
    assert n == 75


# ---- 5. API ----
def test_api_errors(workdir):
    data = gen(workdir, *BREF)
    lib = port_outputs_lib()
    dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
    buf = ctypes.create_string_buffer(data, len(data) + 64)
    base = ctypes.addressof(buf); end = base + len(data)
    nal = base + 3 + (1 if data[2] == 0 else 0)
    f = pkg.Edge264Frame()
    while lib.edge264_get_frame(dec, ctypes.byref(f), 0) != 0:
        sc = lib.edge264_find_start_code(nal, end, 0)
        lib.edge264_decode_NAL(dec, nal, sc, None, None)
        nal = sc + 3
    assert lib.edge264_get_motion(dec, ctypes.byref(f), ctypes.byref(pkg.Edge264Motion())) == errno.ENOENT
    assert lib.edge264_enable_motion(dec) == errno.EBUSY
    d = ctypes.c_void_p(dec); lib.edge264_free(ctypes.byref(d))
    # a backend without the export: oracle/port_backend.c
    plain = checkers.load("port")
    dec = plain.edge264_alloc(0, None, None, 0, None, None, None)
    assert plain.edge264_enable_motion(dec) == errno.ENOTSUP
    d = ctypes.c_void_p(dec); plain.edge264_free(ctypes.byref(d))
    with pytest.raises(RuntimeError, match="ENOTSUP"):
        pkg.decode_bytes(data, plain, motion=True)


def test_ctypes_layout_matches_the_header(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "edge264_motion.h"\nint main(void) { printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %d %d\\n", '
                   "sizeof(Edge264Motion), offsetof(Edge264Motion, mv), offsetof(Edge264Motion, ref_frame_id), offsetof(Edge264Motion, mb_type), "
                   "offsetof(Edge264Motion, mb_qp), offsetof(Edge264Motion, width_mbs), offsetof(Edge264Motion, height_mbs), offsetof(Edge264Motion, on_device), "
                   "sizeof(Edge264Frame), EDGE264_MB_INTER, EDGE264_MB_SKIP); return 0; }\n")
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe], check=True)
    got = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()
    M = pkg.Edge264Motion
    want = [ctypes.sizeof(M)] + [getattr(M, k).offset for k in ("mv", "ref_frame_id", "mb_type", "mb_qp", "width_mbs", "height_mbs", "on_device")] + [96, 4, 5]
    assert [int(x) for x in got] == want


# ---- 6. the device against the restatement ----
def _gpu_inputs(workdir):
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "streams.json")))
    gen264 = os.path.join(ROOT, "tools", "gen264")
    for name, v in gold.items():
        if name.startswith("_"):
            continue
        path = os.path.join(workdir, "gold_" + name + ".264")
        if not os.path.exists(path):
            subprocess.run([gen264, "-o", path] + v["args"].split(), check=True, stderr=subprocess.DEVNULL, timeout=120)
        yield name, open(path, "rb").read()
    rdir = os.path.join(ROOT, "tests", "golden", "reference_streams")
    for fn in sorted(os.listdir(rdir)):
        yield fn, open(os.path.join(rdir, fn), "rb").read()
    yield "gen_avc_1080p", open(os.path.join(ROOT, "tests", "golden", "gen_avc_1080p_intra_cavlc.264"), "rb").read()
    yield "1080p_ipb", gen(workdir, "mv_1080p_ipb", 120, 68, "-n 8 -s 441 --gop IPB --refs 2 --t8x8 50 --density 52 --qp 28 --wp 0")
    for name, seed, data in _damaged(workdir):
        yield "%s/%d" % (name, seed), data


@pytest.mark.gpu
def test_device_export_matches_restatement(workdir):
    n = 0
    for label, data in _gpu_inputs(workdir):
        for t in ((0, 3) if "/" not in label else (0,)):
            g, gc = decode(data, "gpu", t)
            p, pc = decode(data, "port", t)
            assert gc == pc and [f[0] for f in g] == [f[0] for f in p], (label, t)
            for a, b in zip(g, p):
                assert a[3] == b[3], "%s (%d workers) frame %d: samples differ" % (label, t, a[0])
                for k in b[5]:
                    assert np.array_equal(a[5][k], b[5][k]), "%s (%d workers) frame %d: %s differs" % (label, t, a[0], k)
                n += 1
    assert n > 1000


# ---- 7. the export where the samples are: device memory ----
def motion_with_device_alloc(data):
    """Decode with an alloc_cb that hands out cudaMalloc memory: (FrameId, on_device, motion) per frame."""
    cudart = _cudart()
    live = set()

    def alloc(samples, size, mbs, mbs_size, err, arg):
        p = ctypes.c_void_p()
        assert cudart.cudaMalloc(ctypes.byref(p), ctypes.c_size_t(size)) == 0
        live.add(p.value)
        samples[0] = p.value
    def free(samples, mbs, arg):
        live.discard(samples)
        cudart.cudaFree(ctypes.c_void_p(samples))
    a, fr = _ALLOC(alloc), _FREE(free)
    lib = pkg.load()
    buf = ctypes.create_string_buffer(data, len(data) + 64)
    base = ctypes.addressof(buf); end = base + len(data)
    dec = lib.edge264_alloc(0, None, None, 0, a, fr, None)
    assert dec and lib.edge264_enable_motion(dec) == 0
    nal = base + 3 + (1 if data[2] == 0 else 0)
    out, f, m = [], pkg.Edge264Frame(), pkg.Edge264Motion()
    while True:
        sc = lib.edge264_find_start_code(nal, end, 0) if nal < end else end
        before = len(out)
        res = lib.edge264_decode_NAL(dec, nal, sc, None, None)
        while lib.edge264_get_frame(dec, ctypes.byref(f), 0) == 0:
            assert lib.edge264_get_motion(dec, ctypes.byref(f), ctypes.byref(m)) == 0
            assert ctypes.cast(m.mv, ctypes.c_void_p).value in live
            out.append((f.FrameId, m.on_device, pkg.frame_motion(lib, dec, f)))
        if res == errno.ENOBUFS:
            if len(out) == before:
                break
            continue
        if nal >= end:
            break
        nal = sc + 3 if sc + 3 < end else end
    d = ctypes.c_void_p(dec)
    lib.edge264_free(ctypes.byref(d))
    assert not live
    return out


_SUB = """
import sys, ctypes, errno, pickle
sys.path.insert(0, sys.argv[3])
import edge264_b200 as pkg
lib = pkg.load()
data = open(sys.argv[1], 'rb').read()
buf = ctypes.create_string_buffer(data, len(data) + 64); base = ctypes.addressof(buf); end = base + len(data)
dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
assert lib.edge264_enable_motion(dec) == 0
nal, out, f, m = base + 3 + (1 if data[2] == 0 else 0), [], pkg.Edge264Frame(), pkg.Edge264Motion()
while True:
    sc = lib.edge264_find_start_code(nal, end, 0) if nal < end else end
    res = lib.edge264_decode_NAL(dec, nal, sc, None, None)
    while lib.edge264_get_frame(dec, ctypes.byref(f), 0) == 0:
        assert lib.edge264_get_motion(dec, ctypes.byref(f), ctypes.byref(m)) == 0
        out.append((f.FrameId, m.on_device, pkg.frame_motion(lib, dec, f)))
    if res == errno.ENOBUFS:
        continue
    if nal >= end:
        break
    nal = sc + 3 if sc + 3 < end else end
pickle.dump(out, open(sys.argv[2], 'wb'))
"""


@pytest.mark.gpu
def test_device_memory_output(workdir):
    data = gen(workdir, *BREF)
    host = [(f[0], f[5]) for f in decode(data, "gpu")[0]]
    for label, got in (("alloc_cb", motion_with_device_alloc(data)), ("E264B_OUTPUT=device", None)):
        if got is None:
            import pickle
            src = os.path.join(workdir, "mv_dev.264"); out = os.path.join(workdir, "mv_dev.pkl")
            open(src, "wb").write(data)
            subprocess.run([sys.executable, "-c", _SUB, src, out, ROOT], check=True, env=dict(os.environ, E264B_OUTPUT="device"), timeout=300)
            got = pickle.load(open(out, "rb"))
        assert [g[0] for g in got] == [h[0] for h in host], label
        assert all(g[1] == 1 for g in got), label
        assert all(same_motion(g[2], h[1]) for g, h in zip(got, host)), label


# ---- 8. a decoder without the export pays nothing ----
def _stats(data, motion):
    lib = pkg.load()
    lib.e264b_of_decoder.restype = ctypes.c_void_p; lib.e264b_of_decoder.argtypes = [ctypes.c_void_p]
    lib.e264b_stats.argtypes = [ctypes.c_void_p] + [ctypes.POINTER(ctypes.c_uint64)] * 3
    buf = ctypes.create_string_buffer(data, len(data) + 64)
    base = ctypes.addressof(buf); end = base + len(data)
    dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
    if motion:
        assert lib.edge264_enable_motion(dec) == 0
    nal, frames, f = base + 3 + (1 if data[2] == 0 else 0), [], pkg.Edge264Frame()
    while True:
        sc = lib.edge264_find_start_code(nal, end, 0) if nal < end else end
        res = lib.edge264_decode_NAL(dec, nal, sc, None, None)
        while lib.edge264_get_frame(dec, ctypes.byref(f), 0) == 0:
            frames.append(pkg._frame_bytes(f))
        if res == errno.ENOBUFS:
            continue
        if nal >= end:
            break
        nal = sc + 3 if sc + 3 < end else end
    s = [ctypes.c_uint64() for _ in range(3)]
    lib.e264b_stats(lib.e264b_of_decoder(dec), *[ctypes.byref(x) for x in s])
    d = ctypes.c_void_p(dec)
    lib.edge264_free(ctypes.byref(d))
    return [x.value for x in s], frames


@pytest.mark.gpu
def test_export_off_costs_nothing(workdir):
    name, w, h, args = "mv_stats", 20, 12, "-n 12 -s 451 --gop IPB --refs 2"
    data = gen(workdir, name, w, h, args)
    off, s_off = _stats(data, False)
    again, s_again = _stats(data, False)
    on, s_on = _stats(data, True)
    n = len(s_off)
    assert n == 12 and s_on == s_off == s_again
    # the same launches, H2D and D2H bytes as a decoder that never enables the export, run twice; the export adds one
    # launch and one copy of 162 bytes per macroblock per picture
    assert off == again
    assert on == [off[0] + n, off[1], off[2] + n * w * h * 162]


def test_libraries_export_the_motion_api():
    """The product library (loading needs libcudart only) and the CPU restatement library of oracle/ both have it."""
    for path in (checkers._LIBS["gpu"], checkers._LIBS["port"]):
        lib = ctypes.CDLL(path)
        assert hasattr(lib, "edge264_enable_motion") and hasattr(lib, "edge264_get_motion"), path
    assert hasattr(ctypes.CDLL(checkers._LIBS["gpu"]), "e264b_submit_motion")
