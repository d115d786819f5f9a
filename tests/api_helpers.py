"""Helpers the tests share to drive the edge264 C API: the library a backend name stands for, a decoder with features
enabled, the README loop, decoding through an alloc_cb / free_cb pair, and the damaged streams of test_robustness.py."""
import ctypes, errno, random
import edge264_b200 as pkg
from checkers import port_outputs_lib
from conftest import make_stream
from test_robustness import CASES as DAMAGED_CASES, damage

_ALLOC = ctypes.CFUNCTYPE(None, ctypes.POINTER(ctypes.c_void_p), ctypes.c_uint, ctypes.POINTER(ctypes.c_void_p), ctypes.c_uint, ctypes.c_int, ctypes.c_void_p)
_FREE = ctypes.CFUNCTYPE(None, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p)


def lib_of(backend):
    """The product library for "gpu", the CPU restatement with every optional output for "port"."""
    return pkg.load() if backend == "gpu" else port_outputs_lib()


def new_decoder(lib, *, packed=None, resized=None, motion=False, picstats=False, luma_only=False, skip=pkg.SKIP_NONE, n_threads=0, alloc=(None, None)):
    dec = lib.edge264_alloc(n_threads, None, None, 0, alloc[0], alloc[1], None)
    assert dec
    if motion:
        assert lib.edge264_enable_motion(dec) == 0
    if packed is not None:
        assert lib.edge264_enable_packed(dec, *packed) == 0
    if resized is not None:
        assert lib.edge264_enable_resized(dec, *resized) == 0
    if picstats:
        assert lib.edge264_enable_picstats(dec) == 0
    if luma_only:
        assert lib.edge264_enable_luma_only(dec) == 0
    if skip != pkg.SKIP_NONE:
        assert lib.edge264_set_skip(dec, skip) == 0
    return dec


def free_decoder(lib, dec):
    d = ctypes.c_void_p(dec)
    lib.edge264_free(ctypes.byref(d))


def first_frame(lib, dec, data, buf):
    base = ctypes.addressof(buf); end = base + len(data)
    nal = base + 3 + (1 if data[2] == 0 else 0)
    f = pkg.Edge264Frame()
    while lib.edge264_get_frame(dec, ctypes.byref(f), 0) != 0:
        sc = lib.edge264_find_start_code(nal, end, 0)
        lib.edge264_decode_NAL(dec, nal, sc, None, None)
        nal = sc + 3
    return f


def loop(lib, dec, data, on_frame, borrow=0, stop_after=None):
    """The README loop over an already allocated decoder; on_frame(f) for every frame; returns the number of frames."""
    buf = ctypes.create_string_buffer(data, len(data) + 64)
    base = ctypes.addressof(buf); end = base + len(data)
    nal, count = base + 3 + (1 if data[2] == 0 else 0), 0
    while True:
        sc = lib.edge264_find_start_code(nal, end, 0) if nal < end else end
        before = count
        res = lib.edge264_decode_NAL(dec, nal, sc, None, None)
        while True:
            f = pkg.Edge264Frame()
            if lib.edge264_get_frame(dec, ctypes.byref(f), borrow):
                break
            count += 1
            on_frame(f)
        if res == errno.ENOBUFS:
            if count == before:
                break
            continue
        if nal >= end or (stop_after is not None and count >= stop_after):
            break
        nal = sc + 3 if sc + 3 < end else end
    return count


def with_alloc_cb(lib, data, malloc, free, packed=None, resized=None, motion=False, picstats=False, **features):
    """Decode through an alloc_cb / free_cb pair: (frames as (FrameId, w, h, packed, motion, picstats), each output None
    when it is off, [(samples_size, mbs_size)] calls).  features: the other keywords of new_decoder."""
    live, calls = set(), []
    def alloc(samples, size, mbs, mbs_size, err, arg):
        p = malloc(size)
        live.add(p); calls.append((size, mbs_size))
        samples[0] = p
    def release(samples, mbs, arg):
        live.remove(samples)
        free(samples)
    cbs = (_ALLOC(alloc), _FREE(release))
    dec, out = new_decoder(lib, packed=packed, resized=resized, motion=motion, picstats=picstats, alloc=cbs, **features), []
    has_packed = packed is not None or resized is not None
    def see(f):
        out.append((f.FrameId, f.width_Y, f.height_Y, pkg.frame_packed(lib, dec, f) if has_packed else None,
                    pkg.frame_motion(lib, dec, f) if motion else None, pkg.frame_picstats(lib, dec, f) if picstats else None))
        if has_packed:
            p = pkg.Edge264Packed()
            assert lib.edge264_get_packed(dec, ctypes.byref(f), ctypes.byref(p)) == 0 and p.planes[0] in live
        if picstats:
            s = pkg.Edge264PicStats()
            assert lib.edge264_get_picstats(dec, ctypes.byref(f), ctypes.byref(s)) == 0 and ctypes.cast(s.hist, ctypes.c_void_p).value in live
    loop(lib, dec, data, see)
    free_decoder(lib, dec)
    assert not live, "buffers not returned through free_cb"
    return out, calls


def _libc():
    libc = ctypes.CDLL(None)
    libc.calloc.restype = ctypes.c_void_p; libc.calloc.argtypes = [ctypes.c_size_t, ctypes.c_size_t]
    libc.free.argtypes = [ctypes.c_void_p]
    return (lambda n: libc.calloc(1, n + 64)), libc.free


def _cudart():
    """The CUDA runtime the product library was linked with: once that is loaded, its soname resolves to it."""
    pkg.load()
    return ctypes.CDLL("libcudart.so.12")


def _damaged(workdir, seeds=25):
    """The damaged streams of test_robustness.py, same mutations and seeds: the first `seeds` of each of its 25."""
    for name, w, h, args in DAMAGED_CASES:
        src = open(make_stream(workdir, name, w, h, args), "rb").read()
        for seed in range(seeds):
            yield name, seed, damage(src, random.Random(seed * 7919 + len(src)))
