"""edge264_b200 — Python (ctypes) view of the edge264 C API implemented by libedge264_b200.so.

The product is the shared library (C ABI identical to the reference's edge264.h, see include/).
This module only mirrors that interface for tests and benchmarks: same function names, same
argument meaning, same errno return codes (reference edge264.h:64-70, README.md:159-240).
Only the product library is known here; the CPU checkers (oracle/) are bound by tests/checkers.py
through the same `bind()`.
"""
import ctypes, errno, os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "edge264_b200", "libedge264_b200.so")


class Edge264Frame(ctypes.Structure):
    """Layout of reference edge264.h:45-62 (96 bytes)."""
    _fields_ = [("samples", ctypes.POINTER(ctypes.c_uint8) * 3), ("samples_mvc", ctypes.POINTER(ctypes.c_uint8) * 3),
                ("mb_errors", ctypes.POINTER(ctypes.c_uint8)), ("bit_depth_Y", ctypes.c_int8), ("bit_depth_C", ctypes.c_int8),
                ("width_Y", ctypes.c_int16), ("width_C", ctypes.c_int16), ("height_Y", ctypes.c_int16), ("height_C", ctypes.c_int16),
                ("stride_Y", ctypes.c_int16), ("stride_C", ctypes.c_int16), ("stride_mb", ctypes.c_int16), ("FrameId", ctypes.c_int32),
                ("FrameId_mvc", ctypes.c_int32), ("frame_crop_offsets", ctypes.c_int16 * 4), ("return_arg", ctypes.c_void_p)]


_loaded = {}


def load():
    """The product library (CUDA backend).  Mandatory: there is no fallback."""
    return bind(LIB_PATH)


def bind(path):
    """ctypes prototypes of the seven edge264 entry points for any library that implements them."""
    if path in _loaded:
        return _loaded[path]
    if not os.path.exists(path):
        raise OSError(f"{path} is missing — build it with `python __graft_entry__.py build`")
    lib = ctypes.CDLL(path, mode=ctypes.RTLD_LOCAL)
    lib.edge264_find_start_code.restype = ctypes.c_void_p
    lib.edge264_find_start_code.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    lib.edge264_alloc.restype = ctypes.c_void_p
    lib.edge264_alloc.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    lib.edge264_flush.argtypes = [ctypes.c_void_p]
    lib.edge264_free.argtypes = [ctypes.POINTER(ctypes.c_void_p)]
    lib.edge264_decode_NAL.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    lib.edge264_get_frame.argtypes = [ctypes.c_void_p, ctypes.POINTER(Edge264Frame), ctypes.c_int]
    lib.edge264_return_frame.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    _loaded[path] = lib
    return lib


def _frame_bytes(f):
    out = bytearray()
    for pl in range(3):
        w = f.width_C if pl else f.width_Y; h = f.height_C if pl else f.height_Y; st = f.stride_C if pl else f.stride_Y
        base = ctypes.cast(f.samples[pl], ctypes.c_void_p).value
        for y in range(h):
            out += ctypes.string_at(base + y * st, w)
    return bytes(out)


def _frame_errors(f):
    """Edge264Frame.mb_errors as bytes (width_mbs x height_mbs of the coded picture, row-major), or None when the decoder
    reports no macroblock as possibly wrong."""
    if not f.mb_errors:
        return None
    return ctypes.string_at(ctypes.cast(f.mb_errors, ctypes.c_void_p).value, f.stride_mb * (
        (f.height_Y + f.frame_crop_offsets[0] + f.frame_crop_offsets[2] + 15) >> 4))


def decode_bytes(data, lib=None, n_threads=0, errors=False):
    """Decode an Annex-B byte string with the README loop (reference README.md:117-156).
    Returns (frames, return_codes) where frames = [(FrameId, width, height, i420_bytes), ...]; with errors=True each
    frame tuple also carries its per-macroblock error map (bytes, 0..100 per macroblock) or None."""
    gpu = lib is None
    if gpu:
        lib = load()
    buf = ctypes.create_string_buffer(data, len(data) + 64)
    base = ctypes.addressof(buf); end = base + len(data)
    dec = lib.edge264_alloc(n_threads, None, None, 0, None, None, None)
    if not dec:
        raise RuntimeError("edge264_alloc failed" + (" (no CUDA device: the GPU backend has no CPU fallback)" if gpu else ""))
    nal = base + 3 + (1 if data[2] == 0 else 0)
    frames, codes, f = [], [], Edge264Frame()
    drained = False
    while True:
        sc = lib.edge264_find_start_code(nal, end, 0) if nal < end else end
        before = len(frames)
        res = lib.edge264_decode_NAL(dec, nal, sc, None, None)
        if nal >= end:
            drained = True
        while lib.edge264_get_frame(dec, ctypes.byref(f), 0) == 0:
            frames.append((f.FrameId, f.width_Y, f.height_Y, _frame_bytes(f)) + ((_frame_errors(f),) if errors else ()))
        if res == errno.ENOBUFS:
            if len(frames) == before:
                break
            continue
        codes.append(res)
        if res in (errno.ENOTSUP, errno.EBADMSG):
            res = 0
        nal = sc + 3 if sc + 3 < end else end
        if res != 0 or drained:
            break
    d = ctypes.c_void_p(dec)
    lib.edge264_free(ctypes.byref(d))
    return frames, codes


def decode_file_hashes(path, lib=None):
    import hashlib
    frames, _ = decode_bytes(open(path, "rb").read(), lib)
    return [hashlib.md5(fr[3]).hexdigest() for fr in frames]
