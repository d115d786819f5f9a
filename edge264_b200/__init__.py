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


class Edge264Motion(ctypes.Structure):
    """Layout of include/edge264_motion.h: one frame's motion export (pointers into the decoder's buffer of that frame)."""
    _fields_ = [("mv", ctypes.POINTER(ctypes.c_int16)), ("ref_frame_id", ctypes.POINTER(ctypes.c_int32)),
                ("mb_type", ctypes.POINTER(ctypes.c_uint8)), ("mb_qp", ctypes.POINTER(ctypes.c_uint8)),
                ("width_mbs", ctypes.c_int32), ("height_mbs", ctypes.c_int32), ("on_device", ctypes.c_int32)]


PACKED_I420, PACKED_NV12 = 0, 1


class Edge264Packed(ctypes.Structure):
    """Layout of include/edge264_packed.h: one frame's packed output (pointers into the decoder's buffer of that frame).
    Sizes are ceil(cropped size >> log2_scale), strides the row bytes rounded up to 64, planes 256-byte aligned
    (e264_packed_layout in csrc/records.h)."""
    _fields_ = [("planes", ctypes.c_void_p * 3), ("stride", ctypes.c_int32 * 3), ("width", ctypes.c_int32), ("height", ctypes.c_int32),
                ("width_C", ctypes.c_int32), ("height_C", ctypes.c_int32), ("format", ctypes.c_int32), ("log2_scale", ctypes.c_int32),
                ("on_device", ctypes.c_int32)]


class Edge264PicStats(ctypes.Structure):
    """Layout of include/edge264_picstats.h: one frame's statistics (pointers into the decoder's buffer of that frame)."""
    _fields_ = [("hist", ctypes.POINTER(ctypes.c_uint32)), ("sum", ctypes.POINTER(ctypes.c_uint32)), ("sum_sq", ctypes.POINTER(ctypes.c_uint32)),
                ("width_mbs", ctypes.c_int32), ("height_mbs", ctypes.c_int32), ("on_device", ctypes.c_int32)]


SKIP_NONE, SKIP_NONREF, SKIP_NONKEY = 0, 1, 2   # include/edge264_skip.h
LOOP_FILTER_ALL, LOOP_FILTER_REF, LOOP_FILTER_NONE = 0, 1, 2   # include/edge264_loopfilter.h


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
    if hasattr(lib, "edge264_get_motion"):     # the extension of include/edge264_motion.h (absent from the reference's library)
        lib.edge264_enable_motion.argtypes = [ctypes.c_void_p]
        lib.edge264_get_motion.argtypes = [ctypes.c_void_p, ctypes.POINTER(Edge264Frame), ctypes.POINTER(Edge264Motion)]
    if hasattr(lib, "edge264_get_packed"):     # the extension of include/edge264_packed.h
        lib.edge264_enable_packed.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
        lib.edge264_get_packed.argtypes = [ctypes.c_void_p, ctypes.POINTER(Edge264Frame), ctypes.POINTER(Edge264Packed)]
    if hasattr(lib, "edge264_enable_resized"):   # the resized output of include/edge264_packed.h
        lib.edge264_enable_resized.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    if hasattr(lib, "edge264_set_skip"):       # the extension of include/edge264_skip.h
        lib.edge264_set_skip.argtypes = [ctypes.c_void_p, ctypes.c_int]
    if hasattr(lib, "edge264_enable_luma_only"):   # the extension of include/edge264_luma.h
        lib.edge264_enable_luma_only.argtypes = [ctypes.c_void_p]
    if hasattr(lib, "edge264_set_loop_filter"):   # the extension of include/edge264_loopfilter.h
        lib.edge264_set_loop_filter.argtypes = [ctypes.c_void_p, ctypes.c_int]
    if hasattr(lib, "edge264_get_picstats"):   # the extension of include/edge264_picstats.h
        lib.edge264_enable_picstats.argtypes = [ctypes.c_void_p]
        lib.edge264_get_picstats.argtypes = [ctypes.c_void_p, ctypes.POINTER(Edge264Frame), ctypes.POINTER(Edge264PicStats)]
    if hasattr(lib, "edge264_get_second_view"):   # the extension of include/edge264_mvc.h
        lib.edge264_get_second_view.argtypes = [ctypes.c_void_p, ctypes.POINTER(Edge264Frame), ctypes.POINTER(Edge264Frame)]
    if hasattr(lib, "edge264_set_output_latency"):   # the extension of include/edge264_latency.h
        lib.edge264_set_output_latency.argtypes = [ctypes.c_void_p, ctypes.c_int]
    _loaded[path] = lib
    return lib


def _frame_bytes(f, mvc=False):
    """The frame's cropped samples as I420 bytes; mvc=True: those of samples_mvc (the second view of a stereo frame)."""
    out = bytearray()
    for pl in range(3):
        w = f.width_C if pl else f.width_Y; h = f.height_C if pl else f.height_Y; st = f.stride_C if pl else f.stride_Y
        base = ctypes.cast((f.samples_mvc if mvc else f.samples)[pl], ctypes.c_void_p).value
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


class _DeviceBytes:
    """A device buffer as torch sees one (__cuda_array_interface__), to copy it out without another CUDA binding."""
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (ptr, False), "strides": None, "version": 3}


def frame_motion(lib, dec, f):
    """The motion export of frame f (just returned by edge264_get_frame) as a dict of numpy arrays (copies):
    mv int16 [2][4H][4W][2], ref_frame_id int32 [2][2H][2W], mb_type uint8 [H][W], mb_qp uint8 [H][W].  Device memory
    (on_device) is copied through torch."""
    import numpy as np
    m = Edge264Motion()
    r = lib.edge264_get_motion(dec, ctypes.byref(f), ctypes.byref(m))
    if r:
        raise RuntimeError("edge264_get_motion: %s" % errno.errorcode.get(r, r))
    W, H = m.width_mbs, m.height_mbs
    out = {}
    for k, dt, shape in (("mv", np.int16, (2, 4 * H, 4 * W, 2)), ("ref_frame_id", np.int32, (2, 2 * H, 2 * W)),
                         ("mb_type", np.uint8, (H, W)), ("mb_qp", np.uint8, (H, W))):
        ptr = ctypes.cast(getattr(m, k), ctypes.c_void_p).value
        n = int(np.prod(shape)) * np.dtype(dt).itemsize
        if m.on_device:
            import torch
            raw = torch.as_tensor(_DeviceBytes(ptr, n), device="cuda").cpu().numpy()
        else:
            raw = np.frombuffer(ctypes.string_at(ptr, n), np.uint8)
        out[k] = raw.view(dt).reshape(shape)
    return out


def frame_packed(lib, dec, f):
    """The packed output of frame f (just returned by edge264_get_frame) as a dict of numpy arrays (copies, strides
    removed): format, log2_scale, on_device, y [height][width] and cb, cr [height_C][width_C] (I420) or cbcr
    [height_C][width_C][2] (NV12).  Device memory (on_device) is copied through torch."""
    import numpy as np
    p = Edge264Packed()
    r = lib.edge264_get_packed(dec, ctypes.byref(f), ctypes.byref(p))
    if r:
        raise RuntimeError("edge264_get_packed: %s" % errno.errorcode.get(r, r))
    def plane(i, rows, row_bytes):
        n = p.stride[i] * (rows - 1) + row_bytes
        if p.on_device:
            import torch
            raw = torch.as_tensor(_DeviceBytes(p.planes[i], n), device="cuda").cpu().numpy()
        else:
            raw = np.frombuffer(ctypes.string_at(p.planes[i], n), np.uint8)
        return np.lib.stride_tricks.as_strided(raw, (rows, row_bytes), (p.stride[i], 1)).copy()
    out = {"format": p.format, "log2_scale": p.log2_scale, "on_device": p.on_device, "y": plane(0, p.height, p.width)}
    if p.format == PACKED_NV12:
        out["cbcr"] = plane(1, p.height_C, 2 * p.width_C).reshape(p.height_C, p.width_C, 2)
    else:
        out["cb"], out["cr"] = plane(1, p.height_C, p.width_C), plane(2, p.height_C, p.width_C)
    return out


def frame_picstats(lib, dec, f):
    """The statistics of frame f (just returned by edge264_get_frame) as a dict of numpy uint32 arrays (copies): hist
    [3][256], sum [3][H][W], sum_sq [3][H][W], and on_device.  Device memory is copied through torch."""
    import numpy as np
    s = Edge264PicStats()
    r = lib.edge264_get_picstats(dec, ctypes.byref(f), ctypes.byref(s))
    if r:
        raise RuntimeError("edge264_get_picstats: %s" % errno.errorcode.get(r, r))
    W, H = s.width_mbs, s.height_mbs
    out = {"on_device": s.on_device}
    for k, shape in (("hist", (3, 256)), ("sum", (3, H, W)), ("sum_sq", (3, H, W))):
        ptr = ctypes.cast(getattr(s, k), ctypes.c_void_p).value
        n = 4 * int(np.prod(shape))
        if s.on_device:
            import torch
            raw = torch.as_tensor(_DeviceBytes(ptr, n), device="cuda").cpu().numpy()
        else:
            raw = np.frombuffer(ctypes.string_at(ptr, n), np.uint8)
        out[k] = raw.view(np.uint32).reshape(shape)
    return out


def frame_second_view(lib, dec, f):
    """The second view of stereo frame f (just returned by edge264_get_frame) as a frame of its own
    (edge264_get_second_view), or None for a single-view frame."""
    out = Edge264Frame()
    r = lib.edge264_get_second_view(dec, ctypes.byref(f), ctypes.byref(out))
    if r == errno.ENOENT:
        return None
    if r:
        raise RuntimeError("edge264_get_second_view: %s" % errno.errorcode.get(r, r))
    return out


def decode_bytes(data, lib=None, n_threads=0, errors=False, motion=False, packed=None, skip=SKIP_NONE, resized=None, luma_only=False, picstats=False, loop_filter=LOOP_FILTER_ALL,
                 second_view=False, output_latency=-1):
    """Decode an Annex-B byte string with the README loop (reference README.md:117-156).
    Returns (frames, return_codes) where frames = [(FrameId, width, height, i420_bytes), ...]; with errors=True each
    frame tuple also carries its per-macroblock error map (bytes, 0..100 per macroblock) or None; with motion=True it
    carries the frame's motion export (frame_motion); with packed=(format, log2_scale) it ends with the frame's packed
    output (frame_packed); resized=(format, width, height) does the same with the resized output (edge264_enable_resized,
    log2_scale -1); skip=SKIP_NONREF / SKIP_NONKEY leaves those pictures out (edge264_set_skip); luma_only=True decodes
    the Y plane only, chroma comes out as 128 (edge264_enable_luma_only); picstats=True appends the frame's statistics
    (frame_picstats) as the last element of each frame tuple; loop_filter=LOOP_FILTER_REF / LOOP_FILTER_NONE outputs
    the non-reference / all pictures without deblocking (edge264_set_loop_filter); second_view=True appends the second
    view of a stereo frame (include/edge264_mvc.h), None for a single-view frame, else a tuple laid out like the frame
    tuple itself (FrameId_mvc, width, height, i420_bytes and the same optional elements).  A library without
    edge264_get_second_view (the reference's) gives the second view's FrameId, size and samples only.  output_latency=N
    (0..16) caps the output reorder depth at N and waits for each due frame the device is finishing
    (edge264_set_output_latency)."""
    gpu = lib is None
    if gpu:
        lib = load()
    buf = ctypes.create_string_buffer(data, len(data) + 64)
    base = ctypes.addressof(buf); end = base + len(data)
    dec = lib.edge264_alloc(n_threads, None, None, 0, None, None, None)
    if not dec:
        raise RuntimeError("edge264_alloc failed" + (" (no CUDA device: the GPU backend has no CPU fallback)" if gpu else ""))
    if motion:
        r = lib.edge264_enable_motion(dec)
        if r:
            d = ctypes.c_void_p(dec)
            lib.edge264_free(ctypes.byref(d))
            raise RuntimeError("edge264_enable_motion: %s" % errno.errorcode.get(r, r))
    if packed is not None:
        r = lib.edge264_enable_packed(dec, packed[0], packed[1]) if hasattr(lib, "edge264_enable_packed") else errno.ENOTSUP
        if r:
            d = ctypes.c_void_p(dec)
            lib.edge264_free(ctypes.byref(d))
            raise RuntimeError("edge264_enable_packed: %s" % errno.errorcode.get(r, r))
    if resized is not None:
        r = lib.edge264_enable_resized(dec, *resized) if hasattr(lib, "edge264_enable_resized") else errno.ENOTSUP
        if r:
            d = ctypes.c_void_p(dec)
            lib.edge264_free(ctypes.byref(d))
            raise RuntimeError("edge264_enable_resized: %s" % errno.errorcode.get(r, r))
    if skip != SKIP_NONE:
        r = lib.edge264_set_skip(dec, skip) if hasattr(lib, "edge264_set_skip") else errno.ENOTSUP
        if r:
            d = ctypes.c_void_p(dec)
            lib.edge264_free(ctypes.byref(d))
            raise RuntimeError("edge264_set_skip: %s" % errno.errorcode.get(r, r))
    if luma_only:
        r = lib.edge264_enable_luma_only(dec) if hasattr(lib, "edge264_enable_luma_only") else errno.ENOTSUP
        if r:
            d = ctypes.c_void_p(dec)
            lib.edge264_free(ctypes.byref(d))
            raise RuntimeError("edge264_enable_luma_only: %s" % errno.errorcode.get(r, r))
    if loop_filter != LOOP_FILTER_ALL:
        r = lib.edge264_set_loop_filter(dec, loop_filter) if hasattr(lib, "edge264_set_loop_filter") else errno.ENOTSUP
        if r:
            d = ctypes.c_void_p(dec)
            lib.edge264_free(ctypes.byref(d))
            raise RuntimeError("edge264_set_loop_filter: %s" % errno.errorcode.get(r, r))
    if output_latency != -1:
        r = lib.edge264_set_output_latency(dec, output_latency) if hasattr(lib, "edge264_set_output_latency") else errno.ENOTSUP
        if r:
            d = ctypes.c_void_p(dec)
            lib.edge264_free(ctypes.byref(d))
            raise RuntimeError("edge264_set_output_latency: %s" % errno.errorcode.get(r, r))
    if picstats:
        r = lib.edge264_enable_picstats(dec) if hasattr(lib, "edge264_enable_picstats") else errno.ENOTSUP
        if r:
            d = ctypes.c_void_p(dec)
            lib.edge264_free(ctypes.byref(d))
            raise RuntimeError("edge264_enable_picstats: %s" % errno.errorcode.get(r, r))
    nal = base + 3 + (1 if data[2] == 0 else 0)
    frames, codes, f = [], [], Edge264Frame()
    drained = False
    while True:
        sc = lib.edge264_find_start_code(nal, end, 0) if nal < end else end
        before = len(frames)
        res = lib.edge264_decode_NAL(dec, nal, sc, None, None)
        if nal >= end:
            drained = True
        def entry(f):
            return ((f.FrameId, f.width_Y, f.height_Y, _frame_bytes(f)) + ((_frame_errors(f),) if errors else ())
                    + ((frame_motion(lib, dec, f),) if motion else ()) + ((frame_packed(lib, dec, f),) if packed is not None or resized is not None else ())
                    + ((frame_picstats(lib, dec, f),) if picstats else ()))
        while lib.edge264_get_frame(dec, ctypes.byref(f), 0) == 0:
            fr = entry(f)
            if second_view:
                if hasattr(lib, "edge264_get_second_view"):
                    sv = frame_second_view(lib, dec, f)
                    fr += (entry(sv) if sv is not None else None,)
                else:
                    fr += ((f.FrameId_mvc, f.width_Y, f.height_Y, _frame_bytes(f, True)) if f.samples_mvc[0] else None,)
            frames.append(fr)
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
