"""Test-side loaders: the product library next to the CPU checkers (oracle/liboracle_dec.so = the product's host
sources over the plain-C restatement; oracle/_ref/libedge264_ref.so = the unmodified reference compiled here;
port_outputs_lib() = the product's host sources over the restatement with every optional output, built on first use).
Only tests, __graft_entry__.smoke() and the tools under tools/ import this; the shipped package knows nothing of oracle/."""
import ctypes, functools, os, hashlib, subprocess, tempfile
import edge264_b200 as _pkg
from edge264_b200 import Edge264Frame, _frame_bytes, ROOT  # noqa: F401  (re-exported for the tests)

_LIBS = {
    "gpu": _pkg.LIB_PATH,
    "port": os.path.join(ROOT, "oracle", "liboracle_dec.so"),
    "ref": os.path.join(ROOT, "oracle", "_ref", "libedge264_ref.so"),
}


def load(backend="gpu"):
    return _pkg.bind(_LIBS[backend])


@functools.lru_cache(None)
def port_outputs_lib():
    """The whole edge264 API on the CPU with error maps, the motion export, the packed and resized output and the picture
    statistics: the product's host sources over tests/native/port_outputs_backend.c."""
    native, csrc = os.path.join(ROOT, "tests", "native"), os.path.join(ROOT, "edge264_b200", "csrc")
    path = os.path.join(tempfile.mkdtemp(prefix="e264outputs"), "libport_outputs.so")
    src = [os.path.join(native, "port_outputs_backend.c"), os.path.join(native, "port_error_map.c"), os.path.join(ROOT, "oracle", "port_recon.c"),
           os.path.join(ROOT, "oracle", "record_check.c"), os.path.join(csrc, "decoder.c"), os.path.join(csrc, "slice_dec.c")]
    subprocess.run(["gcc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-w", "-o", path] + src + ["-pthread"], check=True)
    lib = _pkg.bind(path)
    lib.e264_test_record_violations.restype = ctypes.c_int
    lib.e264_test_last_violation.restype = ctypes.c_char_p
    return lib


def decode_bytes(data, backend="gpu", n_threads=0):
    return _pkg.decode_bytes(data, None if backend == "gpu" else load(backend), n_threads)


def decode_file_hashes(path, backend="gpu"):
    frames, _ = decode_bytes(open(path, "rb").read(), backend)
    return [hashlib.md5(fr[3]).hexdigest() for fr in frames]
