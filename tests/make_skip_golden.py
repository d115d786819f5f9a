"""Records what the REFERENCE decoder (oracle/_ref, compiled by oracle/Makefile) outputs on the --i-period streams of
tests/test_skip.py into tests/golden/skip.json: for every stream the generator arguments, the byte count and md5 of the
.264 (pinning tools/gen264) and the reference's per-frame digests of the full decode.  Run after building:
python tests/make_skip_golden.py"""
import hashlib, json, os, sys, tempfile
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conftest import ROOT, make_stream, md5_frames
from checkers import decode_bytes
from test_skip import I_STREAMS

tmp = tempfile.mkdtemp()
out = {}
for name, w, h, args in I_STREAMS:
    data = open(make_stream(tmp, name, w, h, args), "rb").read()
    out[name] = {"args": f"-W {w} -H {h} {args}", "bytes": len(data), "stream_md5": hashlib.md5(data).hexdigest(),
                 "md5": md5_frames(decode_bytes(data, "ref")[0])}
json.dump(out, open(os.path.join(ROOT, "tests", "golden", "skip.json"), "w"), indent=1)
print("wrote", len(out), "streams")
