"""Records what the REFERENCE decoder (oracle/_ref, compiled by oracle/Makefile) outputs on the streams of
tests/test_limits.py into tests/golden/limits.json: for every stream the generator arguments, the byte count and md5 of
the .264 (pinning tools/gen264), the reference's per-frame digests, and for the 1920x1088 streams the summary line of
`ref_decode -q`.  Run after building: python tests/make_limits_golden.py"""
import hashlib, json, os, subprocess, sys, tempfile
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conftest import ROOT, make_stream, md5_frames
from checkers import decode_bytes
from test_limits import LIMITS, FULL_LIMITS

tmp = tempfile.mkdtemp()
out = {}
for name, w, h, args in LIMITS + FULL_LIMITS:
    path = make_stream(tmp, name, w, h, args)
    data = open(path, "rb").read()
    e = {"args": f"-W {w} -H {h} {args}", "bytes": len(data), "stream_md5": hashlib.md5(data).hexdigest()}
    if (name, w, h, args) in FULL_LIMITS:
        r = subprocess.run([os.path.join(ROOT, "oracle", "_ref", "ref_decode"), path, "-q"], capture_output=True, text=True, timeout=600, check=True)
        e["ref_summary"] = r.stdout.strip().splitlines()[-1]
    else:
        e["md5"] = md5_frames(decode_bytes(data, "ref")[0])
    out[name] = e
json.dump(out, open(os.path.join(ROOT, "tests", "golden", "limits.json"), "w"), indent=1)
print("wrote", len(out), "streams")
