"""Records what the REFERENCE decoder (oracle/_ref, compiled by oracle/Makefile) outputs on the stereo streams of
tests/test_mvc.py into tests/golden/mvc.json: for the reference's two stored stereo streams and every generated one (with
the generator arguments, byte count and md5 of the .264, pinning tools/gen264) the frames of both views as [FrameId, md5,
FrameId_mvc, md5_mvc] and the return code of every NAL unit; the frames of the --deblock-off twins of the loop-filter
tests; and the API observations (borrowing and returning pairs, flush mid-stream, End of sequence back to single view,
a subset SPS with 3 views).  Run after building: python tests/make_mvc_golden.py"""
import hashlib, json, os, sys, tempfile
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conftest import ROOT, make_stream
import test_mvc as t

tmp = tempfile.mkdtemp()
out = {"stored": {}, "streams": {}, "twins": {}, "api": {}}
for name in t.STORED:
    frames, codes = t.decode(t.stored(name), "ref")
    out["stored"][name] = {"frames": t.summary(frames), "codes": codes}
for s in t.MVC_STREAMS + [t.MVC_1080P]:
    data = t.stream(tmp, s)
    frames, codes = t.decode(data, "ref")
    out["streams"][s[0]] = {"args": "-W %d -H %d %s" % s[1:], "bytes": len(data), "stream_md5": hashlib.md5(data).hexdigest(),
                            "frames": t.summary(frames), "codes": codes}
for i in (2, 5, 8):
    name, w, h, args = t.MVC_STREAMS[i]
    for twin in ("nonref", "all"):
        data = open(make_stream(tmp, name + "_off_" + twin, w, h, args + " --deblock-off " + twin), "rb").read()
        out["twins"][name + "/" + twin] = t.summary(t.decode(data, "ref")[0])
by = {s[0]: s for s in t.MVC_STREAMS}
out["api"]["borrowed"] = {"%s/%d" % (n, hold): t.observe(t.stream(tmp, by[n]), "ref", hold) for n in ("mvc_ipb", "mvc_dpb_ipb") for hold in t.HOLDS}
out["api"]["flush"] = {str(at): t.observe(t.stream(tmp, t.MVC_STREAMS[2]), "ref", 1, flush_at=at) for at in t.FLUSH_AT}
for name, data in t.api_cases(tmp).items():
    out["api"][name] = t.observe(data, "ref")
json.dump(out, open(os.path.join(ROOT, "tests", "golden", "mvc.json"), "w"), separators=(",", ":"))
print("wrote", len(out["stored"]), "stored and", len(out["streams"]), "generated streams,", len(out["twins"]), "twins and the API cases")
