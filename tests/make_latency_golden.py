"""Records what the REFERENCE decoder (oracle/_ref, compiled by oracle/Makefile) outputs on the twin streams of
tests/test_output_latency.py into tests/golden/latency.json: for every pair (stream without VUI, depth N) the reference's
decode of the twin (the same stream with VUI bitstream_restriction stating max_num_reorder_frames N), with the md5 of the
twin pinning tools/gen264: per decode_NAL call [NAL index, return code, indices of the frames its get_frame loop
returned] and per frame [FrameId, md5, FrameId_mvc, md5_mvc]; the same for the API observations (borrowed frames, flush,
End of sequence).  Run after building: python tests/make_latency_golden.py"""
import json, os, sys, tempfile
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conftest import ROOT
from checkers import load
import test_output_latency as t

tmp = tempfile.mkdtemp()
ref = load("ref")
out = {"pairs": {}, "api": {}}
for name, (_, twin, _) in t.cases(tmp, full=True).items():
    out["pairs"][name] = dict(t.observe(twin, ref), twin_md5=t._md5(twin))
for name, (_, _, hold, at) in t.api_cases(tmp).items():
    out["api"][name] = t.observe(t.api_twin(tmp, name), ref, 0, -1, hold, at)
json.dump(out, open(os.path.join(ROOT, "tests", "golden", "latency.json"), "w"), separators=(",", ":"))
print("wrote", len(out["pairs"]), "pairs and", len(out["api"]), "API cases")
