"""The device against the CPU restatement on records drawn at the arithmetic edges, and the record contract
(edge264_b200/csrc/records.h, checked by oracle/record_check.c) on everything the parser emits.

Stream tests only ever hand the kernels what tools/gen264 chooses to write: small levels, QPs near 28, moderate weights,
smooth motion.  tests/native/record_fuzz.c draws records straight into the record ABI instead — every QP on each plane,
levels at the int16 limits and past each overflow threshold, extreme weights and offsets, int16 motion vectors and
vectors at the picture borders, every boundary strength, up to 64 slices, every intra mode for its availability, both
intra kernels — and compares the device's frames with oracle/port_recon.c byte for byte.  Every such picture keeps the
record contract first: the device is only ever given records the parser could emit, and the parser keeps that
contract even on damaged streams."""
import os, re, subprocess
import pytest
from conftest import ROOT, STREAMS, DPB_STREAMS, make_stream
from api_helpers import _damaged

FUZZ_SRC = [os.path.join(ROOT, "tests", "native", "record_fuzz.c"), os.path.join(ROOT, "oracle", "port_recon.c"), os.path.join(ROOT, "oracle", "record_check.c")]
# seed k draws geometry k % 18 of the driver's list (1x1 ... 120x68, 256x2): two rounds cover every geometry twice
SEEDS = "0-35"


@pytest.fixture(scope="module")
def fuzzer(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("fuzz") / "record_fuzz")
    subprocess.run(["gcc", "-O2", "-std=gnu11", "-w", "-pthread"] + FUZZ_SRC + ["-o", exe, "-ldl"], check=True)
    return exe


def _counters(out):
    return {m.group(1): int(m.group(2)) for m in re.finditer(r"^cov (\S+) (\d+)$", out, re.M)}


def test_generator_keeps_the_contract_and_reaches_every_edge(fuzzer):
    """CPU only: every generated picture passes the record checker (the driver stops otherwise) and reconstructs on the
    port, and every edge the draws aim at is reached: counted from the inputs, and in the port for saturation and
    wrap-around events."""
    r = subprocess.run([fuzzer, "--cpu-only", "--seeds", SEEDS], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    cov = _counters(r.stdout)
    assert len(cov) >= 70, r.stdout
    zero = [k for k, v in cov.items() if v == 0]
    assert not zero, "edges never drawn: %s" % zero
    assert cov["qp_y_values"] == 52 and cov["qp_cb_values"] == 40 and cov["qp_cr_values"] == 40   # every QP_Y, every QP'c
    assert cov["pictures"] >= 500


def _check_records(path, n_threads=0):
    tool = os.path.join(ROOT, "oracle", "oracle_decode")
    env = dict(os.environ, E264_CHECK_RECORDS="1")
    r = subprocess.run([tool, path, "-q"] + (["-t", str(n_threads)] if n_threads else []), capture_output=True, text=True, env=env, timeout=300)
    return r.returncode, r.stderr.strip().splitlines()[-1:] if r.returncode else []


@pytest.mark.parametrize("name,w,h,args", STREAMS + DPB_STREAMS, ids=[s[0] for s in STREAMS + DPB_STREAMS])
def test_parser_records_keep_the_contract(workdir, name, w, h, args):
    code, why = _check_records(make_stream(workdir, name, w, h, args))
    assert code == 0, why


def test_stored_streams_keep_the_contract():
    """The reference's own header test streams and the gen_avc 1080p fixture (tests/golden/)."""
    golden = os.path.join(ROOT, "tests", "golden")
    paths = [os.path.join(golden, "reference_streams", f) for f in sorted(os.listdir(os.path.join(golden, "reference_streams")))]
    paths.append(os.path.join(golden, "gen_avc_1080p_intra_cavlc.264"))
    for p in paths:
        code, why = _check_records(p)
        assert code == 0, (os.path.basename(p), why)


def test_damaged_streams_keep_the_contract(workdir):
    """Damaged input must not put a record outside the contract: an intra mode that reads a missing neighbour becomes
    DC, a macroblock that fails to parse is concealed, a missing reference picture is replaced by a present one."""
    path = os.path.join(workdir, "contract_damaged.264")
    for name, seed, data in _damaged(workdir):
        open(path, "wb").write(data)
        for threads in (0, 2):
            code, why = _check_records(path, threads)
            assert code == 0, "%s seed %d (%d workers): %s" % (name, seed, threads, why)


@pytest.mark.gpu
def test_device_matches_port_on_fuzzed_records(fuzzer):
    """Several hundred pictures over every geometry of the driver: the device's frames equal the port's, byte for byte,
    and the device never raises its error word."""
    lib = os.path.join(ROOT, "edge264_b200", "libedge264_b200.so")
    r = subprocess.run([fuzzer, "--lib", lib, "--seeds", SEEDS], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-500:], r.stderr[-3000:])
    assert _counters(r.stdout)["pictures"] >= 500


@pytest.mark.gpu
def test_damaged_streams_decode_identically_on_device_and_port(workdir):
    """The damaged streams of test_robustness.py through the GPU and through the port: identical frames and identical
    return codes (records that keep the contract leave nothing to chance on the device)."""
    from checkers import decode_bytes
    for name, seed, data in _damaged(workdir):
        gpu, gcodes = decode_bytes(data, "gpu")
        port, pcodes = decode_bytes(data, "port")
        assert gcodes == pcodes, "%s seed %d: return codes differ" % (name, seed)
        assert [f[0] for f in gpu] == [f[0] for f in port], "%s seed %d: frame ids differ" % (name, seed)
        for k, (a, b) in enumerate(zip(gpu, port)):
            assert a[3] == b[3], "%s seed %d: frame %d differs" % (name, seed, k)
