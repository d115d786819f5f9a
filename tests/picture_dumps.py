"""The picture dumps the whole-picture statements read (tests/test_deblock_spec.py, tests/test_picture_spec.py), written by
the record fuzzer (tests/native/record_fuzz.c, --dump) and by the CPU restatement's dump backend
(tests/native/port_dbk_backend.c, E264_DBK_DUMP).  A dump is a sequence of entries, each a little-endian uint32 tag and
its body:
  TAG_CONFIGURE  E264PicDesc (the geometry), int32 n_slots          the frame slots are (re)allocated: none holds a picture
  TAG_FILL       int32 slot, int32 y, int32 c                       the slot is set to y on its luma plane, c after it
  TAG_PICTURE    E264PicDesc, its records, its slice records, its n_coefs int16 levels, the picture before deblocking and
                 the picture after it (frame_bytes each)
The loader tracks what each frame slot holds along the dump: the deblocked picture last written to it, the constant last
filled into it, or nothing known (before any, after a configure entry, after a picture of another geometry)."""
import collections, glob, os, re, subprocess, tempfile
import numpy as np
import spec_deblock as spec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

TAG_PICTURE, TAG_FILL, TAG_CONFIGURE = 1, 2, 3
GEOM = ("width_mbs", "height_mbs", "stride_y", "stride_c", "plane_y", "frame_bytes")

# refs: frame slot -> the frame it holds (uint8, frame_bytes) or None where the dump does not determine it, for every slot
# a list of an inter macroblock of the picture uses
Picture = collections.namedtuple("Picture", "pd recs slices pre post levels refs")


def geometry(pd):
    return tuple(int(pd[k]) for k in GEOM)


def used_slots(recs):
    """The frame slots the inter macroblocks of records recs predict from."""
    inter = recs["kind"] == spec.MBK_INTER
    ri, rp = recs["ref_idx"][inter], recs["ref_pic"][inter]
    return sorted({int(s) for s in np.unique(rp[ri >= 0])})


def load_dump(path):
    """The pictures a dump file holds, in order, as Picture tuples (the first five fields are the ones the deblocking
    statement reads)."""
    raw = np.fromfile(path, np.uint8)
    off, pics, geom, slots = 0, [], None, {}

    def take(n):
        nonlocal off
        out = raw[off:off + n]
        assert len(out) == n, f"{path}: truncated entry at byte {off}"
        off += n
        return out
    while off < len(raw):
        tag = int(take(4).view("<u4")[0])
        if tag == TAG_CONFIGURE:
            geom = geometry(take(spec.PICDESC.itemsize).view(spec.PICDESC)[0])
            take(4)
            slots = {}
        elif tag == TAG_FILL:
            slot, y, c = (int(v) for v in take(12).view("<i4"))
            assert geom is not None, f"{path}: a fill before any geometry"
            g = dict(zip(GEOM, geom))
            f = np.empty(g["frame_bytes"], np.uint8)
            f[:g["plane_y"]], f[g["plane_y"]:] = y, c
            slots[slot] = f
        elif tag == TAG_PICTURE:
            pd = take(spec.PICDESC.itemsize).view(spec.PICDESC)[0]
            nmb, ns, fb = int(pd["width_mbs"]) * int(pd["height_mbs"]), int(pd["n_slices"]), int(pd["frame_bytes"])
            if geometry(pd) != geom:
                geom, slots = geometry(pd), {}
            recs = take(nmb * spec.REC.itemsize).view(spec.REC)
            sl = take(ns * spec.SLICE.itemsize).view(spec.SLICE)
            levels = take(2 * int(pd["n_coefs"])).view("<i2")
            pre, post = take(fb), take(fb)
            pics.append(Picture(pd, recs, sl, pre, post, levels, {s: slots.get(s) for s in used_slots(recs)}))
            slots[int(pd["dst_slot"])] = post
        else:
            raise AssertionError(f"{path}: unknown entry tag {tag} at byte {off - 4}")
    return pics


# ---- the producers ----
NATIVE = os.path.join(ROOT, "tests", "native")
CSRC = os.path.join(ROOT, "edge264_b200", "csrc")
# the record fuzzer's seeds: seed k takes geometry k % 18 of its list; geometry 14 (120x68) is left to the fuzzer's own
# comparison with the restatement, the statements take a minute or more over it
FUZZ_SEEDS = [k for k in range(36) if k % 18 != 14]
_built = {}


def port_dbk_lib():
    """The whole edge264 API on the CPU restatement, every picture written out before and after deblocking."""
    if "lib" not in _built:
        import edge264_b200 as pkg
        path = os.path.join(tempfile.mkdtemp(prefix="e264dbk"), "libport_dbk.so")
        src = [os.path.join(NATIVE, "port_dbk_backend.c"), os.path.join(ROOT, "oracle", "port_backend.c"), os.path.join(ROOT, "oracle", "port_recon.c"),
               os.path.join(ROOT, "oracle", "record_check.c"), os.path.join(CSRC, "decoder.c"), os.path.join(CSRC, "slice_dec.c")]
        subprocess.run(["gcc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-w", "-o", path] + src + ["-pthread", "-Wl,--wrap=e264_default_backend"], check=True)
        _built["lib"] = pkg.bind(path)
    return _built["lib"]


def stream_pictures(workdir, tmp_path, name, w, h, args):
    """The pictures of a generated stream through the parser and the CPU restatement, as load_dump gives them."""
    import edge264_b200 as pkg
    from conftest import make_stream
    data = open(make_stream(workdir, name, w, h, args), "rb").read()
    dump = str(tmp_path / (name + ".dbk"))
    os.environ["E264_DBK_DUMP"] = dump
    try:
        frames, _ = pkg.decode_bytes(data, port_dbk_lib())
    finally:
        del os.environ["E264_DBK_DUMP"]
    assert frames
    return load_dump(dump)


def build_fuzzer(outdir, source="record_fuzz.c"):
    """tests/native/record_fuzz.c (or record_fuzz_luma.c) over the restatement, built into outdir."""
    exe = os.path.join(outdir, source[:-2])
    src = [os.path.join(NATIVE, source), os.path.join(ROOT, "oracle", "port_recon.c"), os.path.join(ROOT, "oracle", "record_check.c")]
    subprocess.run(["gcc", "-O2", "-std=gnu11", "-w", "-pthread"] + src + ["-o", exe, "-ldl"], check=True)
    return exe


def run_fuzzer(exe, outdir, seeds, extra):
    """The fuzzer over seeds (a sorted list, run as contiguous ranges) with --dump outdir; returns the dump files in seed
    order and the runs (the fuzzer compares the device with the restatement itself, and still writes a picture that fails
    that comparison, so that the statements judge it first)."""
    os.makedirs(outdir, exist_ok=True)
    ranges, runs = [], []
    for s in seeds:
        if ranges and ranges[-1][1] == s - 1:
            ranges[-1][1] = s
        else:
            ranges.append([s, s])
    for a, b in ranges:
        runs.append(subprocess.run([exe, "--seeds", f"{a}-{b}", "--dump", outdir] + extra, capture_output=True, text=True, timeout=1800))
    files = sorted(glob.glob(os.path.join(outdir, "seed_*.bin")), key=lambda f: int(re.search(r"seed_(\d+)", f).group(1)))
    return files, runs
