"""Whole-picture reconstruction before deblocking against the numpy statement of its composition (tests/spec_picture.py),
an independent judge: the restatement (oracle/port_recon.c port_recon_mb / port_inter_mb / port_recon_picture) and the
kernels (recon_kernels.cuh staging, intra_kernels.cuh, inter_kernels.cuh) compose a picture's records into the stage
functions from one reading of the standard, so a misreading they share (a transposed implicit_w1 index, the chroma
weights taking the luma logWD, a vector read at the wrong block index) passes every test that compares them.  Here:
  - the parser's records of the stream sets, through the restatement (tests/native/port_dbk_backend.c): the statement
    with the reference decoder's arithmetic must give every dumped picture before deblocking, and every intra mode byte
    carries the unavailability bits of 6.4.11.4 exactly;
  - the record fuzzer's pictures (record_fuzz, and record_fuzz_luma for luma-only pictures) through the restatement
    (CPU) and through the device (GPU, whose references are its own earlier pictures: no comparison with the
    restatement).
Each picture is judged on its own from the frames its dump says its reference slots hold; the statement also evaluates
the standard's arithmetic on every macroblock and requires a named deviation wherever the two differ.  The runs print
the coverage of the statement, the deviation counts and their times."""
import collections, multiprocessing, os, time
from concurrent.futures import ProcessPoolExecutor
import numpy as np
import pytest
from conftest import ROOT, STREAMS, DPB_STREAMS
from test_limits import LIMITS
import spec_deblock as sd
import spec_picture as sp
import spec_pixels as px
from picture_dumps import FUZZ_SEEDS, GEOM, build_fuzzer, load_dump, run_fuzzer, stream_pictures

LUMA_SEEDS = list(range(0, 11))     # record_fuzz_luma: luma-only and colour pictures over the geometries 0..10
FN_OF = {"intra4x4": "intra4x4", "intra8x8": "intra8x8", "intra16x16": "intra16x16", "chroma": "intra_chroma"}


def judge(pics, what):
    """spec_picture.reconstruct_pictures(ref=True) of pictures, batched by geometry, against the pictures before
    deblocking.  Returns the statistics (pictures, macroblocks, coverage, deviations, geometries, luma-only pictures) and
    the failures, one line each."""
    groups = collections.defaultdict(list)
    for p in pics:
        groups[tuple(int(p.pd[k]) for k in GEOM)].append(p)
    out = dict(pics=len(pics), mbs=sum(len(p.recs) for p in pics), cov=collections.Counter(), dev=collections.Counter(),
               geoms={k[:2] for k in groups}, failures=[])
    for key, ps in groups.items():
        g = dict(zip(GEOM, key))
        slices = np.zeros((len(ps), 64), sd.SLICE)
        for i, p in enumerate(ps):
            slices[i, :len(p.slices)] = p.slices
        missing = [(i, s) for i, p in enumerate(ps) for s, f in p.refs.items() if f is None]
        if missing:
            out["failures"].append(f"{what}: picture {missing[0][0]} of {key[0]}x{key[1]} predicts from frame slot {missing[0][1]}, "
                                   f"whose content the dump does not determine")
            continue
        planes, d = sp.reconstruct_pictures(g, np.stack([p.recs for p in ps]), slices, [p.levels for p in ps], [p.refs for p in ps],
                                            np.array([bool(p.pd["luma_only"]) for p in ps]))
        out["cov"] += d["cov"]
        out["dev"] += d["dev"]
        want = sd.planes_of(np.stack([p.pre for p in ps]), g)
        bad = np.nonzero(np.any([(a != b).reshape(len(ps), -1).any(1) for a, b in zip(planes, want)], 0))[0]
        if len(bad):
            b = bad[0]
            c = next(k for k in range(3) if (planes[k][b] != want[k][b]).any())
            y, x = [int(v[0]) for v in np.nonzero(planes[c][b] != want[c][b])]
            out["failures"].append(f"{what}: {len(bad)} of {len(ps)} pictures of {key[0]}x{key[1]} macroblocks differ from the statement; "
                                   f"first: picture {b}, {sd.PLANES[c]} sample ({x}, {y}) statement {planes[c][b, y, x]} got {want[c][b, y, x]}; "
                                   f"{sp.explain(ps[b].recs, ps[b].slices, g, c, x, y)}")
        for b, a, c in d["unexplained"][:1]:
            n = 16 if c == 0 else 8
            out["failures"].append(f"{what}: picture {b} of {key[0]}x{key[1]}, macroblock {a}, {sd.PLANES[c]}: the standard's arithmetic "
                                   f"differs from the decoder's without a named deviation of that plane ({len(d['unexplained'])} such "
                                   f"macroblock planes); {sp.explain(ps[b].recs, ps[b].slices, g, c, n * (a % key[0]), n * (a // key[0]))}")
        for p in ps:   # which intra kernel the device runs (recon.cu: intra-rows when n_intra > nmb / 2), on pictures with inter
            nmb, ni = len(p.recs), int(p.pd["n_intra"])
            if 0 < ni < nmb:
                out["cov"]["intra_kernel_with_inter", "rows" if 2 * ni > nmb else "list"] += 1
    out["luma_only"] = int(out["cov"]["luma_only_pictures"])
    return out


def judge_file(path):
    return judge(load_dump(path), os.path.basename(path))


def judge_files(files):
    """judge_file over files in worker processes; the summed statistics and every failure."""
    tot = dict(pics=0, mbs=0, cov=collections.Counter(), dev=collections.Counter(), geoms=set(), failures=[], luma_only=0)
    with ProcessPoolExecutor(max_workers=min(8, os.cpu_count() or 1), mp_context=multiprocessing.get_context("spawn")) as ex:
        for r in ex.map(judge_file, files):
            for k in ("pics", "mbs", "luma_only"):
                tot[k] += r[k]
            tot["cov"] += r["cov"]
            tot["dev"] += r["dev"]
            tot["geoms"] |= r["geoms"]
            tot["failures"] += r["failures"]
    return tot


def print_report(tot, what, seconds):
    print(f"coverage of the statement, {what}:")
    for k in sorted(tot["cov"], key=str):
        print("  %-50s %d" % (" ".join(map(str, k)) if isinstance(k, tuple) else k, tot["cov"][k]))
    print(f"deviations, {what} (macroblock planes where one is present / where the standard's arithmetic also differs):")
    for name in sp.DEVIATIONS:
        print("  %-30s %d / %d" % (name, tot["dev"][name, "present"], tot["dev"][name, "differs"]))
    print(f"{what}: {tot['pics']} pictures ({tot['luma_only']} luma-only), {tot['mbs']} macroblocks judged, "
          f"{tot['dev']['macroblocks', 'differs']} where the standard's arithmetic differs, statement {seconds:.1f} s")


# ---- 6.4.11.4 ----
def mb_available(sidx, a, dx, dy):
    """6.4.10 / 6.4.12: the macroblock at (dx, dy) from macroblock a is available: inside the picture, decoded before a
    (a smaller address) and in the same slice.  sidx (H, W) the slice of each macroblock."""
    H, W = sidx.shape
    x, y = a % W + dx, a // W + dy
    return 0 <= x < W and 0 <= y < H and y * W + x < a and sidx[y, x] == sidx[a // W, a % W]


def unavailability(sidx, a, kind, blk):
    """The unavailability bits (A 1, B 2, C 4, D 8) of 6.4.11.4 for block blk of macroblock a: an Intra4x4 block
    (luma4x4BlkIdx), an Intra8x8 block (8x8 index), or -1 for the Intra16x16 / chroma prediction (A, B and D only)."""
    if blk < 0:
        return sum(bit for bit, dx, dy in ((1, -1, 0), (2, 0, -1), (8, -1, -1)) if not mb_available(sidx, a, dx, dy))
    N = 4 if kind == sp.MBK_I4x4 else 8
    bx, by = ((sp.BLK_X[blk], sp.BLK_Y[blk]) if N == 4 else (blk & 1, blk >> 1))
    un = 0
    for bit, (xs, ys) in ((1, (-1, 0)), (2, (0, -1)), (4, (N, -1)), (8, (-1, -1))):
        xn, yn = N * bx + xs, N * by + ys           # a sample of the neighbouring block, relative to the macroblock
        mx, my = xn // 16, yn // 16
        if (mx, my) == (0, 0):                      # inside the macroblock: available once decoded
            ok = (sd.blk_z(xn // 4, yn // 4) if N == 4 else (yn // 8) * 2 + xn // 8) < blk
        else:
            ok = mb_available(sidx, a, mx, my)
        un |= 0 if ok else bit
    return un


def derivable_unavailability():
    """Every unavailability value 6.4.11.4 gives, per prediction function, over the positions of a 3x3 picture and every
    first macroblock of the slice: what a picture of slices in raster order can present to each mode."""
    out = collections.defaultdict(set)
    for a in range(9):
        for start in range(a + 1):
            sidx = (np.arange(9) >= start).astype(int).reshape(3, 3)
            for z in range(16):
                out["intra4x4"].add(unavailability(sidx, a, sp.MBK_I4x4, z))
            for i8 in range(4):
                out["intra8x8"].add(unavailability(sidx, a, sp.MBK_I8x8, i8))
            out["intra16x16"].add(unavailability(sidx, a, sp.MBK_I16x16, -1))
            out["chroma"].add(unavailability(sidx, a, sp.MBK_I16x16, -1))
    return out


def required(cov):
    """The coverage entries that must be non-zero on the fuzzed pictures (tests/spec_picture.py counts them)."""
    reach = derivable_unavailability()
    keys = [(FN_OF[fn], m, un) for fn in FN_OF for m, un in px.allowed(fn) if un in reach[fn]]
    keys += [("C_substituted", "inside_mb"), ("C_substituted", "right_edge"), "intra_from_inter_neighbour", "I_PCM",
             ("concealment", "intra"), ("concealment", "inter"), "luma_only_pictures", "colour_pictures", "one_slot_both_lists",
             "mixed_list_usage_8x8", ("implicit_w1", -64), ("implicit_w1", 128), "chroma_dc_only_blocks",
             ("intra16x16_dc", "with_ac"), ("intra16x16_dc", "without_ac")]
    keys += [("luma_fraction", (x, y)) for x in range(4) for y in range(4)] + [("chroma_fraction", (x, y)) for x in range(8) for y in range(8)]
    keys += [("clamped", p, e) for p in ("luma", "chroma") for e in ("left", "right", "top", "bottom")]
    keys += [("wp", w, u) for w in sp.WP_NAMES for u in ("L0", "L1", "bi")]
    keys += [("explicit_logwd", c, v) for c in ("luma", "chroma") for v in (0, 7)]
    keys += [("transform", t, k) for t in ("4x4", "8x8") for k in ("intra", "inter")]
    keys += [("deviation_differs", n) for n in sp.DEVIATIONS]
    keys += [("intra_kernel_with_inter", k) for k in ("rows", "list")]
    return {k: cov[k] for k in keys}


def check_coverage(tot):
    reach = required(tot["cov"])
    zero = [k for k, v in reach.items() if v == 0]
    assert not zero, f"coverage entries never reached: {zero}"


# ---- the parser's records ----
@pytest.fixture(scope="module")
def parser_pictures(workdir, tmp_path_factory):
    tmp = tmp_path_factory.mktemp("picspec")
    return [(name, stream_pictures(workdir, tmp, name, w, h, args)) for name, w, h, args in STREAMS + DPB_STREAMS + LIMITS]


def test_parser_records_reconstruct_as_the_standard_says(parser_pictures):
    """The stream sets through the parser and the restatement: the statement, with the reference decoder's arithmetic,
    gives every picture before deblocking.  The restatement is held bit-exact with the reference decoder on these streams
    elsewhere (tests/test_oracle_vs_ref.py), so this ties the statement to the reference itself."""
    t0 = time.perf_counter()
    tot = dict(pics=0, mbs=0, cov=collections.Counter(), dev=collections.Counter(), failures=[], luma_only=0)
    for name, pics in parser_pictures:
        r = judge(pics, name)
        for k in ("pics", "mbs", "luma_only"):
            tot[k] += r[k]
        tot["cov"] += r["cov"]
        tot["dev"] += r["dev"]
        tot["failures"] += r["failures"]
    print_report(tot, "streams", time.perf_counter() - t0)
    assert not tot["failures"], "\n".join(tot["failures"][:10])
    assert tot["pics"] > 0 and tot["cov"]["wp", "implicit", "bi"] and tot["cov"]["wp", "explicit", "bi"] and tot["cov"]["I_PCM"]


def test_parser_unavailability_bits_are_6_4_11_4(parser_pictures):
    """Every intra mode byte of the parser's records carries exactly the unavailability of 6.4.11.4, derived from the
    macroblock's position and slice_idx (the parser refuses constrained_intra_pred_flag, so no inter neighbour is ever
    marked unavailable for being inter: equality, where the record contract asks only containment)."""
    n = collections.Counter()
    for name, pics in parser_pictures:
        for i, p in enumerate(pics):
            H, W = int(p.pd["height_mbs"]), int(p.pd["width_mbs"])
            sidx = p.recs["slice_idx"].astype(int).reshape(H, W)
            for a, r in enumerate(p.recs):
                kind = int(r["kind"])
                if kind in (sp.MBK_IPCM, sd.MBK_INTER):
                    continue
                got = [("chroma", -1, int(r["chroma_mode"]) >> 4)]
                if kind == sp.MBK_I16x16:
                    got.append(("intra16x16", -1, int(r["i16_mode"]) >> 4))
                else:
                    got += [("intra4x4" if kind == sp.MBK_I4x4 else "intra8x8", b, int(r["modes"][b]) >> 4) for b in range(16 if kind == sp.MBK_I4x4 else 4)]
                for fn, b, un in got:
                    want = unavailability(sidx, a, kind, b)
                    assert un == want, f"{name}, picture {i}, macroblock {a} ({a % W}, {a // W}), {fn} block {b}: unavailability {un:#x}, 6.4.11.4 gives {want:#x}"
                    n[fn] += 1
    print("mode bytes checked:", dict(n))
    assert all(n[fn] for fn in ("chroma", "intra16x16", "intra4x4", "intra8x8"))


# ---- fuzzed records ----
@pytest.fixture(scope="module")
def fuzzers(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("picfuzz"))
    return build_fuzzer(d), build_fuzzer(d, "record_fuzz_luma.c")


def fuzz_and_judge(fuzzers, tmp_path, extra, what):
    t0 = time.perf_counter()
    files, runs = run_fuzzer(fuzzers[0], str(tmp_path / "colour"), FUZZ_SEEDS, extra)
    lfiles, lruns = run_fuzzer(fuzzers[1], str(tmp_path / "luma"), LUMA_SEEDS, extra)
    t1 = time.perf_counter()
    assert len(files) == len(FUZZ_SEEDS) and len(lfiles) == len(LUMA_SEEDS)
    tot = judge_files(files + lfiles)
    print_report(tot, what, time.perf_counter() - t1)
    print(f"{what}: fuzzers {t1 - t0:.1f} s, geometries {sorted(tot['geoms'])}")
    assert not tot["failures"], "\n".join(tot["failures"][:10])
    for r in runs + lruns:
        assert r.returncode == 0, (r.stdout[-500:], r.stderr[-3000:])
    assert tot["pics"] >= 800 and tot["luma_only"] > 0 and tot["pics"] > tot["luma_only"]
    check_coverage(tot)
    return tot


def test_fuzzed_records_reconstruct_as_the_standard_says(fuzzers, tmp_path):
    """The record fuzzer's pictures through the restatement: the statement gives every picture before deblocking, with a
    named deviation wherever the standard's arithmetic differs, and reaches every coverage entry."""
    fuzz_and_judge(fuzzers, tmp_path, ["--cpu-only"], "fuzzed records, restatement")


@pytest.mark.gpu
def test_device_reconstructs_as_the_standard_says(fuzzers, tmp_path):
    """The record fuzzer's pictures through the device: every picture the device reconstructs before deblocking is the
    statement's, its references being the device's own earlier deblocked pictures.  The seeds cover 1x1, 1x9 and 9x1
    pictures, pictures wider than an inter chunk (64 macroblocks) and taller than a deblocking band (16 rows), and P/B
    pictures with intra fractions on both sides of the switch between the intra-rows and intra-list kernels (the coverage
    entries intra_kernel_with_inter, required non-zero)."""
    lib = os.path.join(ROOT, "edge264_b200", "libedge264_b200.so")
    tot = fuzz_and_judge(fuzzers, tmp_path, ["--lib", lib], "fuzzed records, device")
    geoms = tot["geoms"]
    assert {(1, 1), (1, 9), (9, 1)} <= geoms and max(h for _, h in geoms) > 16 and max(w for w, _ in geoms) > 64
