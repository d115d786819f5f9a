"""Deblocking (8.7) against the standard's equations in numpy (tests/spec_deblock.py), an independent judge: the device's
deblocking (deblock_kernels.cuh) and the CPU restatement's (oracle/port_recon.c) were written from one reading of the
standard and read one copy of the tables, so an error they share passes every test that compares them.  Here:
  - the tables of edge264_b200/csrc/h264_tables.h against the ones typed from the standard;
  - the line filters of the restatement (port_deblock_lines) and of the device (dbk_math.cuh built for the host) on
    lines at both sides of every decision, for every indexA x indexB x bS;
  - the boundary strength of both (port_bs_batch, dbk_bs_pair) on drawn block pairs covering every rule;
  - whole pictures: the statement applied to the picture before deblocking must give the deblocked picture, byte for
    byte, on the parser's records of the stream sets (CPU backend tests/native/port_dbk_backend.c), on the record
    fuzzer's pictures through the restatement (CPU) and through the device (GPU, independent of the restatement).
The whole-picture runs print the statement's coverage counts and assert that each is non-zero."""
import collections, ctypes, os, re, subprocess, time
import numpy as np
import pytest
from conftest import ROOT, STREAMS, DPB_STREAMS
from checkers import _LIBS
from test_limits import LIMITS
import spec_deblock as spec
from picture_dumps import FUZZ_SEEDS, GEOM, build_fuzzer, load_dump, run_fuzzer, stream_pictures

NATIVE = os.path.join(ROOT, "tests", "native")
CSRC = os.path.join(ROOT, "edge264_b200", "csrc")
I32 = np.int32


def ptr(a):
    return a.ctypes     # keeps the array alive through the call


@pytest.fixture(scope="module")
def dbl(tmp_path_factory):
    """dbk_math.cuh built for the host (tests/native/dbk_math_lib.cpp)."""
    so = str(tmp_path_factory.mktemp("dbl") / "libdbk_math.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fno-strict-aliasing", "-shared", "-fPIC", os.path.join(NATIVE, "dbk_math_lib.cpp"), "-o", so], check=True)
    return ctypes.CDLL(so)


@pytest.fixture(scope="module")
def port():
    return ctypes.CDLL(_LIBS["port"])


# ---- tables ----
def c_table(name):
    src = open(os.path.join(CSRC, "h264_tables.h")).read()
    m = re.search(r"\b%s\[[^=]*=\s*\{(.*?)\};" % name, src, re.S)
    return [int(x) for x in re.findall(r"\d+", m.group(1))]


def test_tables_are_the_standards():
    """Tables 8-15, 8-16 and 8-17 as the parser, the restatement and the device read them."""
    assert c_table("h264_qpc") == spec.QPC
    assert c_table("h264_alpha") == spec.ALPHA
    assert c_table("h264_beta") == spec.BETA
    assert c_table("h264_tc0") == [spec.TC0[b][i] for i in range(52) for b in range(3)]


# ---- line filters ----
def threshold_lines(rng, bs, ias):
    """Lines for every indexA in ias x every indexB at boundary strength bs: |p0 - q0| at alpha - 1 and alpha and, for the
    strong filter, at (alpha >> 2) + 1 and + 2; |p1 - p0|, |q1 - q0|, ap and aq at beta - 1 and beta, or 0; each pattern
    twice, around a sample near 0, near 255 or anywhere, with random signs.  Then as many random lines of small steps.
    Returns the lines (n, 8) and per line bS, indexA, indexB."""
    ia, ib, pat = [x.ravel() for x in np.meshgrid(ias, np.arange(52), np.arange(405), indexing="ij")]
    ia, ib, pat = np.tile(ia, 2), np.tile(ib, 2), np.tile(pat, 2)
    n = len(ia)
    a, b = spec._ALPHA[ia], spec._BETA[ib]
    da = np.stack([a - 1, a, (a >> 2) + 1, (a >> 2) + 2, np.zeros_like(a)], 1)[np.arange(n), pat % 5]
    rest = pat // 5
    d = [np.stack([b - 1, b, np.zeros_like(b)], 1)[np.arange(n), (rest // 3 ** k) % 3] for k in range(4)]   # |p1-p0| |q1-q0| ap aq
    centre = np.select([rng.random(n) < 1 / 3, rng.random(n) < 1 / 2], [rng.integers(0, 4, n), rng.integers(252, 256, n)], rng.integers(0, 256, n))

    def step(base, dist):
        s = np.where(rng.random(n) < 0.5, -1, 1)
        v = base + s * np.maximum(dist, 0)
        v = np.where((v < 0) | (v > 255), base - s * np.maximum(dist, 0), v)
        return np.clip(v, 0, 255)
    p0 = centre
    q0 = step(p0, da)
    p1, q1, p2, q2 = step(p0, d[0]), step(q0, d[1]), step(p0, d[2]), step(q0, d[3])
    p3, q3 = step(p2, rng.integers(0, 8, n)), step(q2, rng.integers(0, 8, n))
    lines = np.stack([p3, p2, p1, p0, q0, q1, q2, q3], 1)
    m = n // 4      # random lines: small steps from a random start, random indices
    walk = np.cumsum(rng.integers(-6, 7, (m, 8)), 1) + rng.integers(0, 256, (m, 1))
    lines = np.concatenate([lines, np.clip(walk, 0, 255)])
    ia = np.concatenate([ia, rng.integers(0, 52, m)])
    ib = np.concatenate([ib, rng.integers(0, 52, m)])
    return lines.astype(np.int64), np.full(len(ia), bs), ia, ib


def test_line_filters_match_the_standard(dbl, port):
    """8.7.2.3 / 8.7.2.4 on the restatement and on the device's dbk_line_luma / dbk_line_chroma, against the statement,
    for every indexA x indexB x bS 1..4 (and bS 0 on the device, which leaves every line), both sides of every decision."""
    rng = np.random.default_rng(8702)
    cov, n_lines = collections.Counter(), 0
    for bs in (0, 1, 2, 3, 4):
        for ias in np.array_split(np.arange(52), 4):
            lines, b, ia, ib = threshold_lines(rng, bs, ias)
            n = len(lines)
            alpha, beta = spec._ALPHA[ia], spec._BETA[ib]
            tc0 = spec._TC0[min(bs, 3), ia]
            args = [np.ascontiguousarray(x, I32) for x in (b, alpha, beta, tc0)]
            for chroma in (0, 1):
                s = lines[:, 2:6] if chroma else lines
                want, br = (spec.filter_chroma if chroma else spec.filter_luma)(s, b, alpha, beta, tc0)
                got = {}
                if bs:
                    u8 = np.ascontiguousarray(s, np.uint8)
                    port.port_deblock_lines(chroma, n, ptr(u8), *[ptr(x) for x in args])
                    got["port"] = u8
                dev = np.ascontiguousarray(s, I32)
                if chroma:
                    dbl.dbl_chroma(n, ptr(dev), *[ptr(x) for x in args])
                else:
                    dbl.dbl_luma(n, ptr(dev), *[ptr(x) for x in args], ptr(np.ascontiguousarray(rng.integers(0, 2, n), I32)))
                    if bs < 4:
                        inner = np.ascontiguousarray(s, I32)
                        dbl.dbl_luma_internal(n, ptr(inner), *[ptr(x) for x in args])
                        got["dbk_line_luma<false>"] = inner
                got["dbk_line_chroma" if chroma else "dbk_line_luma<true>"] = dev
                for who, g in got.items():
                    bad = np.nonzero((np.asarray(g, np.int64) != want).any(1))[0]
                    assert len(bad) == 0, (f"{who}, bS {bs}: {len(bad)} of {n} lines differ; first: line {s[bad[0]].tolist()} indexA {ia[bad[0]]} "
                                           f"indexB {ib[bad[0]]} alpha {alpha[bad[0]]} beta {beta[bad[0]]} tC0 {tc0[bad[0]]}: want {want[bad[0]].tolist()} got {np.asarray(g)[bad[0]].tolist()}")
                plane = "chroma" if chroma else "luma"
                for k, v in br.items():
                    cov[plane, k] += int(v.sum())
                cov[plane, "not_filtered_bs>0"] += int((~br["filtered"] & (b > 0)).sum())
                cov[plane, "weak_delta_unclipped"] += int((br["filtered"] & (b < 4) & ~br["delta_clipped"]).sum())
                # each decision of filterSamplesFlag at both sides
                p1, p0, q0, q1 = np.moveaxis(s[:, 0:4] if chroma else s[:, 2:6], 1, 0)
                for name, dist, thr in (("|p0-q0|", np.abs(p0 - q0), alpha), ("|p1-p0|", np.abs(p1 - p0), beta), ("|q1-q0|", np.abs(q1 - q0), beta)):
                    cov[plane, name + "=thr-1"] += int(((dist == thr - 1) & (thr > 0)).sum())
                    cov[plane, name + "=thr"] += int(((dist == thr) & (thr > 0)).sum())
                if not chroma:
                    for name, dist in (("ap", np.abs(s[:, 1] - p0)), ("aq", np.abs(s[:, 6] - q0))):
                        cov[plane, name + "=beta-1"] += int(((dist == beta - 1) & (beta > 0)).sum())
                        cov[plane, name + "=beta"] += int(((dist == beta) & (beta > 0)).sum())
                    small = (alpha >> 2) + 2
                    cov[plane, "|p0-q0|=(alpha>>2)+1 filtered"] += int(((np.abs(p0 - q0) == small - 1) & br["filtered"]).sum())
                    cov[plane, "|p0-q0|=(alpha>>2)+2 filtered"] += int(((np.abs(p0 - q0) == small) & br["filtered"]).sum())
            n_lines += n
    for k in sorted(cov):
        print("%-8s %-34s %d" % (k[0], k[1], cov[k]))
    print(f"{n_lines} lines, each as luma and as chroma")
    luma_only = {"strong_p_3tap", "strong_p_1tap", "strong_q_3tap", "strong_q_1tap", "weak_p1", "weak_q1"}
    zero = [k for k, v in cov.items() if v == 0 and not (k[0] == "chroma" and k[1] in luma_only)]
    assert not zero, zero


# ---- boundary strength ----
def pair_fields(r, b):
    """boundary_strength's fields of block b[i] of record r[i]."""
    n = len(r)
    intra = r["kind"] != spec.MBK_INTER
    coded, t8 = r["coded"].astype(np.int64), (r["flags"] & spec.MBF_T8x8) != 0
    coef = np.where(t8, (coded >> (b & ~3)) & 15, (coded >> b) & 1) != 0
    ri, rp = r["ref_idx"][np.arange(n), :, b >> 2], r["ref_pic"][np.arange(n), :, b >> 2]
    return intra, coef, np.where(ri < 0, -1, rp).astype(np.int64), r["mv"][np.arange(n), :, b, :].astype(np.int64)


def draw_pairs(rng, n):
    """n pairs of records and blocks (p, bp, q, bq, mb_edge) that keep the record contract: intra on either side or none,
    coefficients with and without MBF_T8x8 (in groups of four under it), the same pictures, other pictures, the lists
    swapped, one picture in both lists, one list against two, other reference indices for the same picture; vectors
    3 and 4 apart on each component, and at the ends of int16.  Unused lists carry random vectors."""
    p, q = np.zeros(n, spec.REC), np.zeros(n, spec.REC)
    bp, bq = rng.integers(0, 16, n), rng.integers(0, 16, n)
    mb_edge = rng.integers(0, 2, n)
    for r in (p, q):
        r["kind"] = np.where(rng.random(n) < 0.15, rng.integers(0, 4, n), spec.MBK_INTER)
        t8 = (r["kind"] == 1) | ((r["kind"] == spec.MBK_INTER) & (rng.random(n) < 0.4))
        r["flags"] = np.where(t8, spec.MBF_T8x8, 0) | spec.MBF_DEBLOCK
        coded = np.where(rng.random(n) < 0.3, rng.integers(0, 1 << 16, n), 0)
        coded = np.where(rng.random(n) < 0.5, coded & (1 << rng.integers(0, 16, n)), coded)      # often a single bit
        groups = sum(np.where((coded >> (4 * g)) & 15, 15 << (4 * g), 0) for g in range(4))
        r["coded"] = np.where(t8, groups, coded)
        r["mv"] = rng.integers(-32768, 32768, (n, 2, 16, 2))             # unused lists keep these
        use = rng.integers(1, 4, (n, 4))                                 # per 8x8: list 0, list 1, both
        for l in (0, 1):
            on = (use >> l) & 1 == 1
            r["ref_idx"][:, l] = np.where(on, rng.integers(0, 16, (n, 4)), -1)
            r["ref_pic"][:, l] = np.where(on, rng.integers(0, 4, (n, 4)), -1)
    # q's block: its pictures and vectors from p's block, by scenario
    ip, iq, idx = bp >> 2, bq >> 2, np.arange(n)
    scen = rng.integers(0, 6, n)    # 0 same, 1 swapped, 2 one picture twice on both sides, 3 one list against two, 4 one list each, 5 as drawn
    pic_p = p["ref_pic"][idx, :, ip].astype(np.int64)
    twice = scen == 2
    pic_p[twice] = pic_p[twice][:, :1].clip(0)
    pic_p[scen == 4, rng.integers(0, 2, n)[scen == 4]] = -1
    pic_p[(scen == 4) & (pic_p[:, 0] < 0) & (pic_p[:, 1] < 0), 0] = 1
    p["ref_pic"][idx, :, ip] = pic_p
    p["ref_idx"][idx, :, ip] = np.where(pic_p < 0, -1, rng.integers(0, 16, (n, 2)))
    sw = scen == 1
    pic_q = np.where(sw[:, None], pic_p[:, ::-1], pic_p)
    one_two = scen == 3
    drop = rng.integers(0, 2, n)
    both = one_two & (pic_q[:, 0] >= 0) & (pic_q[:, 1] >= 0)
    pic_q[both, drop[both]] = -1
    single = one_two & ~both
    pic_q[single] = np.where(pic_q[single] < 0, pic_q[single].max(1, keepdims=True), pic_q[single])
    keep = scen == 5
    pic_q[keep] = q["ref_pic"][idx, :, iq][keep]
    pic_q[keep] = np.where(q["ref_idx"][idx, :, iq][keep] < 0, -1, pic_q[keep])
    q["ref_pic"][idx, :, iq] = pic_q
    q["ref_idx"][idx, :, iq] = np.where(pic_q < 0, -1, rng.integers(0, 16, (n, 2)))
    vp = p["mv"][idx, :, bp].astype(np.int64)
    vp = np.where(rng.random((n, 1, 1)) < 0.9, vp % 64 - 32, vp)
    p["mv"][idx, :, bp] = vp
    dv = rng.choice([0, 0, 1, -1, 3, -3, 4, -4, 7, -7], (n, 2, 2))
    vq = np.clip(np.where(sw[:, None, None], vp[:, ::-1], vp) + dv, -32768, 32767)
    ext = rng.random(n) < 0.05
    p["mv"][idx[ext], :, bp[ext]] = -32768
    vq[ext] = rng.choice([-32768, 32767], (ext.sum(), 2, 2))
    q["mv"][idx, :, bq] = vq
    for r in (p, q):     # intra records use no list (records.h)
        intra = r["kind"] != spec.MBK_INTER
        r["ref_idx"][intra] = -1
        r["ref_pic"][intra] = -1
    return p, bp, q, bq, mb_edge


def test_boundary_strength_matches_the_standard(dbl, port):
    """8.7.2.1 on the restatement (port_bs_batch) and on the device's dbk_bs_pair, against the statement, on drawn block
    pairs; every rule of the standard decides some of them."""
    rng = np.random.default_rng(8721)
    n = 400000
    p, bp, q, bq, mb_edge = draw_pairs(rng, n)
    (ip, cp, pic_p, mv_p), (iq, cq, pic_q, mv_q) = pair_fields(p, bp), pair_fields(q, bq)
    want, rule = spec.boundary_strength(ip, iq, cp, cq, pic_p, pic_q, mv_p, mv_q, mb_edge != 0)
    args = [ptr(p), ptr(np.ascontiguousarray(bp, I32)), ptr(q), ptr(np.ascontiguousarray(bq, I32)), ptr(np.ascontiguousarray(mb_edge, I32))]
    for who, fn in (("port_bs", port.port_bs_batch), ("dbk_bs_pair", dbl.dbl_bs)):
        out = np.zeros(n, I32)
        fn(n, *args, ptr(out))
        bad = np.nonzero(out != want)[0]
        assert len(bad) == 0, (f"{who}: {len(bad)} of {n} pairs differ; first: p {p[bad[0]]} block {bp[bad[0]]}, q {q[bad[0]]} block {bq[bad[0]]}, "
                               f"macroblock edge {mb_edge[bad[0]]}: want {want[bad[0]]} ({spec.BS_RULES[rule[bad[0]]]}) got {out[bad[0]]}")
    counts = collections.Counter(spec.BS_RULES[r] for r in rule)
    # the vector rules on both sides of the threshold, per component
    mvcase = (rule >= 4)
    d = np.abs(mv_p - mv_q)
    for c, name in ((0, "x"), (1, "y")):
        for v in (3, 4):
            counts["dmv_%s_%d" % (name, v)] = int((mvcase[:, None] & (d[..., c] == v)).sum())
    counts["int16_extreme"] = int((mvcase & (np.abs(mv_p - mv_q) >= 65535).any((1, 2))).sum())
    counts["swapped_lists"] = int(((rule >= 4) & (pic_p[:, 0] != pic_p[:, 1]) & (pic_p.min(1) >= 0) & (pic_p[:, 0] == pic_q[:, 1])).sum())
    counts["one_list_vs_two"] = int(((pic_p >= 0).sum(1) != (pic_q >= 0).sum(1)).sum())
    counts["t8x8_coefficients"] = int(((rule == 2) & (((p["flags"] | q["flags"]) & spec.MBF_T8x8) != 0)).sum())
    for r in range(5):
        counts["bS %d" % r] = int((want == r).sum())
    for k in sorted(counts):
        print("%-22s %d" % (k, counts[k]))
    zero = [k for k in spec.BS_RULES + list(counts) if counts[k] == 0]
    assert not zero, zero


# ---- whole pictures ----


def check_pictures(pics, what):
    """The statement applied to each picture before deblocking, batched over pictures of one geometry, must give the
    picture after it.  Returns the coverage counts, and the numbers of pictures and of lines."""
    groups = collections.defaultdict(list)
    for p in pics:
        groups[tuple(int(p[0][k]) for k in GEOM)].append(p)
    cov, lines = collections.Counter(), 0
    for key, ps in groups.items():
        g = dict(zip(GEOM, key))
        slices = np.zeros((len(ps), 64), spec.SLICE)
        for i, p in enumerate(ps):
            slices[i, :len(p[2])] = p[2]
        pre = np.stack([p[3] for p in ps])
        post, d = spec.deblock_pictures(g, np.stack([p[1] for p in ps]), slices, pre)
        # the samples of the three planes (the bytes between and after them belong to no picture)
        mine, theirs, before = spec.planes_of(post, g), spec.planes_of(np.stack([p[4] for p in ps]), g), spec.planes_of(pre, g)
        bad = np.nonzero(np.any([(a != b).reshape(len(ps), -1).any(1) for a, b in zip(mine, theirs)], 0))[0]
        if len(bad):
            b = bad[0]
            plane = next(k for k in range(3) if (mine[k][b] != theirs[k][b]).any())
            y, x = [int(v[0]) for v in np.nonzero(mine[plane][b] != theirs[plane][b])]
            why = spec.explain(d, b, g, plane, x, y)
            raise AssertionError(f"{what}: {len(bad)} of {len(ps)} pictures of {g['width_mbs']}x{g['height_mbs']} macroblocks differ from the "
                                 f"statement; first: picture {b}, {spec.PLANES[plane]} sample ({x}, {y}) statement {mine[plane][b, y, x]} got "
                                 f"{theirs[plane][b, y, x]} (before deblocking {before[plane][b, y, x]}); the edges that reach it: {why}")
        cov += d["cov"]
        lines += sum(v for k, v in d["cov"].items() if k[0] == "lines")
    return cov, len(pics), lines


def print_coverage(cov, what):
    print(f"coverage of the statement, {what}:")
    for k in sorted(cov, key=str):
        print("  %-50s %d" % (" ".join(map(str, k)) if isinstance(k, tuple) else k, cov[k]))


def required(cov):
    """The coverage entries that must be non-zero: lines the filter changed for each plane x edge kind x reachable bS
    (bS 4 on macroblock edges only, bS 3 on internal edges only), both strong-filter branches and the weak filter's p1 /
    q1 update on each side, p0 / q0 clipped at 0 and at 255, indexA and indexB clipped at 0 and at 51, edges left
    unfiltered by disable_deblocking_filter_idc 2 across slices, internal luma edges skipped under transform_size_8x8_flag."""
    keys = [("changed", p, k, b) for p in spec.PLANES for k in spec.KINDS for b in ((1, 2, 3) if k == "internal" else (1, 2, 4))]
    keys += ["strong_p_3tap", "strong_p_1tap", "strong_q_3tap", "strong_q_1tap", "weak_p1", "weak_q1", "p0_clip_0", "p0_clip_255",
             "q0_clip_0", "q0_clip_255", "index_a_clip_0", "index_a_clip_51", "index_b_clip_0", "index_b_clip_51",
             "idc2_edges_unfiltered", "t8x8_internal_edges_skipped"]
    return {k: cov[k] for k in keys}


def test_parser_records_deblock_as_the_standard_says(workdir, tmp_path):
    """The stream sets through the parser and the restatement: statement(picture before deblocking) == the deblocked
    picture for every picture.  They include disable_deblocking_filter_idc 2 with slices, filter offsets of +-12, QP 0 and
    51, chroma QP offsets of +-12, PCM and 8x8 transforms.  Where a stream's generator arguments fix the chroma QP offsets,
    the records' QPc are Table 8-15 of QPY plus the offset (QPY 0 for I_PCM)."""
    cov, n_pics, n_lines, n_qpc = collections.Counter(), 0, 0, 0
    t0 = time.perf_counter()
    for name, w, h, args in STREAMS + DPB_STREAMS + LIMITS:
        pics = stream_pictures(workdir, tmp_path, name, w, h, args)
        c, n, l = check_pictures(pics, name)
        cov, n_pics, n_lines = cov + c, n_pics + n, n_lines + l
        m = re.search(r"--cqp-offset (-?\d+),(-?\d+)", args)
        if m:
            offs = [int(m.group(1)), int(m.group(2))]
            for p in pics:
                qp = p[1]["qp"].astype(np.int64)
                for k in (1, 2):
                    want = np.array(spec.QPC)[np.clip(qp[:, 0] + offs[k - 1], 0, 51)]
                    assert np.array_equal(qp[:, k], want), f"{name}: QPc of plane {k} is not Table 8-15 of QPY + {offs[k - 1]}"
                n_qpc += len(qp)
    print_coverage(cov, "streams")
    print(f"{n_pics} pictures, {n_lines} edge lines, {n_qpc} macroblocks with checked QPc, {time.perf_counter() - t0:.1f} s")
    assert n_qpc > 0
    reach = required(cov)
    zero = [k for k in reach if reach[k] == 0]
    assert not zero, zero


@pytest.fixture(scope="module")
def fuzzer(tmp_path_factory):
    return build_fuzzer(str(tmp_path_factory.mktemp("dbkfuzz")))


def fuzz_pictures(fuzzer, tmp_path, extra):
    """The fuzzer's dump files and its runs (it compares the device with the restatement itself, and still writes a
    picture that fails that comparison, so that the statement judges it first)."""
    files, runs = run_fuzzer(fuzzer, str(tmp_path / "dump"), FUZZ_SEEDS, extra)
    assert [int(re.search(r"seed_(\d+)", f).group(1)) for f in files] == FUZZ_SEEDS
    return files, runs


def fuzzer_passed(runs):
    for r in runs:
        assert r.returncode == 0, (r.stdout[-500:], r.stderr[-3000:])


def check_fuzz(files, what):
    cov, n_pics, n_lines = collections.Counter(), 0, 0
    t0 = time.perf_counter()
    for f in files:
        c, n, l = check_pictures(load_dump(f), f"{what}, {os.path.basename(f)}")
        cov, n_pics, n_lines = cov + c, n_pics + n, n_lines + l
    print_coverage(cov, what)
    print(f"{what}: {n_pics} pictures, {n_lines} edge lines, statement {time.perf_counter() - t0:.1f} s")
    reach = required(cov)
    zero = [k for k in reach if reach[k] == 0]
    assert not zero, zero
    return n_pics


def test_fuzzed_records_deblock_as_the_standard_says(fuzzer, tmp_path):
    """The record fuzzer's pictures through the restatement: statement(picture before deblocking) == the deblocked picture,
    and every coverage entry is reached."""
    files, runs = fuzz_pictures(fuzzer, tmp_path, ["--cpu-only"])
    assert check_fuzz(files, "fuzzed records, restatement") >= 800
    fuzzer_passed(runs)


@pytest.mark.gpu
def test_device_deblocks_as_the_standard_says(fuzzer, tmp_path):
    """The record fuzzer's pictures through the device, each reconstructed twice (deblocking flags cleared, then as
    drawn): statement(device's picture before deblocking) == the device's deblocked picture, independently of the
    restatement.  The seeds cover all-intra pictures (the intra-rows kernel writes the digests), P/B pictures across
    INTER_CHUNK boundaries (63..129 macroblocks wide), pictures taller than a deblocking band (16 rows) and than an
    intra-rows block (8 rows), and 1-macroblock-wide and -high pictures."""
    lib = os.path.join(ROOT, "edge264_b200", "libedge264_b200.so")
    t0 = time.perf_counter()
    files, runs = fuzz_pictures(fuzzer, tmp_path, ["--lib", lib])
    t1 = time.perf_counter()
    n = check_fuzz(files, "fuzzed records, device")
    print(f"fuzzer on the device {t1 - t0:.1f} s, whole test {time.perf_counter() - t0:.1f} s")
    fuzzer_passed(runs)
    assert n >= 800
    geoms = {(int(p[0]["width_mbs"]), int(p[0]["height_mbs"])) for f in files for p in load_dump(f)[:1]}
    assert {(1, 1), (1, 9), (9, 1)} <= geoms and max(h for _, h in geoms) > 16 and max(w for w, _ in geoms) > 64
