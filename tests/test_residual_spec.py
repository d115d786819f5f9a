"""Residual reconstruction against the standard's equations (tests/spec_residual.py), an independent judge: until now the
residual path was checked against the reference's own functions (tests/test_kat.py) and the device against the CPU
restatement (the record fuzzer), so an error all three shared would pass.  Here:
  - the restatement's port_idct4x4, port_idct8x8, port_luma_dc, port_chroma_dc and port_dc4x4 (CPU);
  - mc_math.cuh's mc_add_res4 compiled for the host, over every prediction x every int16 residual (CPU);
  - the kernels' residual_stage through e264b_kat_residual, on records of every kind, colour and luma-only (GPU).
Per block type, the claims are: every draw the standard bounds (its values inside int16) equals the standard, with the one
measured exception of the 8x8 rounding below; every draw equals the reference's arithmetic (spec_residual.ref_*); the
number of draws where that arithmetic differs from the standard is nonzero and pinned; every (type, qP) cell has
conforming draws within 1/8 of the bound."""
import ctypes, os, subprocess
import numpy as np
import pytest
from conftest import ROOT
from checkers import _LIBS
import spec_residual as spec

NEAR = 7 << 12   # 7/8 of 2^15


# ---- tables ----
def header_table(name):
    """an array of edge264_b200/csrc/h264_tables.h, parsed from its initialiser"""
    import re
    txt = open(os.path.join(ROOT, "edge264_b200", "csrc", "h264_tables.h")).read()
    m = re.search(r"\b" + name + r"\b[^=]*=\s*\{(.*?)\};", txt, re.S)
    return np.array([int(v) for v in re.findall(r"-?\d+", m.group(1))], np.int64)


def test_tables_match_the_standard():
    """The header's normAdjust values, default lists (raster) and zig-zag scans equal the ones typed from the standard;
    the typed default lists are symmetric, and the typed scans are the frame zig-zag of Figures 8-8 and 8-9."""
    assert np.array_equal(header_table("h264_norm4x4").reshape(6, 3), spec.V4)
    assert np.array_equal(header_table("h264_norm8x8").reshape(6, 6), spec.V8)
    assert np.array_equal(header_table("h264_zigzag4x4"), spec.ZIGZAG4)
    assert np.array_equal(header_table("h264_zigzag8x8"), spec.ZIGZAG8)
    for name, lst in (("h264_default4x4_intra", spec.DEFAULT_4x4_INTRA), ("h264_default4x4_inter", spec.DEFAULT_4x4_INTER),
                      ("h264_default8x8_intra", spec.DEFAULT_8x8_INTRA), ("h264_default8x8_inter", spec.DEFAULT_8x8_INTER)):
        w = spec.weight_matrix(lst)
        assert np.array_equal(header_table(name), w.ravel()), name
        assert np.array_equal(w, w.T), name
    for N, zz in ((4, spec.ZIGZAG4), (8, spec.ZIGZAG8)):
        assert sorted(zz) == list(range(N * N))
        diag = [(p // N + p % N) for p in zz]                    # anti-diagonals in order, alternating direction
        assert diag == sorted(diag)
        for s in range(2 * N - 1):
            rows = [p // N for p in zz if p // N + p % N == s]
            assert rows == sorted(rows, reverse=s % 2 == 0)
    assert [spec.class4(i, j) for i, j in ((0, 0), (1, 1), (0, 1), (1, 0), (2, 2), (3, 1))] == [0, 1, 2, 2, 0, 1]
    assert spec.CLASS8[0].tolist() == [0, 3, 4, 3, 0, 3, 4, 3] and spec.CLASS8[2].tolist() == [4, 5, 2, 5, 4, 5, 2, 5]
    assert spec.CLASS8[1].tolist() == [3, 1, 5, 1, 3, 1, 5, 1]


# ---- draws ----
def lists(rng, n, N, inter):
    """(n, N, N) weight matrices, each drawn as Flat_16, the default list (intra or inter: `inter` (n,) bools), all 1,
    all 255 or random 1..255"""
    kind = rng.integers(0, 5, n)
    d4 = np.stack([spec.weight_matrix(spec.DEFAULT_4x4_INTRA), spec.weight_matrix(spec.DEFAULT_4x4_INTER)])
    d8 = np.stack([spec.weight_matrix(spec.DEFAULT_8x8_INTRA), spec.weight_matrix(spec.DEFAULT_8x8_INTER)])
    w = rng.integers(1, 256, (n, N, N))
    w[kind == 0] = 16
    w[kind == 1] = (d4 if N == 4 else d8)[np.asarray(inter, int)[kind == 1]]
    w[kind == 2] = 1
    w[kind == 3] = 255
    return w


class BlockType:
    """A block type: its name, block size N, number of qPs, whether it is chroma, and the range of the DC values its blocks
    take as d00 (0: none).  transform_types attaches its functions on (levels, weights, qP, dc): scale, maxval (the
    largest bounded value), std (the standard), ok (the bound), dev (the reference's arithmetic) and port (the
    restatement)."""
    def __init__(self, name, N, nq, chroma, dc_range):
        self.name, self.N, self.nq, self.chroma, self.dc_range = name, N, nq, chroma, dc_range


def block_draws(t, rng, q):
    """The draws of one (type, qP) cell: (levels, weights, dc or None).  Basis blocks (one level of +-1, +-L and +-(L+1) at
    every position, L the largest level whose d stays in int16), random blocks scaled so that their largest bounded
    value is log-uniform in 2^3 .. 2^17.5, random blocks scaled to 0.85 .. 1.0 of the bound, and blocks of -32768 /
    32767 / random levels."""
    N, P = t.N, t.N * t.N
    inter = rng.integers(0, 2, 1)[0] if t.chroma else t.inter
    parts = []
    # basis
    n = P * 6
    w = lists(rng, n, N, np.full(n, inter))
    pos = np.repeat(np.arange(P), 6)
    onehot = np.zeros((n, P), np.int64)
    onehot[np.arange(n), pos] = 1
    onehot = onehot.reshape(n, N, N)
    qq = np.full(n, q)
    dval = lambda L: np.abs(t.scale(onehot * L[:, None, None], w, qq)).reshape(n, -1).max(1)
    lo, hi = np.ones(n, np.int64), np.full(n, 32767)
    for _ in range(16):      # the largest L in 1..32767 with |d| <= 2^15 - 1 (1 when even 1 is past it)
        mid = (lo + hi + 1) >> 1
        good = dval(mid) <= spec.HI
        lo, hi = np.where(good, mid, lo), np.where(good, hi, mid - 1)
    L = lo
    sel = np.arange(n) % 6
    amp = np.select([sel < 2, sel < 4], [np.ones(n, np.int64), L], np.minimum(L + 1, 32767)) * np.where(sel % 2, -1, 1)
    c = onehot * amp[:, None, None]
    dc = None
    if t.dc_range:
        dc = rng.choice([-1, 1], n) * rng.integers(0, 1 << 15, n)
    parts.append((c, w, dc))
    # random, log-uniform and near the bound
    for k, (tlo, thi, logu) in enumerate(((3, 17.5, True), (0.85, 1.0, False))):
        n = 96 if logu else 48
        w = lists(rng, n, N, np.full(n, inter))
        dens = rng.uniform(0.05, 1, (n, 1, 1))
        c0 = rng.integers(-64, 65, (n, N, N)) * (rng.uniform(0, 1, (n, N, N)) < dens)
        c0[:, 0, 0] += rng.integers(-64, 65, n)
        dc0 = rng.integers(-4096, 4097, n) if t.dc_range else None
        if t.dc_range:
            c0[:, 0, 0] = 0
        qq = np.full(n, q)
        m0 = np.maximum(t.maxval(c0, w, qq, dc0), 1)
        T = 2.0 ** rng.uniform(tlo, thi, n) if logu else (1 << 15) * rng.uniform(tlo, thi, n)
        f = T / m0
        c = np.clip(np.rint(c0 * f[:, None, None]), -32768, 32767).astype(np.int64)
        dc = np.rint(dc0 * f).astype(np.int64) if t.dc_range else None
        parts.append((c, w, dc))
    # extremes
    n = 32
    w = lists(rng, n, N, np.full(n, inter))
    c = rng.choice(np.array([0, 32767, -32768, 1, -1]), (n, N, N))
    c = np.where(rng.uniform(0, 1, (n, N, N)) < 0.2, rng.integers(-32768, 32768, (n, N, N)), c)
    dc = None
    if t.dc_range:
        c[:, 0, 0] = 0
        dc = rng.integers(-t.dc_range, t.dc_range + 1, n)
    parts.append((c, w, dc))
    c = np.concatenate([p[0] for p in parts])
    w = np.concatenate([p[1] for p in parts])
    dc = np.concatenate([p[2] for p in parts]) if t.dc_range else None
    return c, w, dc


def port_lib():
    lib = ctypes.CDLL(_LIBS["port"])
    vp, ci = ctypes.c_void_p, ctypes.c_int
    lib.port_idct4x4.argtypes = [vp, vp, ci, ci, ci, vp]
    lib.port_idct8x8.argtypes = [vp, vp, ci, vp]
    lib.port_luma_dc.argtypes = [vp, vp, ci, vp]
    lib.port_chroma_dc.argtypes = [vp, ci, ci, vp]
    lib.port_dc4x4.argtypes = [ci, vp]
    return lib


def transform_types(lib):
    """The transform block types: 4x4 intra / inter, 8x8 intra / inter, Intra16x16 AC (4x4 with the luma DC as d00) and
    chroma AC (4x4 with the chroma DC as d00, QP'c 0..39)."""
    out = []
    for name, N, nq, inter, chroma, dc_range in (("4x4 intra", 4, 52, 0, False, 0), ("4x4 inter", 4, 52, 1, False, 0),
                                                 ("8x8 intra", 8, 52, 0, False, 0), ("8x8 inter", 8, 52, 1, False, 0),
                                                 ("Intra16x16 AC", 4, 52, 0, False, 1 << 25), ("chroma AC", 4, 40, 0, True, 1 << 26)):
        t = BlockType(name, N, nq, chroma, dc_range)
        t.inter = inter
        if N == 4:
            t.scale, t.maxval = (lambda c, w, q: spec.scale4x4(c, w, q)), spec.max4x4
            t.std, t.ok, t.dev = spec.residual4x4, spec.residual4x4_ok, spec.ref_idct4x4_sat16

            def port(c, w, q, dc, lib=lib):
                c16, w8 = np.ascontiguousarray(c, np.int16), np.ascontiguousarray(w, np.uint8)
                r = np.zeros((len(c), 4, 4), np.int16)
                for i in range(len(c)):
                    lib.port_idct4x4(c16[i].ctypes.data, w8[i].ctypes.data, int(q[i]), dc is not None, 0 if dc is None else int(dc[i]), r[i].ctypes.data)
                return r.astype(np.int64)
        else:
            t.scale, t.maxval = spec.scale8x8, lambda c, w, q, dc: spec.max8x8(c, w, q)
            t.std, t.ok, t.dev = (lambda c, w, q, dc: spec.residual8x8(c, w, q)), (lambda c, w, q, dc: spec.residual8x8_ok(c, w, q)), (lambda c, w, q, dc: spec.ref_idct8x8_int16(c, w, q))

            def port(c, w, q, dc, lib=lib):
                c16, w8 = np.ascontiguousarray(c, np.int16), np.ascontiguousarray(w, np.uint8)
                r = np.zeros((len(c), 8, 8), np.int16)
                for i in range(len(c)):
                    lib.port_idct8x8(c16[i].ctypes.data, w8[i].ctypes.data, int(q[i]), r[i].ctypes.data)
                return r.astype(np.int64)
        t.port = port
        out.append(t)
    return out


def transform_draws(t, seed):
    """The draws of every (qP) cell of t, concatenated: (levels, weights, qP, dc or None)."""
    rng = np.random.default_rng(seed)
    C, W, DC, Q = [], [], [], []
    for q in range(t.nq):
        c, w, dc = block_draws(t, rng, q)
        C.append(c); W.append(w); Q.append(np.full(len(c), q))
        if dc is not None:
            DC.append(dc)
    c, w, q = np.concatenate(C), np.concatenate(W), np.concatenate(Q)
    dc = np.concatenate(DC) if DC else None
    return c, w, q, dc


def check_claims(name, std, dev, got, ok, mx, cell, top=None):
    """The four claims for one block type; returns the counts of draws in bound, out of bound, differing from the
    standard, and differing from it in bound."""
    n = len(std)
    flat = lambda a: a.reshape(n, -1)
    d_got = (flat(got) != flat(dev)).any(1)
    assert not d_got.any(), f"{name}: {d_got.sum()} draws differ from the reference's arithmetic, first {np.nonzero(d_got)[0][0]}"
    differ = (flat(dev) != flat(std)).any(1)
    inb = differ & ok
    if top is None:
        assert not inb.any(), f"{name}: {inb.sum()} conforming draws differ from the standard"
    else:   # the 8x8 rounding: exactly the conforming draws with some m >= 2^15 - 32
        assert np.array_equal(inb, ok & top), f"{name}: conforming draws differing from the standard are not those with m >= 2^15 - 32"
    cells = sorted(set(cell.tolist()))
    bare = [q for q in cells if not (ok & (cell == q) & (mx >= NEAR)).any()]
    assert not bare, f"{name}: no conforming draw within 1/8 of the bound at qP {bare}"
    return int(ok.sum()), int((~ok).sum()), int(differ.sum()), int(inb.sum())


def test_restatement_transforms_match_the_standard():
    lib = port_lib()
    rows = []
    for k, t in enumerate(transform_types(lib)):
        c, w, q, dc = transform_draws(t, 100 + k)
        std, ok, dev = t.std(c, w, q, dc), t.ok(c, w, q, dc), t.dev(c, w, q, dc)
        mx = t.maxval(c, w, q, dc)
        top = None
        if t.N == 8:
            top = (spec.transform8x8_m(spec.scale8x8(c, w, q)) >= spec.HI - 31).reshape(len(c), -1).any(1)
        got = t.port(c, w, q, dc)
        rows.append((t.name, len(c)) + check_claims(t.name, std, dev, got, ok, mx, q, top))
    rows += dc_rows(lib)
    print(f"{'block type':16s} {'draws':>8s} {'in bound':>9s} {'outside':>8s} {'ref != std':>10s} {'of them in bound':>16s}")
    for r in rows:
        print(f"{r[0]:16s} {r[1]:8d} {r[2]:9d} {r[3]:8d} {r[4]:10d} {r[5]:16d}")
    got = {r[0]: r[4] for r in rows}
    assert all(v > 0 for v in got.values()), got
    assert got == DIFFERING_PINNED, got
    assert {r[0]: r[5] for r in rows} == IN_BOUND_DIFFERING_PINNED


def dc_draws(rng, shape, nq, maxval):
    """DC levels per qP: basis (1, -1, 32767, -32768 at every position), random blocks scaled log-uniformly up to past the bound
    and to 0.85 .. 1.0 of it, and -32768 / 32767 / random levels; with each list's (0, 0) weight drawn like the lists"""
    C, W, Q = [], [], []
    P = int(np.prod(shape))
    for q in range(nq):
        basis = np.zeros((P * 4, P), np.int64)
        basis[np.arange(P * 4), np.repeat(np.arange(P), 4)] = np.tile([1, -1, 32767, -32768], P)
        basis = basis.reshape(-1, *shape)
        n = 96 + 48
        c0 = rng.integers(-64, 65, (n, *shape))
        w00 = lists(rng, n + len(basis) + 32, 4, rng.integers(0, 2, n + len(basis) + 32))[:, 0, 0]
        qq = np.full(n, q)
        m0 = np.maximum(maxval(c0, w00[:n], qq), 1)
        T = np.concatenate([2.0 ** rng.uniform(3, 18, 96), (1 << 15) * rng.uniform(0.85, 1.0, 48)])
        c = np.clip(np.rint(c0 * (T / m0).reshape(-1, *[1] * len(shape))), -32768, 32767).astype(np.int64)
        ext = rng.choice(np.array([0, 32767, -32768]), (32, *shape))
        C += [c, basis, ext]
        W.append(w00)
        Q.append(np.full(n + len(basis) + 32, q))
    return np.concatenate(C), np.concatenate(W), np.concatenate(Q)


def dc_rows(lib):
    """Intra16x16 DC (port_luma_dc), chroma DC (port_chroma_dc) and the DC-only blocks (port_dc4x4)."""
    rows = []
    rng = np.random.default_rng(200)
    lmax = lambda c, w, q: np.maximum(np.abs(spec.luma_dc_f(c)).reshape(len(c), -1).max(1), np.abs(spec.luma_dc(c, w, q)).reshape(len(c), -1).max(1))
    c, w, q = dc_draws(rng, (4, 4), 52, lmax)
    c16 = np.ascontiguousarray(c, np.int16)
    lst = np.ascontiguousarray(np.repeat(w[:, None], 16, 1), np.uint8)
    got = np.zeros((len(c), 16), np.int32)
    for i in range(len(c)):
        lib.port_luma_dc(c16[i].ctypes.data, lst[i].ctypes.data, int(q[i]), got[i].ctypes.data)
    rows.append(("Intra16x16 DC", len(c)) + check_claims("Intra16x16 DC", spec.luma_dc(c, w, q), spec.ref_luma_dc_wrap32(c, w, q),
                                                         got.reshape(-1, 4, 4).astype(np.int64), spec.luma_dc_ok(c, w, q), lmax(c, w, q), q))
    cmax = lambda c, w, q: np.maximum(np.abs(spec.chroma_dc_f(c)).reshape(len(c), -1).max(1), np.abs(spec.chroma_dc(c, w, q)).reshape(len(c), -1).max(1))
    c, w, q = dc_draws(rng, (2, 2), 40, cmax)
    c16 = np.ascontiguousarray(c, np.int16)
    got = np.zeros((len(c), 4), np.int32)
    for i in range(len(c)):
        lib.port_chroma_dc(c16[i].ctypes.data, int(w[i]), int(q[i]), got[i].ctypes.data)
    rows.append(("chroma DC", len(c)) + check_claims("chroma DC", spec.chroma_dc(c, w, q), spec.ref_chroma_dc_wrap32(c, w, q),
                                                     got.reshape(-1, 2, 2).astype(np.int64), spec.chroma_dc_ok(c, w, q), cmax(c, w, q), q))
    # DC-only blocks: dc near the bound, near where (dc + 32) >> 6 leaves int16, log-uniform up to the DC paths' 2^26
    edge = 32767 * 64 - 32
    dc = np.concatenate([np.arange(-(1 << 15) - 64, -(1 << 15) + 64), np.arange((1 << 15) - 64, (1 << 15) + 64),
                         np.arange(edge - 64, edge + 128), np.arange(-edge - 128, -edge + 64),
                         rng.choice([-1, 1], 4096) * np.rint(2.0 ** rng.uniform(0, 26, 4096)).astype(np.int64)])
    got = np.zeros((len(dc), 16), np.int16)
    for i in range(len(dc)):
        lib.port_dc4x4(int(dc[i]), got[i].ctypes.data)
    rows.append(("DC only", len(dc)) + check_claims("DC only", spec.dc_only4x4(dc), spec.ref_dc_only_trunc16(dc), got.reshape(-1, 4, 4).astype(np.int64),
                                                    spec.dc_only4x4_ok(dc), np.abs(dc), np.zeros(len(dc), int)))
    return rows


# the seeded draws where the reference's arithmetic differs from the standard, per block type, and how many of them the
# standard bounds: only the 8x8 transform's, where some m of 8.5.13.2 lies in 2^15 - 32 .. 2^15 - 1
DIFFERING_PINNED = {"4x4 intra": 1459, "4x4 inter": 1489, "8x8 intra": 14853, "8x8 inter": 14799, "Intra16x16 AC": 1658,
                    "chroma AC": 1275, "Intra16x16 DC": 890, "chroma DC": 216, "DC only": 822}
IN_BOUND_DIFFERING_PINNED = {"4x4 intra": 0, "4x4 inter": 0, "8x8 intra": 642, "8x8 inter": 647, "Intra16x16 AC": 0,
                             "chroma AC": 0, "Intra16x16 DC": 0, "chroma DC": 0, "DC only": 0}


# ---- picture construction: the host build of mc_add_res4 ----
@pytest.fixture(scope="module")
def mcl(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("mcl") / "libmc_math.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", os.path.join(ROOT, "tests", "native", "mc_math_lib.cpp"), "-o", so], check=True)
    return ctypes.CDLL(so)


def test_residual_add_matches_the_standard(mcl):
    """mc_add_res4 over every prediction 0..255 x every int16 residual: 8-357 (Clip1(pred + r)) wherever pred + r stays in
    int16, the reference's 16-bit add (ref_add_int16) everywhere.  A residual of a conforming block lies in -512..512."""
    p, r = [a.ravel() for a in np.meshgrid(np.arange(256), np.arange(-32768, 32768), indexing="ij")]
    pw = p.astype(np.uint32).reshape(-1, 4)
    ru = (r & 0xffff).astype(np.uint32).reshape(-1, 4)
    words = np.ascontiguousarray(pw[:, 0] | pw[:, 1] << 8 | pw[:, 2] << 16 | pw[:, 3] << 24)
    r01, r23 = np.ascontiguousarray(ru[:, 0] | ru[:, 1] << 16), np.ascontiguousarray(ru[:, 2] | ru[:, 3] << 16)
    out = np.zeros(len(words), np.uint32)
    mcl.mcl_add_res4(len(words), words.ctypes, r01.ctypes, r23.ctypes, out.ctypes)
    got = ((out[:, None] >> (8 * np.arange(4, dtype=np.uint32))) & 255).ravel().astype(np.int64)
    std, dev = spec.construct(p, r), spec.ref_add_int16(p, r)
    assert np.array_equal(got, dev)
    in16 = p + r <= spec.HI
    assert np.array_equal(got[in16], std[in16])
    differ = int((got != std).sum())
    print(f"mc_add_res4: {len(p)} samples, {differ} differ from 8-357 (pred + r past 32767)")
    assert differ == 255 * 256 // 2   # pred p > 0 with r >= 32768 - p: sum of 1..255
    assert (np.abs(r) <= 512).sum() > 0 and np.array_equal(got[np.abs(r) <= 512], std[np.abs(r) <= 512])


# ---- the device: residual_stage on whole records ----
REC = np.dtype([("kind", "u1"), ("flags", "u1"), ("qp", "u1", 3), ("chroma_mode", "u1"), ("i16_mode", "u1"), ("slice_idx", "u1"),
                ("coded", "<u4"), ("coef_off", "<u4"), ("modes", "u1", 16), ("ref_idx", "i1", (2, 4)), ("ref_pic", "i1", (2, 4)),
                ("err", "u1"), ("reserved", "u1", 15), ("mv", "<i2", (2, 16, 2))])
SLICE = np.dtype([("head", "u1", 8), ("wp_w", "<i2", (2, 16, 3)), ("wp_o", "<i2", (2, 16, 3)), ("implicit_w1", "<i2", (16, 16)),
                  ("scaling4x4", "u1", (6, 16)), ("scaling8x8", "u1", (2, 64))])
KINDS = [(spec.MBK_I4x4, 0), (spec.MBK_I8x8, 1), (spec.MBK_I16x16, 0), (spec.MBK_INTER, 0), (spec.MBK_INTER, 1)]


def record_draws(seed, n=3000, n_slices=8):
    """n records of every non-PCM kind with random coded-bit subsets (chroma DC-only ones among them), QP'Y 0..51 and
    QP'c 0..39, over n_slices slices whose eight lists are drawn independently; each block's levels are scaled
    log-uniformly up to 2^6, or in 40 % of the records up to 2^15 with some blocks of -32768 / 32767.  Returns (records, slices, pool)."""
    rng = np.random.default_rng(seed)
    sl = np.zeros(n_slices, SLICE)
    for s in range(n_slices):
        inter = np.array([0, 0, 0, 1, 1, 1])
        sl[s]["scaling4x4"] = lists(rng, 6, 4, inter).reshape(6, 16)
        sl[s]["scaling8x8"] = lists(rng, 2, 8, np.array([0, 1])).reshape(2, 64)
    recs = np.zeros(n, REC)
    pool = []
    off = 0

    def block(k, dc_slot):
        s = 2.0 ** rng.uniform(0, 15 if wild else 6)
        c = np.rint(rng.uniform(-s, s, k) * (rng.uniform(0, 1, k) < rng.uniform(0.1, 1))).astype(np.int64)
        if wild and rng.uniform() < 0.1:
            c = rng.choice(np.array([0, 32767, -32768]), k)
        if dc_slot:
            c[0] = 0
        return c
    for i in range(n):
        kind, t8 = KINDS[i % len(KINDS)]
        wild = rng.uniform() < 0.4
        r = recs[i]
        r["kind"], r["flags"], r["slice_idx"] = kind, t8, rng.integers(0, n_slices)
        r["qp"] = [rng.integers(0, 52), rng.integers(0, 40), rng.integers(0, 40)]
        dens = rng.uniform(0, 1)
        if t8:
            luma = sum(0xf << (4 * k) for k in range(4) if rng.uniform() < dens)
        else:
            luma = sum(1 << b for b in range(16) if rng.uniform() < dens)
        cdc = (spec.CODED_CB_DC if rng.uniform() < 0.5 else 0) | (spec.CODED_CR_DC if rng.uniform() < 0.5 else 0)
        cac = 0 if rng.uniform() < 0.3 else sum(1 << (16 + k) for k in range(8) if rng.uniform() < dens)
        ydc = spec.CODED_Y_DC if kind == spec.MBK_I16x16 and rng.uniform() < 0.8 else 0
        coded = luma | cdc | cac | ydc
        r["coded"], r["coef_off"] = coded, off
        run = []
        if ydc:
            run.append(block(16, False))
        if t8:
            run += [block(64, False) for k in range(4) if (luma >> (4 * k)) & 1]
        else:
            run += [block(16, kind == spec.MBK_I16x16) for b in range(16) if (luma >> b) & 1]
        if cdc:
            run += [block(4, False) if coded & bit else np.zeros(4, np.int64) for bit in (spec.CODED_CB_DC, spec.CODED_CR_DC)]
        run += [block(16, True) for k in range(8) if (cac >> (16 + k)) & 1]
        run = np.concatenate(run) if run else np.zeros(0, np.int64)
        run = np.concatenate([run, np.zeros(-len(run) % 8, np.int64)])
        pool.append(run)
        off += len(run)
    return recs, sl, np.concatenate(pool).astype(np.int16)


@pytest.mark.gpu
def test_device_residual_matches_the_standard():
    """e264b_kat_residual (the kernels' residual_stage, colour and luma-only) on drawn records against mb_residual: equal
    to the reference's arithmetic on every record, to the standard on every conforming one (but those with an 8x8 m at
    2^15 - 32 or above); luma-only gives the colour decode's luma and a zero chroma residual."""
    lib = ctypes.CDLL(_LIBS["gpu"])
    vp, ci = ctypes.c_void_p, ctypes.c_int
    lib.e264b_kat_residual.argtypes = [vp, ci, vp, ci, vp, ci, ci, vp]
    assert REC.itemsize == 192 and SLICE.itemsize == 1128
    counts = {"conforming": 0, "8x8 top": 0, "outside": 0, "ref != std": 0}
    # one slice (the commonest picture) and odd numbers of slices and records: parts of odd size in the entry point's layout
    for seed, n, n_slices in ((300, 3000, 8), (301, 501, 1), (302, 333, 3)):
        recs, sl, pool = record_draws(seed, n, n_slices)
        out = {}
        for lo in (0, 1):
            o = np.zeros((n, 384), np.int16)
            assert lib.e264b_kat_residual(recs.ctypes.data, n, sl.ctypes.data, len(sl), pool.ctypes.data, len(pool), lo, o.ctypes.data) == 0
            out[lo] = o.astype(np.int64)
        for i, r in enumerate(recs):
            s = sl[r["slice_idx"]]
            args = (int(r["kind"]), int(r["flags"]) & 1, int(r["coded"]), [int(v) for v in r["qp"]], pool[r["coef_off"]:].astype(np.int64), s["scaling4x4"], s["scaling8x8"])
            dev, ok, top = spec.mb_residual(*args, ref=True)
            std = spec.mb_residual(*args)[0]
            assert np.array_equal(out[0][i], dev), f"{n_slices} slices, record {i} (kind {r['kind']}, coded {r['coded']:#x}): not the reference's arithmetic at {np.nonzero(out[0][i] != dev)[0][:8]}"
            if ok and not top:
                assert np.array_equal(out[0][i], std), f"{n_slices} slices, conforming record {i}: differs from the standard"
            assert np.array_equal(out[1][i, :256], dev[:256]) and not out[1][i, 256:].any(), f"{n_slices} slices, record {i}: luma-only"
            lum = spec.mb_residual(*args, luma_only=True, ref=True)[0]
            assert not lum[256:].any() and np.array_equal(lum[:256], dev[:256])
            counts["conforming"] += ok and not top
            counts["8x8 top"] += ok and top
            counts["outside"] += not ok
            counts["ref != std"] += not np.array_equal(dev, std)
        print(f"e264b_kat_residual: {n} records over {n_slices} slices x 2 modes, totals so far", counts)
        if n_slices == 8:
            assert counts["conforming"] > n // 5 and counts["outside"] > n // 10 and counts["ref != std"] > 0
            kinds = {(int(r["kind"]), int(r["flags"]) & 1) for r in recs}
            assert kinds == set(KINDS)
            cdc_only = ((recs["coded"] & (spec.CODED_CB_DC | spec.CODED_CR_DC)) != 0) & ((recs["coded"] & 0xff0000) == 0)
            assert cdc_only.sum() > 100
