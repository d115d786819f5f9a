"""Residual reconstruction of ITU-T H.264 (04/2017) for 8-bit 4:2:0, written in numpy from the standard's text: scaling
(8.5.9, 8.5.12.1, 8.5.13.1), the 4x4 and 8x8 inverse transforms (8.5.12.2, 8.5.13.2), the Intra16x16 luma DC transform
(8.5.10), the 4:2:0 chroma DC transform (8.5.11.1, 8.5.11.2) and picture construction (8.5.14).

Every function works on n draws at once, in int64.  Blocks are (n, N, N) arrays indexed [row][column] (the levels of a
record, records.h, are in this raster order); weight matrices are (n, N, N) or (N, N) in the same order, qP is (n,).  The
transforms run the horizontal pass first, as the text does ("each (horizontal) row ... then each (vertical) column").

For each function a companion (*_ok) says whether a draw keeps every value the text bounds inside -2^15 .. 2^15 - 1
(-2^(7 + BitDepth) .. 2^(7 + BitDepth) - 1 at BitDepth 8): d, e, f, g, h of the 4x4 path; d, e, f, g, h, k, m of the 8x8
path; f and dcY of the luma DC; f and dcC of the chroma DC.  A bitstream whose draw fails it is not conforming.

The arithmetic of the reference decoder that the project reproduces is stated apart, as named functions with their
citations (ref_*); the standard's formulas do not contain it."""
import numpy as np

LO, HI = -(1 << 15), (1 << 15) - 1

# 8-315: the v matrix of normAdjust4x4, rows m = qP % 6
V4 = np.array([[10, 16, 13], [11, 18, 14], [13, 20, 16], [14, 23, 18], [16, 25, 20], [18, 29, 23]], np.int64)
# 8-318: the v matrix of normAdjust8x8
V8 = np.array([[20, 18, 32, 19, 25, 24], [22, 19, 35, 21, 28, 26], [26, 23, 42, 24, 33, 31],
               [28, 25, 45, 26, 35, 33], [32, 28, 51, 30, 40, 38], [36, 32, 58, 34, 46, 43]], np.int64)


def class4(i, j):
    """8-314: the column of v that normAdjust4x4(m, i, j) takes."""
    return 0 if i % 2 == 0 and j % 2 == 0 else 1 if i % 2 == 1 and j % 2 == 1 else 2


def class8(i, j):
    """8-317: the column of v that normAdjust8x8(m, i, j) takes."""
    if i % 4 == 0 and j % 4 == 0: return 0
    if i % 2 == 1 and j % 2 == 1: return 1
    if i % 4 == 2 and j % 4 == 2: return 2
    if (i % 4 == 0 and j % 2 == 1) or (i % 2 == 1 and j % 4 == 0): return 3
    if (i % 4 == 0 and j % 4 == 2) or (i % 4 == 2 and j % 4 == 0): return 4
    return 5


CLASS4 = np.array([[class4(i, j) for j in range(4)] for i in range(4)])
CLASS8 = np.array([[class8(i, j) for j in range(8)] for i in range(8)])

# Table 8-13 and Table 8-14, frame (zig-zag) scan: the raster position (row * N + column) of scan index idx
ZIGZAG4 = np.array([0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15])
ZIGZAG8 = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,
                    7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
                    39, 46, 53, 60, 61, 54, 47, 55, 62, 63])

# Table 7-3 / 7-4 (scan order) and Flat_4x4_16 / Flat_8x8_16 (7.4.2.1.1.1)
FLAT_4x4_16 = np.full(16, 16, np.int64)
FLAT_8x8_16 = np.full(64, 16, np.int64)
DEFAULT_4x4_INTRA = np.array([6, 13, 13, 20, 20, 20, 28, 28, 28, 28, 32, 32, 32, 37, 37, 42], np.int64)
DEFAULT_4x4_INTER = np.array([10, 14, 14, 20, 20, 20, 24, 24, 24, 24, 27, 27, 27, 30, 30, 34], np.int64)
DEFAULT_8x8_INTRA = np.array([6, 10, 10, 13, 11, 13, 16, 16, 16, 16, 18, 18, 18, 18, 18, 23, 23, 23, 23, 23, 23, 25, 25, 25,
                              25, 25, 25, 25, 27, 27, 27, 27, 27, 27, 27, 27, 29, 29, 29, 29, 29, 29, 29, 31, 31, 31, 31,
                              31, 31, 33, 33, 33, 33, 33, 36, 36, 36, 36, 38, 38, 38, 40, 40, 42], np.int64)
DEFAULT_8x8_INTER = np.array([9, 13, 13, 15, 13, 15, 17, 17, 17, 17, 19, 19, 19, 19, 19, 21, 21, 21, 21, 21, 21, 22, 22, 22,
                              22, 22, 22, 22, 24, 24, 24, 24, 24, 24, 24, 24, 25, 25, 25, 25, 25, 25, 25, 27, 27, 27, 27,
                              27, 27, 28, 28, 28, 28, 28, 30, 30, 30, 30, 32, 32, 32, 33, 33, 35], np.int64)


def weight_matrix(scan_list):
    """8.5.6 / 8.5.7 inverse frame scan of a scaling list (16 or 64 entries, scan order) into weightScale (N, N)."""
    lst = np.asarray(scan_list, np.int64)
    N = 4 if len(lst) == 16 else 8
    out = np.empty(N * N, np.int64)
    out[ZIGZAG4 if N == 4 else ZIGZAG8] = lst
    return out.reshape(N, N)


def _i64(*a):
    return [np.asarray(x, np.int64) for x in a]


def _in16(*arrays):
    """per draw: every value of every array inside LO..HI (arrays are (n, ...))"""
    ok = np.ones(len(arrays[0]), bool)
    for a in arrays:
        ok &= ((a >= LO) & (a <= HI)).reshape(len(a), -1).all(1)
    return ok


def _wrap(x, bits):
    """two's complement wrap of x to a signed `bits`-bit value"""
    h = 1 << (bits - 1)
    return ((np.asarray(x, np.int64) + h) & ((1 << bits) - 1)) - h


def level_scale4x4(m, w):
    """8-313: LevelScale4x4(m, i, j) = weightScale4x4(i, j) * normAdjust4x4(m, i, j); m (n,), w (n, 4, 4) or (4, 4)."""
    m, w = _i64(m, w)
    return w * V4[m][:, CLASS4]


def level_scale8x8(m, w):
    """8-316: LevelScale8x8(m, i, j) = weightScale8x8(i, j) * normAdjust8x8(m, i, j)."""
    m, w = _i64(m, w)
    return w * V8[m][:, CLASS8]


# ---- 4x4 ----
def scale4x4(c, w, qP, dc=None):
    """8.5.12.1: d from the levels c.  dc (n,), when given, is d00 (Intra16x16 luma and chroma blocks: the output of the DC
    transform), else d00 is scaled like the other coefficients."""
    c, w, qP = _i64(c, w, qP)
    LS, s = level_scale4x4(qP % 6, w), (qP // 6)[:, None, None]
    d = np.where(s >= 4, (c * LS) << np.maximum(s - 4, 0), (c * LS + (1 << np.maximum(3 - s, 0))) >> np.maximum(4 - s, 0))
    if dc is not None:
        d[:, 0, 0] = np.asarray(dc, np.int64)
    return d


def _pass4(x):
    """one 1-D pass of 8.5.12.2 along the last axis: (e, f) of 8-338..8-345 (the column pass: g, h)"""
    x0, x1, x2, x3 = x[..., 0], x[..., 1], x[..., 2], x[..., 3]
    e0, e1, e2, e3 = x0 + x2, x0 - x2, (x1 >> 1) - x3, x1 + (x3 >> 1)
    return np.stack([e0, e1, e2, e3], -1), np.stack([e0 + e3, e1 + e2, e1 - e2, e0 - e3], -1)


def _t4(d):
    e, f = _pass4(d)                          # rows
    g, h = _pass4(f.swapaxes(-1, -2))         # columns
    return e, f, g.swapaxes(-1, -2), h.swapaxes(-1, -2)


def transform4x4(d):
    """8.5.12.2: r = (h + 2^5) >> 6."""
    return (_t4(np.asarray(d, np.int64))[3] + 32) >> 6


def transform4x4_ok(d):
    d = np.asarray(d, np.int64)
    return _in16(d, *_t4(d))


def residual4x4(c, w, qP, dc=None):
    return transform4x4(scale4x4(c, w, qP, dc))


def residual4x4_ok(c, w, qP, dc=None):
    return transform4x4_ok(scale4x4(c, w, qP, dc))


def max4x4(c, w, qP, dc=None):
    """the largest magnitude among the bounded values of each draw"""
    d = scale4x4(c, w, qP, dc)
    return np.max([np.abs(a).reshape(len(a), -1).max(1) for a in (d, *_t4(d))], 0)


# ---- 8x8 ----
def scale8x8(c, w, qP):
    """8.5.13.1"""
    c, w, qP = _i64(c, w, qP)
    LS, s = level_scale8x8(qP % 6, w), (qP // 6)[:, None, None]
    return np.where(s >= 6, (c * LS) << np.maximum(s - 6, 0), (c * LS + (1 << np.maximum(5 - s, 0))) >> np.maximum(6 - s, 0))


def _pass8(x, wrap=lambda v: v):
    """one 1-D pass of 8.5.13.2 along the last axis: (e, f, g) of 8-353..8-376 (the column pass: h, k, m); `wrap` is
    applied to each stage's results (identity for the standard)"""
    d = [x[..., k] for k in range(8)]
    e = [d[0] + d[4], -d[3] + d[5] - d[7] - (d[7] >> 1), d[0] - d[4], d[1] + d[7] - d[3] - (d[3] >> 1),
         (d[2] >> 1) - d[6], -d[1] + d[7] + d[5] + (d[5] >> 1), d[2] + (d[6] >> 1), d[3] + d[5] + d[1] + (d[1] >> 1)]
    e = [wrap(v) for v in e]
    f = [e[0] + e[6], e[1] + (e[7] >> 2), e[2] + e[4], e[3] + (e[5] >> 2), e[2] - e[4], (e[3] >> 2) - e[5], e[0] - e[6],
         e[7] - (e[1] >> 2)]
    f = [wrap(v) for v in f]
    g = [f[0] + f[7], f[2] + f[5], f[4] + f[3], f[6] + f[1], f[6] - f[1], f[4] - f[3], f[2] - f[5], f[0] - f[7]]
    g = [wrap(v) for v in g]
    return np.stack(e, -1), np.stack(f, -1), np.stack(g, -1)


def _t8(d):
    e, f, g = _pass8(d)
    h, k, m = (a.swapaxes(-1, -2) for a in _pass8(g.swapaxes(-1, -2)))
    return e, f, g, h, k, m


def transform8x8(d):
    """8.5.13.2: r = (m + 2^5) >> 6."""
    return (_t8(np.asarray(d, np.int64))[5] + 32) >> 6


def transform8x8_ok(d):
    d = np.asarray(d, np.int64)
    return _in16(d, *_t8(d))


def transform8x8_m(d):
    """m of 8.5.13.2 (the value before the final rounding)"""
    return _t8(np.asarray(d, np.int64))[5]


def residual8x8(c, w, qP):
    return transform8x8(scale8x8(c, w, qP))


def residual8x8_ok(c, w, qP):
    return transform8x8_ok(scale8x8(c, w, qP))


def max8x8(c, w, qP):
    d = scale8x8(c, w, qP)
    return np.max([np.abs(a).reshape(len(a), -1).max(1) for a in (d, *_t8(d))], 0)


# ---- DC transforms ----
_A4 = np.array([[1, 1, 1, 1], [1, 1, -1, -1], [1, -1, -1, 1], [1, -1, 1, -1]], np.int64)
_A2 = np.array([[1, 1], [1, -1]], np.int64)


def luma_dc_f(c):
    """8-320: f = A c A of the (n, 4, 4) Intra16x16 DC levels"""
    return _A4 @ np.asarray(c, np.int64) @ _A4


def luma_dc(c, w00, qP):
    """8.5.10, 8-321 / 8-322: dcY (n, 4, 4), one value per 4x4 luma block in raster order.  w00 (n,) is
    weightScale4x4(0, 0) of the Intra Y list."""
    w00, qP = _i64(w00, qP)
    f, LS, s = luma_dc_f(c), (w00 * V4[qP % 6, 0])[:, None, None], (qP // 6)[:, None, None]
    return np.where(s >= 6, (f * LS) << np.maximum(s - 6, 0), (f * LS + (1 << np.maximum(5 - s, 0))) >> np.maximum(6 - s, 0))


def luma_dc_ok(c, w00, qP):
    return _in16(luma_dc_f(c), luma_dc(c, w00, qP))


def chroma_dc_f(c):
    """8-328 (4:2:0): f = A c A of the (n, 2, 2) chroma DC levels c = [[c0, c1], [c2, c3]]"""
    return _A2 @ np.asarray(c, np.int64) @ _A2


def chroma_dc(c, w00, qP):
    """8.5.11.2, 8-330 (4:2:0): dcC = ((f * LevelScale4x4(qP % 6, 0, 0)) << (qP / 6)) >> 5, dcC[i][j] the DC of chroma
    block 2 i + j; w00 is weightScale4x4(0, 0) of the block's list, qP the plane's QP'c."""
    w00, qP = _i64(w00, qP)
    return ((chroma_dc_f(c) * (w00 * V4[qP % 6, 0])[:, None, None]) << (qP // 6)[:, None, None]) >> 5


def chroma_dc_ok(c, w00, qP):
    return _in16(chroma_dc_f(c), chroma_dc(c, w00, qP))


def dc_only4x4(dc):
    """8.5.12 on a block whose only nonzero d is d00 = dc (an Intra16x16 or chroma block without AC levels)"""
    dc = np.asarray(dc, np.int64)
    d = np.zeros((len(dc), 4, 4), np.int64)
    d[:, 0, 0] = dc
    return transform4x4(d)


def dc_only4x4_ok(dc):
    d = np.zeros((len(dc), 4, 4), np.int64)
    d[:, 0, 0] = dc
    return transform4x4_ok(d)


def construct(pred, r):
    """8.5.14 (8-357 with 8-bit samples): Clip1(pred + r)"""
    pred, r = _i64(pred, r)
    return np.clip(pred + r, 0, 255)


# ---- the reference's arithmetic (reproduced by oracle/port_recon.c and the kernels) ----
def ref_idct4x4_sat16(c, w, qP, dc=None):
    """DEVIATION (edge264_residual.c:108-172): 8.5.12 with d computed as ((c * LS) << (qP / 6) + 8) >> 4 in 32 bits, which
    equals 8-336 / 8-337 but wraps where c * LS << (qP / 6) leaves 32 bits, and the output saturated to int16.  The sums
    of e..h run in 32 bits and cannot wrap: |d| < 2^27 and every dc the DC paths produce is below 2^26."""
    c, w, qP = _i64(c, w, qP)
    d = _wrap(((c * level_scale4x4(qP % 6, w)) << (qP // 6)[:, None, None]) + 8, 32) >> 4
    if dc is not None:
        d[:, 0, 0] = np.asarray(dc, np.int64)
    h = _t4(d)[3]
    assert (np.abs(h) < 1 << 31).all()
    return np.clip((h + 32) >> 6, LO, HI)


def ref_idct8x8_int16(c, w, qP):
    """DEVIATION (edge264_residual.c:194-343): 8.5.13 in wrapping int16.  Below qP 36 d saturates to int16
    (sat16((c * LS + 2^(5 - qP/6)) >> (6 - qP/6))), from qP 36 up it wraps (int16(c * int16(LS << (qP/6 - 6))));
    every value of the two passes wraps to int16; the rounding 2^5 is added to g0j before the column pass, in int16
    (residual.c:300), and r = that pass's output >> 6."""
    c, w, qP = _i64(c, w, qP)
    LS, s = level_scale8x8(qP % 6, w), (qP // 6)[:, None, None]
    lo = np.clip((c * LS + (1 << np.maximum(5 - s, 0))) >> np.maximum(6 - s, 0), LO, HI)
    hi = _wrap(c * _wrap(LS << np.maximum(s - 6, 0), 16), 16)
    d = np.where(s < 6, lo, hi)
    w16 = lambda v: _wrap(v, 16)
    g = _pass8(d, w16)[2].swapaxes(-1, -2)       # columns on the last axis
    g[..., 0] = w16(g[..., 0] + 32)
    m = _pass8(g, w16)[2].swapaxes(-1, -2)
    return m >> 6


def ref_dc_only_trunc16(dc):
    """DEVIATION (edge264_residual.c:174-178 add_dc4x4, :401-409, :480-484): a block without AC levels takes
    (dc + 32) >> 6 truncated to int16 at every sample."""
    v = _wrap((np.asarray(dc, np.int64) + 32) >> 6, 16)
    return np.broadcast_to(v[:, None, None], (len(v), 4, 4)).copy()


def ref_luma_dc_wrap32(c, w00, qP):
    """DEVIATION (edge264_residual.c:388-392): dcY = (f * (LevelScale4x4(qP % 6, 0, 0) << (qP / 6)) + 32) >> 6 in 32 bits,
    which equals 8-321 / 8-322 but wraps where the product leaves 32 bits."""
    w00, qP = _i64(w00, qP)
    LS = ((w00 * V4[qP % 6, 0]) << (qP // 6))[:, None, None]
    return _wrap(luma_dc_f(c) * LS + 32, 32) >> 6


def ref_chroma_dc_wrap32(c, w00, qP):
    """DEVIATION (edge264_residual.c:472-475): 8-330 with f * (LevelScale4x4(qP % 6, 0, 0) << (qP / 6)) in 32 bits,
    wrapping where it leaves them."""
    w00, qP = _i64(w00, qP)
    LS = ((w00 * V4[qP % 6, 0]) << (qP // 6))[:, None, None]
    return _wrap(chroma_dc_f(c) * LS, 32) >> 5


def ref_add_int16(pred, r):
    """DEVIATION (the reference's 16-bit adds of prediction and residual): Clip1 of pred + r wrapped to int16."""
    pred, r = _i64(pred, r)
    return np.clip(_wrap(pred + r, 16), 0, 255)


# ---- one macroblock ----
MBK_I4x4, MBK_I8x8, MBK_I16x16, MBK_IPCM, MBK_INTER = 0, 1, 2, 3, 4
CODED_Y_DC, CODED_CB_DC, CODED_CR_DC = 1 << 24, 1 << 25, 1 << 26


def blk_xy(b):
    """6.4.3: the column and row (in 4x4 blocks) of luma4x4BlkIdx b"""
    return (b & 1) | ((b >> 1) & 2), ((b >> 1) & 1) | ((b >> 2) & 2)


def mb_residual(kind, t8, coded, qp, levels, sc4, sc8, luma_only=False, ref=False):
    """The residual of one 4:2:0 macroblock that is not I_PCM, (384,): Y 16x16 raster, then Cb 8x8, Cr 8x8.

    kind, t8 (transform_size_8x8_flag), coded (CODED_* bits), qp (QP'Y, QP'c of Cb, Cr) are the record's fields; levels is
    the record's coefficient run in the order of records.h; sc4 (6, 16) and sc8 (2, 64) the slice's weight matrices in
    raster order, lists Y/Cb/Cr intra, Y/Cb/Cr inter and Y intra/inter.  The 4x4 list of a block is 1 + plane + 3 inter
    for chroma and 3 inter for luma, the 8x8 list is inter.  luma_only leaves the chroma residual zero.  With ref, the
    reference's arithmetic (ref_*) replaces the standard's.

    Returns (residual, ok, top): ok says every block and DC transform kept its bounded values inside int16 (a conforming
    macroblock), top that an 8x8 block's m reached 2^15 - 32 (where ref_idct8x8_int16's rounding leaves int16)."""
    lv = np.asarray(levels, np.int64)
    sc4, sc8 = np.asarray(sc4, np.int64).reshape(6, 4, 4), np.asarray(sc8, np.int64).reshape(2, 8, 8)
    inter, i16 = int(kind == MBK_INTER), kind == MBK_I16x16
    res = np.zeros(384, np.int64)
    Y = res[:256].reshape(16, 16)
    ok, top, pos = True, False, 0
    one = lambda v: np.array([v], np.int64)
    dcY = np.zeros((4, 4), np.int64)
    if coded & CODED_Y_DC:
        c = lv[pos:pos + 16].reshape(1, 4, 4)
        pos += 16
        dcY = (ref_luma_dc_wrap32 if ref else luma_dc)(c, one(sc4[0, 0, 0]), one(qp[0]))[0]
        ok &= bool(luma_dc_ok(c, one(sc4[0, 0, 0]), one(qp[0]))[0])
    if t8:
        blocks = [i8 for i8 in range(4) if (coded >> (4 * i8)) & 1]
        if blocks:
            k = len(blocks)
            c = lv[pos:pos + 64 * k].reshape(k, 8, 8)
            pos += 64 * k
            q = np.full(k, qp[0])
            r = ref_idct8x8_int16(c, sc8[inter], q) if ref else residual8x8(c, sc8[inter], q)
            ok &= bool(residual8x8_ok(c, sc8[inter], q).all())
            top |= bool((transform8x8_m(scale8x8(c, sc8[inter], q)) >= HI - 31).any())
            for n, i8 in enumerate(blocks):
                Y[(i8 >> 1) * 8:(i8 >> 1) * 8 + 8, (i8 & 1) * 8:(i8 & 1) * 8 + 8] = r[n]
    else:
        blocks = [b for b in range(16) if (coded >> b) & 1]
        if blocks:
            k = len(blocks)
            c = lv[pos:pos + 16 * k].reshape(k, 4, 4)
            pos += 16 * k
            q = np.full(k, qp[0])
            dc = np.array([dcY[blk_xy(b)[1], blk_xy(b)[0]] for b in blocks]) if i16 else None
            r = ref_idct4x4_sat16(c, sc4[3 * inter], q, dc) if ref else residual4x4(c, sc4[3 * inter], q, dc)
            ok &= bool(residual4x4_ok(c, sc4[3 * inter], q, dc).all())
            for n, b in enumerate(blocks):
                x, y = blk_xy(b)
                Y[y * 4:y * 4 + 4, x * 4:x * 4 + 4] = r[n]
        if i16 and coded & CODED_Y_DC:
            rest = [b for b in range(16) if not (coded >> b) & 1]
            if rest:
                dc = np.array([dcY[blk_xy(b)[1], blk_xy(b)[0]] for b in rest])
                r = ref_dc_only_trunc16(dc) if ref else dc_only4x4(dc)
                ok &= bool(dc_only4x4_ok(dc).all())
                for n, b in enumerate(rest):
                    x, y = blk_xy(b)
                    Y[y * 4:y * 4 + 4, x * 4:x * 4 + 4] = r[n]
    if luma_only:
        return res, ok, top
    any_dc = bool(coded & (CODED_CB_DC | CODED_CR_DC))
    dcC = np.zeros((2, 2, 2), np.int64)
    if any_dc:
        c = lv[pos:pos + 8].reshape(2, 2, 2)
        pos += 8
        w00, q = np.array([sc4[1 + 3 * inter, 0, 0], sc4[2 + 3 * inter, 0, 0]]), np.array([qp[1], qp[2]])
        dcC = (ref_chroma_dc_wrap32 if ref else chroma_dc)(c, w00, q)
        ok &= bool(chroma_dc_ok(c, w00, q).all())
    for pl in range(2):
        C = res[256 + 64 * pl:320 + 64 * pl].reshape(8, 8)
        lst = sc4[1 + pl + 3 * inter]
        for i in range(4):
            if (coded >> (16 + 4 * pl + i)) & 1:
                c = lv[pos:pos + 16].reshape(1, 4, 4)
                pos += 16
                dc, q = one(dcC[pl, i >> 1, i & 1]), one(qp[1 + pl])
                r = (ref_idct4x4_sat16 if ref else residual4x4)(c, lst, q, dc)
                ok &= bool(residual4x4_ok(c, lst, q, dc)[0])
            elif any_dc:
                dc = one(dcC[pl, i >> 1, i & 1])
                r = (ref_dc_only_trunc16 if ref else dc_only4x4)(dc)
                ok &= bool(dc_only4x4_ok(dc)[0])
            else:
                continue
            C[(i >> 1) * 4:(i >> 1) * 4 + 4, (i & 1) * 4:(i & 1) * 4 + 4] = r[0]
    return res, ok, top
