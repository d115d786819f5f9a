"""The pixel equations of ITU-T H.264 (04/2017) for 8-bit 4:2:0, written in numpy from the standard's text: intra prediction
(8.3.1.2, 8.3.2.2, 8.3.3, 8.3.4), luma and chroma sample interpolation (8.4.2.2.1, 8.4.2.2.2) and weighted sample
prediction (8.4.2.3).

Every function works on n draws at once, in int64.  An intra neighbourhood is three arrays: `corner` (n,) = p[-1,-1],
`top` (n, 16) = p[0..15,-1] (Intra4x4 reads 8 of them, chroma 8), `left` (n, 16) = p[-1,0..15].  `un` holds the
unavailable neighbours as the records carry them: A (left) = 1, B (top) = 2, C (top-right) = 4, D (top-left) = 8.  A mode
is only defined where the neighbours it requires are available (REQUIRES); samples of unavailable neighbours are never
read, whatever they hold.

The deviations of the reference decoder that the project reproduces are stated apart, as named functions with their
citations (ref_wp_bi_int16, ref_luma_j_int16); the standard's formulas do not contain them."""
import numpy as np

A, B, C, D = 1, 2, 4, 8

# neighbours each mode requires (the standard's "shall be used only when ... are marked as available for Intra prediction")
REQUIRES = {
    # 8.3.1.2.1-9 and 8.3.2.2.2-10: Vertical, Horizontal, DC, Diagonal-Down-Left, Diagonal-Down-Right, Vertical-Right,
    # Horizontal-Down, Vertical-Left, Horizontal-Up.  C is never required: p[3,-1] (p[7,-1]) stands in for it.
    "intra4x4": [B, A, 0, B, A | B | D, A | B | D, A | B | D, B, A],
    "intra8x8": [B, A, 0, B, A | B | D, A | B | D, A | B | D, B, A],
    # 8.3.3.1-4: Vertical, Horizontal, DC, Plane
    "intra16x16": [B, A, 0, A | B | D],
    # 8.3.4.1-4 (intra_chroma_pred_mode): DC, Horizontal, Vertical, Plane
    "chroma": [0, A, B, A | B | D],
}
# the neighbours whose availability a function distinguishes (Intra16x16 and chroma have no top-right)
NEIGHBOURS = {"intra4x4": A | B | C | D, "intra8x8": A | B | C | D, "intra16x16": A | B | D, "chroma": A | B | D}


def allowed(fn):
    """Every (mode, un) pair the standard allows for fn: the mode's required neighbours available, the others either way."""
    bits = NEIGHBOURS[fn]
    return [(m, un) for m, req in enumerate(REQUIRES[fn]) for un in range(16) if un & ~bits == 0 and un & req == 0]


def _i64(*a):
    return [np.asarray(x, np.int64) for x in a]


def _directional(N, mode, pt, pl):
    """8.3.1.2.4-9 (N = 4) and 8.3.2.2.5-10 (N = 8, on the filtered samples): pt(x) = p[x,-1], pl(y) = p[-1,y], either at
    -1 = p[-1,-1].  The equations of the two sub-clauses are the same in N."""
    out = {}
    for y in range(N):
        for x in range(N):
            if mode == 3:     # Diagonal_Down_Left
                v = (pt(2 * N - 2) + 3 * pt(2 * N - 1) + 2) >> 2 if x == y == N - 1 else (pt(x + y) + 2 * pt(x + y + 1) + pt(x + y + 2) + 2) >> 2
            elif mode == 4:   # Diagonal_Down_Right
                if x > y: v = (pt(x - y - 2) + 2 * pt(x - y - 1) + pt(x - y) + 2) >> 2
                elif x < y: v = (pl(y - x - 2) + 2 * pl(y - x - 1) + pl(y - x) + 2) >> 2
                else: v = (pt(0) + 2 * pt(-1) + pl(0) + 2) >> 2
            elif mode == 5:   # Vertical_Right
                z = 2 * x - y
                if z >= 0 and z % 2 == 0: v = (pt(x - (y >> 1) - 1) + pt(x - (y >> 1)) + 1) >> 1
                elif z > 0: v = (pt(x - (y >> 1) - 2) + 2 * pt(x - (y >> 1) - 1) + pt(x - (y >> 1)) + 2) >> 2
                elif z == -1: v = (pl(0) + 2 * pl(-1) + pt(0) + 2) >> 2
                else: v = (pl(y - 2 * x - 1) + 2 * pl(y - 2 * x - 2) + pl(y - 2 * x - 3) + 2) >> 2
            elif mode == 6:   # Horizontal_Down
                z = 2 * y - x
                if z >= 0 and z % 2 == 0: v = (pl(y - (x >> 1) - 1) + pl(y - (x >> 1)) + 1) >> 1
                elif z > 0: v = (pl(y - (x >> 1) - 2) + 2 * pl(y - (x >> 1) - 1) + pl(y - (x >> 1)) + 2) >> 2
                elif z == -1: v = (pl(0) + 2 * pl(-1) + pt(0) + 2) >> 2
                else: v = (pt(x - 2 * y - 1) + 2 * pt(x - 2 * y - 2) + pt(x - 2 * y - 3) + 2) >> 2
            elif mode == 7:   # Vertical_Left
                k = x + (y >> 1)
                v = (pt(k) + pt(k + 1) + 1) >> 1 if y % 2 == 0 else (pt(k) + 2 * pt(k + 1) + pt(k + 2) + 2) >> 2
            else:             # Horizontal_Up
                z, k = x + 2 * y, y + (x >> 1)
                if z > 2 * N - 3: v = pl(N - 1)
                elif z == 2 * N - 3: v = (pl(N - 2) + 3 * pl(N - 1) + 2) >> 2
                elif z % 2 == 0: v = (pl(k) + pl(k + 1) + 1) >> 1
                else: v = (pl(k) + 2 * pl(k + 1) + pl(k + 2) + 2) >> 2
            out[x, y] = v
    return np.stack([np.stack([out[x, y] for x in range(N)], -1) for y in range(N)], -2)


def _nxn(N, mode, un, corner, top, left):
    """Vertical, Horizontal, DC and the directional modes of an NxN block from (already substituted / filtered) samples."""
    n = corner.shape[0]
    hasA, hasB = not un & A, not un & B
    pt = lambda x: corner if x == -1 else top[:, x]
    pl = lambda y: corner if y == -1 else left[:, y]
    if mode == 0: return np.broadcast_to(top[:, None, :N], (n, N, N)).copy()
    if mode == 1: return np.broadcast_to(left[:, :N, None], (n, N, N)).copy()
    if mode == 2:
        sh = {4: 2, 8: 3}[N]
        st, sl = top[:, :N].sum(1), left[:, :N].sum(1)
        if hasA and hasB: dc = (st + sl + N) >> (sh + 1)
        elif hasA: dc = (sl + (N >> 1)) >> sh
        elif hasB: dc = (st + (N >> 1)) >> sh
        else: dc = np.full(n, 128, np.int64)   # 1 << (BitDepthY - 1)
        return np.broadcast_to(dc[:, None, None], (n, N, N)).copy()
    return _directional(N, mode, pt, pl)


def intra4x4(mode, un, corner, top, left):
    """8.3.1.2: (n, 4, 4) predicted samples; top holds p[0..7,-1] at least."""
    corner, top, left = _i64(corner, top, left)
    top = top[:, :8].copy()
    if un & C and not un & B:   # 8.3.1.2: p[4..7,-1] not available, p[3,-1] available: substituted
        top[:, 4:8] = top[:, 3:4]
    return _nxn(4, mode, un, corner, top, left)


def intra8x8_filter(un, corner, top, left):
    """8.3.2.2.1 reference sample filtering: (p'[-1,-1], p'[0..15,-1], p'[-1,0..7]), after substituting p[7,-1] for the
    unavailable p[8..15,-1].  Samples of unavailable neighbours are returned as they came in."""
    corner, top, left = _i64(corner, top, left)
    top, left = top[:, :16].copy(), left[:, :8]
    hasA, hasB, hasD = not un & A, not un & B, not un & D
    if un & C and hasB:
        top[:, 8:16] = top[:, 7:8]
    ft, fl, fc = top.copy(), left.copy(), corner.copy()
    if hasB:   # all p[x,-1], x = 0..15, available
        ft[:, 0] = (corner + 2 * top[:, 0] + top[:, 1] + 2) >> 2 if hasD else (3 * top[:, 0] + top[:, 1] + 2) >> 2
        ft[:, 1:15] = (top[:, 0:14] + 2 * top[:, 1:15] + top[:, 2:16] + 2) >> 2
        ft[:, 15] = (top[:, 14] + 3 * top[:, 15] + 2) >> 2
    if hasD:   # p[-1,-1] available
        if hasB and hasA: fc = (top[:, 0] + 2 * corner + left[:, 0] + 2) >> 2
        elif hasB: fc = (3 * corner + top[:, 0] + 2) >> 2
        elif hasA: fc = (3 * corner + left[:, 0] + 2) >> 2
        # neither p[0,-1] nor p[-1,0] available: p'[-1,-1] = p[-1,-1]
    if hasA:   # all p[-1,y], y = 0..7, available
        fl[:, 0] = (corner + 2 * left[:, 0] + left[:, 1] + 2) >> 2 if hasD else (3 * left[:, 0] + left[:, 1] + 2) >> 2
        fl[:, 1:7] = (left[:, 0:6] + 2 * left[:, 1:7] + left[:, 2:8] + 2) >> 2
        fl[:, 7] = (left[:, 6] + 3 * left[:, 7] + 2) >> 2
    return fc, ft, fl


def intra8x8(mode, un, corner, top, left):
    """8.3.2.2: (n, 8, 8) predicted samples from the filtered reference samples."""
    return _nxn(8, mode, un, *intra8x8_filter(un, corner, top, left))


def _plane_raw(corner, top, left, N, xCF, yCF, bscale):
    """The unclipped plane prediction of 8.3.3.4 (N = 16, scale 5) and 8.3.4.4 (N = 8 for 4:2:0, scale 34)."""
    pt = lambda x: corner if x == -1 else top[:, x]
    pl = lambda y: corner if y == -1 else left[:, y]
    h = N // 2
    H = sum((k + 1) * (pt(h + xCF + k) - pt(h - 2 + xCF - k)) for k in range(h + xCF))
    V = sum((k + 1) * (pl(h + yCF + k) - pl(h - 2 + yCF - k)) for k in range(h + yCF))
    a = 16 * (pl(N - 1) + pt(N - 1))
    b, c = (bscale * H + 32) >> 6, (bscale * V + 32) >> 6
    x, y = np.arange(N)[None, None, :], np.arange(N)[None, :, None]
    return (a[:, None, None] + b[:, None, None] * (x - (h - 1) - xCF) + c[:, None, None] * (y - (h - 1) - yCF) + 16) >> 5


def intra16x16_plane_raw(corner, top, left):
    corner, top, left = _i64(corner, top, left)
    return _plane_raw(corner, top, left, 16, 0, 0, 5)


def intra16x16(mode, un, corner, top, left):
    """8.3.3: (n, 16, 16) predicted samples."""
    corner, top, left = _i64(corner, top, left)
    n = corner.shape[0]
    hasA, hasB = not un & A, not un & B
    if mode == 0: return np.broadcast_to(top[:, None, :16], (n, 16, 16)).copy()
    if mode == 1: return np.broadcast_to(left[:, :16, None], (n, 16, 16)).copy()
    if mode == 2:
        st, sl = top[:, :16].sum(1), left[:, :16].sum(1)
        dc = (st + sl + 16) >> 5 if hasA and hasB else (sl + 8) >> 4 if hasA else (st + 8) >> 4 if hasB else np.full(n, 128, np.int64)
        return np.broadcast_to(dc[:, None, None], (n, 16, 16)).copy()
    return np.clip(_plane_raw(corner, top, left, 16, 0, 0, 5), 0, 255)


def chroma_plane_raw(corner, top, left):
    corner, top, left = _i64(corner, top, left)
    return _plane_raw(corner, top, left, 8, 0, 0, 34)   # 4:2:0: xCF = yCF = 0, b = (34 - 29 * (chroma_format_idc == 3)) H


def intra_chroma(mode, un, corner, top, left):
    """8.3.4 for one 8x8 chroma block of 4:2:0: (n, 8, 8) predicted samples."""
    corner, top, left = _i64(corner, top, left)
    n = corner.shape[0]
    hasA, hasB = not un & A, not un & B
    if mode == 0:   # 8.3.4.1-3: DC of each 4x4 chroma block at (xO, yO)
        out = np.empty((n, 8, 8), np.int64)
        for yO in (0, 4):
            for xO in (0, 4):
                st, sl = top[:, xO:xO + 4].sum(1), left[:, yO:yO + 4].sum(1)
                both, t, l, none = (st + sl + 4) >> 3, (st + 2) >> 2, (sl + 2) >> 2, np.full(n, 128, np.int64)
                if (xO, yO) == (0, 0) or (xO > 0 and yO > 0):   # 8.3.4.1: both, else left, else top
                    v = both if hasA and hasB else l if hasA else t if hasB else none
                elif xO > 0:                                     # 8.3.4.2 (yO = 0): the top first
                    v = t if hasB else l if hasA else none
                else:                                            # 8.3.4.3 (xO = 0, yO > 0): the left first
                    v = l if hasA else t if hasB else none
                out[:, yO:yO + 4, xO:xO + 4] = v[:, None, None]
        return out
    if mode == 1: return np.broadcast_to(left[:, :8, None], (n, 8, 8)).copy()
    if mode == 2: return np.broadcast_to(top[:, None, :8], (n, 8, 8)).copy()
    return np.clip(_plane_raw(corner, top, left, 8, 0, 0, 34), 0, 255)


# ---- inter prediction ----
def chroma_sample(plane, xInt, yInt, xFrac, yFrac):
    """8.4.2.2.2: one chroma sample per draw.  plane (H, W); integer sample positions outside it are clamped (8-229..8-232)."""
    plane = np.asarray(plane, np.int64)
    xInt, yInt, xFrac, yFrac = _i64(xInt, yInt, xFrac, yFrac)
    h, w = plane.shape
    xa, xb = np.clip(xInt, 0, w - 1), np.clip(xInt + 1, 0, w - 1)
    ya, yb = np.clip(yInt, 0, h - 1), np.clip(yInt + 1, 0, h - 1)
    return chroma_interp(plane[ya, xa], plane[ya, xb], plane[yb, xa], plane[yb, xb], xFrac, yFrac)


def chroma_interp(sA, sB, sC, sD, xFrac, yFrac):
    """8-266: the sample between sA (xInt, yInt), sB (xInt+1, yInt), sC (xInt, yInt+1), sD (xInt+1, yInt+1)."""
    sA, sB, sC, sD, xFrac, yFrac = _i64(sA, sB, sC, sD, xFrac, yFrac)
    return ((8 - xFrac) * (8 - yFrac) * sA + xFrac * (8 - yFrac) * sB + (8 - xFrac) * yFrac * sC + xFrac * yFrac * sD + 32) >> 6


def wp_default(p0, p1):
    """8.4.2.3.1, both lists: (p0 + p1 + 1) >> 1."""
    p0, p1 = _i64(p0, p1)
    return (p0 + p1 + 1) >> 1


def wp_explicit_uni(p, w, o, logWD):
    """8.4.2.3.2, one list (8-270 / 8-271); o is already scaled by 1 << (BitDepth - 8) = 1."""
    p, w, o, logWD = _i64(p, w, o, logWD)
    rnd = np.where(logWD >= 1, np.left_shift(1, np.maximum(logWD - 1, 0)), 0)
    return np.clip(np.where(logWD >= 1, (p * w + rnd) >> logWD, p * w) + o, 0, 255)


def wp_explicit_bi(p0, p1, w0, w1, o0, o1, logWD):
    """8.4.2.3.2, both lists (8-272)."""
    p0, p1, w0, w1, o0, o1, logWD = _i64(p0, p1, w0, w1, o0, o1, logWD)
    return np.clip(((p0 * w0 + p1 * w1 + np.left_shift(1, logWD)) >> (logWD + 1)) + ((o0 + o1 + 1) >> 1), 0, 255)


def wp_implicit(p0, p1, w1):
    """8.4.2.3 with implicit weights (8.4.3): logWD = 5, o0 = o1 = 0, w0 = 64 - w1, through 8-272."""
    w1 = np.asarray(w1, np.int64)
    return wp_explicit_bi(p0, p1, 64 - w1, w1, 0, 0, 5)


def bi_sum(p0, p1, w0, w1, o0, o1, logWD):
    """The pre-shift sum of the reference's explicit bi-prediction (ref_wp_bi_int16): the standard's rounding and the
    offsets folded into one term, ((o0 + o1 + 1) | 1) << logWD = ((o0 + o1 + 1) >> 1) << (logWD + 1) + 2^logWD."""
    p0, p1, w0, w1, o0, o1, logWD = _i64(p0, p1, w0, w1, o0, o1, logWD)
    return p0 * w0 + p1 * w1 + np.left_shift((o0 + o1 + 1) | 1, logWD)


def ref_wp_bi_int16(p0, p1, w0, w1, o0, o1, logWD):
    """DEVIATION of the reference decoder (edge264_inter.c:17-29, :1176-1178), reproduced by the restatement and the device:
    explicit bi-prediction computes bi_sum in int16 with saturation before the shift.  Where the sum stays in int16 this is
    8-272 exactly; where it leaves int16 the result can differ, and only at logWD 7 (32767 >> 8 = 127 where the standard
    clips to 255; at logWD <= 6 the saturated value still clips to the same 0 or 255)."""
    logWD = np.asarray(logWD, np.int64)
    return np.clip(np.clip(bi_sum(p0, p1, w0, w1, o0, o1, logWD), -32768, 32767) >> (logWD + 1), 0, 255)


# ---- luma sample interpolation ----
def _tap6(a, b, c, d, e, f):
    return a - 5 * b + 20 * c + 20 * d - 5 * e + f


# Table 8-12: the sample each (xFrac, yFrac) takes
LUMA_SAMPLE = {(0, 0): "G", (0, 1): "d", (0, 2): "h", (0, 3): "n", (1, 0): "a", (1, 1): "e", (1, 2): "i", (1, 3): "p",
               (2, 0): "b", (2, 1): "f", (2, 2): "j", (2, 3): "q", (3, 0): "c", (3, 1): "g", (3, 2): "k", (3, 3): "r"}
J_FRACTIONS = [(2, 1), (1, 2), (2, 2), (3, 2), (2, 3)]   # f, i, j, k, q: the samples that take j


def _luma_gather(plane, xInt, yInt):
    """P(dx, dy): the full sample at (xInt + dx, yInt + dy) of each draw in the (H, W) plane, the position clamped into
    the picture (8-228, 8-229)."""
    plane = np.asarray(plane)
    xInt, yInt = _i64(xInt, yInt)
    h, w = plane.shape
    return lambda dx, dy: plane[np.clip(yInt + dy, 0, h - 1), np.clip(xInt + dx, 0, w - 1)].astype(np.int64)


def _luma_samples(P, jval):
    """8-243..8-261: every sample of Table 8-12 by name, from the full samples P and the centre sample j"""
    clip = lambda v: np.clip(v, 0, 255)
    b1, h1 = _tap6(*[P(dx, 0) for dx in range(-2, 4)]), _tap6(*[P(0, dy) for dy in range(-2, 4)])      # 8-241, 8-242
    s1, m1 = _tap6(*[P(dx, 1) for dx in range(-2, 4)]), _tap6(*[P(1, dy) for dy in range(-2, 4)])
    b, h, s, m = (clip((v + 16) >> 5) for v in (b1, h1, s1, m1))                                    # 8-243, 8-244, 8-247, 8-248
    G, H, M, j = P(0, 0), P(1, 0), P(0, 1), jval
    avg = lambda u, v: (u + v + 1) >> 1
    return {"G": G, "b": b, "h": h, "j": j, "a": avg(G, b), "c": avg(H, b), "d": avg(G, h), "n": avg(M, h),      # 8-250..8-257
            "f": avg(b, j), "i": avg(h, j), "k": avg(j, m), "q": avg(j, s),
            "e": avg(b, h), "g": avg(b, m), "p": avg(h, s), "r": avg(m, s)}                           # 8-258..8-261


def luma_j1(P):
    """8-245: j1 = cc - 5 dd + 20 h1 + 20 m1 - 5 ee + ff, from the vertical intermediates of columns -2..3"""
    return _tap6(*[_tap6(*[P(dx, dy) for dy in range(-2, 4)]) for dx in range(-2, 4)])


def luma_sample(plane, xInt, yInt, xFrac, yFrac):
    """8.4.2.2.1: one luma sample per draw at integer position (xInt, yInt) and quarter-sample fraction (xFrac, yFrac);
    positions outside the plane are clamped."""
    P = _luma_gather(plane, xInt, yInt)
    smp = _luma_samples(P, np.clip((luma_j1(P) + 512) >> 10, 0, 255))                             # 8-246
    xFrac, yFrac = _i64(xFrac, yFrac)
    return np.select([(xFrac == fx) & (yFrac == fy) for fx, fy in LUMA_SAMPLE], [smp[v] for v in LUMA_SAMPLE.values()])


def luma_j_int16(P, hfirst):
    """ref_luma_j_int16's centre sample from the full samples P, and its inner sum t unwrapped"""
    s6 = ([_tap6(*[P(dx, dy) for dx in range(-2, 4)]) for dy in range(-2, 4)] if hfirst else      # b1 of rows -2..3
          [_tap6(*[P(dx, dy) for dy in range(-2, 4)]) for dx in range(-2, 4)])                     # h1 of columns -2..3
    af, be, cd = s6[0] + s6[5], s6[1] + s6[4], s6[2] + s6[3]
    t = ((af - be) >> 2) + (cd - be)
    t16 = ((t + 32768) & 65535) - 32768
    return np.clip(((t16 >> 2) + cd + 32) >> 6, 0, 255), t


def luma_j_inner(plane, xInt, yInt, xFrac):
    """the inner sum t of ref_luma_j_int16, unwrapped, in the pass order xFrac selects"""
    P = _luma_gather(plane, xInt, yInt)
    return np.where(np.asarray(xFrac) == 2, luma_j_int16(P, True)[1], luma_j_int16(P, False)[1])


def ref_luma_j_int16(plane, xInt, yInt, xFrac, yFrac):
    """DEVIATION of the reference decoder (edge264_inter.c:4-9, :559-640), reproduced by the restatement and the device:
    j is ((t >> 2) + (c+d) + 32) >> 6 with t = ((a+f - (b+e)) >> 2) + (c+d - (b+e)) WRAPPED to int16, a..f the six
    first-pass sums, horizontal first for xFrac 2 (f, j, q) and vertical first for odd xFrac (i, k).  Without the wrap
    this is (j1 + 512) >> 10 exactly (nested floors of integer sums); with it, it differs where t leaves int16."""
    P = _luma_gather(plane, xInt, yInt)
    xFrac, yFrac = _i64(xFrac, yFrac)
    smp = _luma_samples(P, np.where(xFrac == 2, luma_j_int16(P, True)[0], luma_j_int16(P, False)[0]))
    return np.select([(xFrac == fx) & (yFrac == fy) for fx, fy in LUMA_SAMPLE], [smp[v] for v in LUMA_SAMPLE.values()])
