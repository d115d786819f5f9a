"""The deblocking filter of ITU-T H.264 (04/2017), clause 8.7, for 8-bit 4:2:0 frame pictures, written in int64 numpy from
the standard's text.  There is no MBAFF and no field picture here, so mixedModeEdgeFlag is 0 throughout and vertical
vector differences are counted in quarter frame samples.

The parts, each usable on its own:
  - the tables: Table 8-15 (QPc), Table 8-16 (alpha', beta'), Table 8-17 (t'C0), typed from the standard;
  - boundary_strength: 8.7.2.1 between two 4x4 luma blocks given as the fields the records carry, every rule a named
    condition;
  - thresholds: 8.7.2.2, qPav, indexA / indexB and the table look-ups;
  - filter_luma / filter_chroma: 8.7.2.3 and 8.7.2.4 on many lines at once (samples p3..q3, or p1..q1 for chroma);
  - deblock_pictures: 8.7 and 8.7.1 over a batch of pictures of one geometry in the layout of E264PicDesc (records.h),
    with the records and slices that describe them.  It returns the deblocked pictures and what it derived, with
    coverage counts of the branches it took.

Every function works on arrays of any shape and broadcasts its arguments; samples and results are int64."""
import collections
import numpy as np

I = np.int64

# ---- tables ----
# Table 8-15: QPc as a function of qPI (qPI < 30: QPc = qPI)
QPC = list(range(30)) + [29, 30, 31, 32, 32, 33, 34, 34, 35, 35, 36, 36, 37, 37, 37, 38, 38, 38, 39, 39, 39, 39]
# Table 8-16: alpha' by indexA and beta' by indexB, 0..51 (both 0 for indexA / indexB 0..15)
ALPHA = [0] * 16 + [4, 4, 5, 6, 7, 8, 9, 10, 12, 13, 15, 17, 20, 22, 25, 28, 32, 36, 40, 45, 50, 56, 63, 71, 80, 90, 101, 113,
                    127, 144, 162, 182, 203, 226, 255, 255]
BETA = [0] * 16 + [2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13, 14, 14, 15, 15, 16, 16,
                   17, 17, 18, 18]
# Table 8-17: t'C0 by indexA 0..51, one row per bS 1, 2, 3
TC0 = [
    [0] * 23 + [1] * 10 + [2] * 4 + [3] * 3 + [4] * 3 + [5, 6, 6, 7, 8, 9, 10, 11, 13],          # bS = 1
    [0] * 21 + [1] * 10 + [2] * 4 + [3] * 3 + [4] * 2 + [5, 5, 6, 7, 8, 8, 10, 11, 12, 13, 15, 17],   # bS = 2
    [0] * 17 + [1] * 10 + [2] * 4 + [3] * 3 + [4] * 3 + [5, 6, 6, 7, 8, 9, 10, 11, 13, 14, 16, 18, 20, 23, 25],   # bS = 3
]
assert len(QPC) == len(ALPHA) == len(BETA) == 52 and all(len(r) == 52 for r in TC0)
_ALPHA, _BETA, _TC0 = np.array(ALPHA, I), np.array(BETA, I), np.array([[0] * 52] + TC0, I)   # _TC0[bS][indexA], row 0 unused

# the record ABI (edge264_b200/csrc/records.h)
MBK_INTER = 4
MBF_T8x8, MBF_EDGE_L, MBF_EDGE_T, MBF_DEBLOCK = 0x01, 0x02, 0x04, 0x08
REC = np.dtype([("kind", "u1"), ("flags", "u1"), ("qp", "u1", 3), ("chroma_mode", "u1"), ("i16_mode", "u1"), ("slice_idx", "u1"),
                ("coded", "<u4"), ("coef_off", "<u4"), ("modes", "u1", 16), ("ref_idx", "i1", (2, 4)), ("ref_pic", "i1", (2, 4)),
                ("err", "u1"), ("reserved", "u1", 15), ("mv", "<i2", (2, 16, 2))])
SLICE = np.dtype([("filter_offset_a", "i1"), ("filter_offset_b", "i1"), ("deblock_idc", "u1"), ("slice_type", "u1"), ("wp_mode", "u1"),
                  ("luma_log2_wd", "u1"), ("chroma_log2_wd", "u1"), ("reserved", "u1"), ("wp_w", "<i2", (2, 16, 3)), ("wp_o", "<i2", (2, 16, 3)),
                  ("implicit_w1", "<i2", (16, 16)), ("scaling4x4", "u1", (6, 16)), ("scaling8x8", "u1", (2, 64))])
PICDESC = np.dtype([(n, "<i4") for n in ("width_mbs", "height_mbs", "stride_y", "stride_c", "plane_y", "frame_bytes", "dst_slot",
                                          "n_slices", "n_coefs", "any_deblock", "n_intra", "staging")]
                   + [("err_pic", "u1"), ("luma_only", "u1"), ("reserved", "u1", 2), ("taint", "<u4")])
assert REC.itemsize == 192 and SLICE.itemsize == 1128 and PICDESC.itemsize == 56


def blk_z(x, y):
    """luma4x4BlkIdx of the 4x4 block in column x, row y of a macroblock (6.4.3)."""
    return (x & 1) | ((y & 1) << 1) | ((x & 2) << 1) | ((y & 2) << 2)


def clip3(lo, hi, v):
    return np.minimum(np.maximum(v, lo), hi)


def clip1(v):
    return clip3(0, 255, v)


# ---- 8.7.2.1 boundary strength ----
BS_RULES = ["intra_mb_edge", "intra_internal", "coefficients", "pictures_or_count", "one_vector_each", "two_pictures_paired",
            "one_picture_twice", "none"]


def far(a, b):
    """Two vectors (..., 2) in quarter frame samples differ by 4 or more horizontally or vertically."""
    return (np.abs(np.asarray(a, I) - np.asarray(b, I)) >= 4).any(-1)


def boundary_strength(intra_p, intra_q, coef_p, coef_q, pic_p, pic_q, mv_p, mv_q, mb_edge):
    """bS of the edge between the block containing p0 and the block containing q0, and the rule that decided it (an index
    into BS_RULES).  intra_*: the macroblock is intra; coef_*: the block's transform coefficients are not all zero (the 4x4
    block, or the 8x8 block containing it under transform_size_8x8_flag); pic_* (..., 2): the reference picture of each
    list, -1 where the list is unused; mv_* (..., 2, 2): [list][x, y]; mb_edge: the edge is a macroblock edge."""
    intra_p, intra_q, coef_p, coef_q, mb_edge = [np.asarray(x, bool) for x in (intra_p, intra_q, coef_p, coef_q, mb_edge)]
    pic_p, pic_q, mv_p, mv_q = [np.asarray(x, I) for x in (pic_p, pic_q, mv_p, mv_q)]
    intra = intra_p | intra_q
    # bS 4: either sample in an intra macroblock and the edge is a macroblock edge; bS 3: intra on an internal edge
    r_intra_mb, r_intra_in = intra & mb_edge, intra & ~mb_edge
    # bS 2: either block contains non-zero transform coefficient levels
    r_coef = coef_p | coef_q
    # bS 1: different reference pictures or a different number of motion vectors.  Pictures are compared as pictures,
    # whichever list or index names them: the two lists' pictures as a multiset, an unused list counting as -1
    r_pics = (np.sort(pic_p, -1) != np.sort(pic_q, -1)).any(-1)
    # from here p and q predict from the same pictures with as many vectors
    n_vec = (pic_p >= 0).sum(-1)
    # one motion vector each: the vectors of the lists in use
    lp, lq = np.where(pic_p[..., 0] >= 0, 0, 1), np.where(pic_q[..., 0] >= 0, 0, 1)
    vp = np.take_along_axis(mv_p, lp[..., None, None], -2)[..., 0, :]
    vq = np.take_along_axis(mv_q, lq[..., None, None], -2)[..., 0, :]
    r_one = (n_vec == 1) & far(vp, vq)
    straight = far(mv_p[..., 0, :], mv_q[..., 0, :]) | far(mv_p[..., 1, :], mv_q[..., 1, :])
    crossed = far(mv_p[..., 0, :], mv_q[..., 1, :]) | far(mv_p[..., 1, :], mv_q[..., 0, :])
    # two motion vectors for two different pictures: the two vectors for the same picture are compared
    two_diff = (n_vec == 2) & (pic_p[..., 0] != pic_p[..., 1])
    r_two_paired = two_diff & np.where(pic_p[..., 0] == pic_q[..., 0], straight, crossed)
    # two motion vectors for the same picture on both sides: both pairings must differ
    r_twice = (n_vec == 2) & (pic_p[..., 0] == pic_p[..., 1]) & straight & crossed
    conds = [r_intra_mb, r_intra_in, r_coef, r_pics, r_one, r_two_paired, r_twice]
    bs = np.select(conds, [4, 3, 2, 1, 1, 1, 1], 0)
    rule = np.select(conds, list(range(7)), 7)
    return bs, rule


def block_fields(kind, flags, coded, ref_idx, ref_pic, mv, b):
    """The fields boundary_strength takes for 4x4 block b of records given as arrays (..., ) kind / flags / coded,
    (..., 2, 4) ref_idx / ref_pic, (..., 2, 16, 2) mv."""
    coded, flags = np.asarray(coded, np.int64), np.asarray(flags, np.int64)
    intra = np.asarray(kind) != MBK_INTER
    coef = np.where(flags & MBF_T8x8, (coded >> (b & ~3)) & 15, (coded >> b) & 1) != 0
    pic = np.where(np.asarray(ref_idx)[..., b >> 2] < 0, -1, np.asarray(ref_pic, I)[..., b >> 2])
    return intra, coef, pic, np.asarray(mv, I)[..., :, b, :]


def rec_fields(r, b):
    return block_fields(r["kind"], r["flags"], r["coded"], r["ref_idx"], r["ref_pic"], r["mv"], b)


# ---- 8.7.2.2 thresholds ----
def thresholds(qp_p, qp_q, offset_a, offset_b, bs=None):
    """qPav, the unclipped indexA / indexB, and alpha, beta (and t'C0 of bs when given) for an edge between macroblocks of
    quantisation parameters qp_p and qp_q (QPY for luma, the plane's QPc for chroma), FilterOffsetA / B of the slice that
    contains q0."""
    qpav = (np.asarray(qp_p, I) + np.asarray(qp_q, I) + 1) >> 1
    raw_a, raw_b = qpav + np.asarray(offset_a, I), qpav + np.asarray(offset_b, I)
    ia, ib = clip3(0, 51, raw_a), clip3(0, 51, raw_b)
    out = dict(qpav=qpav, raw_a=raw_a, raw_b=raw_b, index_a=ia, index_b=ib, alpha=_ALPHA[ia], beta=_BETA[ib])
    if bs is not None:
        out["tc0"] = _TC0[np.clip(np.asarray(bs, I), 0, 3), ia]
    return out


# ---- 8.7.2.3 / 8.7.2.4 sample filters ----
def filter_luma(s, bs, alpha, beta, tc0):
    """Lines s (..., 8) = p3, p2, p1, p0, q0, q1, q2, q3 across a luma edge: the filtered lines and the branches taken."""
    s = np.asarray(s, I)
    p3, p2, p1, p0, q0, q1, q2, q3 = np.moveaxis(s, -1, 0)
    bs, alpha, beta, tc0 = [np.asarray(x, I) for x in (bs, alpha, beta, tc0)]
    f = (bs != 0) & (np.abs(p0 - q0) < alpha) & (np.abs(p1 - p0) < beta) & (np.abs(q1 - q0) < beta)   # filterSamplesFlag
    ap, aq = np.abs(p2 - p0), np.abs(q2 - q0)
    # bS < 4 (8.7.2.3), chromaEdgeFlag 0
    tc = tc0 + (ap < beta) + (aq < beta)
    raw = (((q0 - p0) << 2) + (p1 - q1) + 4) >> 3
    delta = clip3(-tc, tc, raw)
    w = [p3, p2, np.where(ap < beta, p1 + clip3(-tc0, tc0, (p2 + ((p0 + q0 + 1) >> 1) - (p1 << 1)) >> 1), p1), clip1(p0 + delta),
         clip1(q0 - delta), np.where(aq < beta, q1 + clip3(-tc0, tc0, (q2 + ((p0 + q0 + 1) >> 1) - (q1 << 1)) >> 1), q1), q2, q3]
    # bS == 4 (8.7.2.4), chromaStyleFilteringFlag 0
    small = np.abs(p0 - q0) < ((alpha >> 2) + 2)
    sp, sq = (ap < beta) & small, (aq < beta) & small
    st = [p3, np.where(sp, (2 * p3 + 3 * p2 + p1 + p0 + q0 + 4) >> 3, p2), np.where(sp, (p2 + p1 + p0 + q0 + 2) >> 2, p1),
          np.where(sp, (p2 + 2 * p1 + 2 * p0 + 2 * q0 + q1 + 4) >> 3, (2 * p1 + p0 + q1 + 2) >> 2),
          np.where(sq, (p1 + 2 * p0 + 2 * q0 + 2 * q1 + q2 + 4) >> 3, (2 * q1 + q0 + p1 + 2) >> 2),
          np.where(sq, (p0 + q0 + q1 + q2 + 2) >> 2, q1), np.where(sq, (2 * q3 + 3 * q2 + q1 + q0 + p0 + 4) >> 3, q2), q3]
    strong = bs == 4
    out = np.where(f[..., None], np.where(strong[..., None], np.stack(st, -1), np.stack(w, -1)), s)
    weak = f & ~strong
    br = dict(filtered=f, delta_clipped=weak & (np.abs(raw) > tc), strong_p_3tap=f & strong & sp, strong_p_1tap=f & strong & ~sp, strong_q_3tap=f & strong & sq,
              strong_q_1tap=f & strong & ~sq, weak_p1=weak & (ap < beta), weak_q1=weak & (aq < beta),
              p0_clip_0=weak & (p0 + delta < 0), p0_clip_255=weak & (p0 + delta > 255), q0_clip_0=weak & (q0 - delta < 0),
              q0_clip_255=weak & (q0 - delta > 255))
    return out, br


def filter_chroma(s, bs, alpha, beta, tc0):
    """Lines s (..., 4) = p1, p0, q0, q1 across a chroma edge (4:2:0, chromaStyleFilteringFlag 1)."""
    s = np.asarray(s, I)
    p1, p0, q0, q1 = np.moveaxis(s, -1, 0)
    bs, alpha, beta, tc0 = [np.asarray(x, I) for x in (bs, alpha, beta, tc0)]
    f = (bs != 0) & (np.abs(p0 - q0) < alpha) & (np.abs(p1 - p0) < beta) & (np.abs(q1 - q0) < beta)
    tc = tc0 + 1
    raw = (((q0 - p0) << 2) + (p1 - q1) + 4) >> 3
    delta = clip3(-tc, tc, raw)
    w = np.stack([p1, clip1(p0 + delta), clip1(q0 - delta), q1], -1)
    st = np.stack([p1, (2 * p1 + p0 + q1 + 2) >> 2, (2 * q1 + q0 + p1 + 2) >> 2, q1], -1)
    strong = bs == 4
    out = np.where(f[..., None], np.where(strong[..., None], st, w), s)
    weak = f & ~strong
    br = dict(filtered=f, delta_clipped=weak & (np.abs(raw) > tc), p0_clip_0=weak & (p0 + delta < 0), p0_clip_255=weak & (p0 + delta > 255), q0_clip_0=weak & (q0 - delta < 0),
              q0_clip_255=weak & (q0 - delta > 255))
    return out, br


# ---- 8.7, 8.7.1 whole pictures ----
PLANES = ("Y", "Cb", "Cr")
KINDS = ("internal", "left", "top")


def edge_flags(recs, slices):
    """filterLeftMbEdgeFlag, filterTopMbEdgeFlag and whether the macroblock is filtered at all, from the slices alone
    (8.7): disable_deblocking_filter_idc 1 filters nothing, 2 no edge towards a macroblock of another slice, and no edge
    lies on the picture's border.  recs (B, H, W), slices (B, n)."""
    B, H, W = recs.shape
    sidx = recs["slice_idx"].astype(I)
    idc = np.take_along_axis(slices["deblock_idc"].astype(I), sidx.reshape(B, -1), 1).reshape(B, H, W)
    on = idc != 1
    left, top = np.zeros((B, H, W), bool), np.zeros((B, H, W), bool)
    left[:, :, 1:] = on[:, :, 1:] & ((idc[:, :, 1:] != 2) | (sidx[:, :, 1:] == sidx[:, :, :-1]))
    top[:, 1:] = on[:, 1:] & ((idc[:, 1:] != 2) | (sidx[:, 1:] == sidx[:, :-1]))
    across = np.zeros((B, H, W), I)   # macroblock edges with a neighbour left unfiltered by idc 2 (another slice)
    across[:, :, 1:] += on[:, :, 1:] & (idc[:, :, 1:] == 2) & (sidx[:, :, 1:] != sidx[:, :, :-1])
    across[:, 1:] += on[:, 1:] & (idc[:, 1:] == 2) & (sidx[:, 1:] != sidx[:, :-1])
    return on, left, top, across


def derive(recs, slices):
    """Everything 8.7.2.1 and 8.7.2.2 derive from the records of a batch of pictures: recs (B, H, W) REC, slices (B, n)
    SLICE.  bs (B, H, W, 2, 4, 4) [direction: 0 vertical, 1 horizontal][edge][segment] is 0 on edges that are not
    filtered; the thresholds are (B, H, W, 3 planes, 3 kinds)."""
    B, H, W = recs.shape
    on, left, top, across = edge_flags(recs, slices)
    flags = recs["flags"].astype(I)
    # the records carry the same decision (records.h): MBF_DEBLOCK never in an idc 1 slice, and where it is set, the
    # edge flags are the derived ones.  A macroblock without MBF_DEBLOCK in an idc 0 / 2 slice is a concealed one, which
    # belongs to no decoded slice: it is left as it is, and its neighbours still filter their edges towards it.
    dbk = (flags & MBF_DEBLOCK) != 0
    assert not (dbk & ~on).any(), "MBF_DEBLOCK in a slice with disable_deblocking_filter_idc 1"
    assert np.array_equal(((flags & MBF_EDGE_L) != 0) & dbk, left & dbk), "MBF_EDGE_L differs from filterLeftMbEdgeFlag"
    assert np.array_equal(((flags & MBF_EDGE_T) != 0) & dbk, top & dbk), "MBF_EDGE_T differs from filterTopMbEdgeFlag"
    assert not ((flags & (MBF_EDGE_L | MBF_EDGE_T)) != 0)[~dbk].any(), "an edge flag without MBF_DEBLOCK"
    left, top = left & dbk, top & dbk
    t8 = (flags & MBF_T8x8) != 0
    lrec = recs[:, :, np.maximum(np.arange(W) - 1, 0)]     # the left / top neighbour (the macroblock itself on the border)
    trec = recs[:, np.maximum(np.arange(H) - 1, 0)]
    bs = np.zeros((B, H, W, 2, 4, 4), I)
    rule = np.zeros((B, H, W, 2, 4, 4), I)
    for d in range(2):
        for e in range(4):
            for k in range(4):
                bq = blk_z(k, e) if d else blk_z(e, k)
                bp = (blk_z(k, e - 1) if d else blk_z(e - 1, k)) if e else (blk_z(k, 3) if d else blk_z(3, k))
                p = recs if e else (trec if d else lrec)
                ip, cp, pp, mp = rec_fields(p, bp)
                iq, cq, pq, mq = rec_fields(recs, bq)
                b, r = boundary_strength(ip, iq, cp, cq, pp, pq, mp, mq, e == 0)
                filtered = (top if d else left) if e == 0 else dbk
                bs[..., d, e, k] = np.where(filtered, b, 0)
                rule[..., d, e, k] = r
    # luma edges 1 and 3 are not filtered under transform_size_8x8_flag (8.7: "transform_size_8x8_flag ... is equal to 1")
    t8_skipped = (t8 & dbk)[..., None, None] & (bs[..., (1, 3), :] != 0).any(-1)
    luma_bs = bs.copy()
    luma_bs[..., (1, 3), :] = np.where(t8[..., None, None, None], 0, bs[..., (1, 3), :])
    sl = np.take_along_axis(slices, recs["slice_idx"].astype(I).reshape(B, -1), 1).reshape(B, H, W)
    qp = recs["qp"].astype(I)
    qp_l, qp_t = qp[:, :, np.maximum(np.arange(W) - 1, 0)], qp[:, np.maximum(np.arange(H) - 1, 0)]
    th = thresholds(np.stack([qp, qp_l, qp_t], -1), qp[..., None], sl["filter_offset_a"][..., None, None], sl["filter_offset_b"][..., None, None])
    return dict(bs=bs, luma_bs=luma_bs, rule=rule, dbk=dbk, left=left, top=top, across=across, t8=t8, t8_skipped=t8_skipped, th=th)


def planes_of(frames, g):
    """(B, frame_bytes) uint8 in the layout of E264PicDesc -> [Y, Cb, Cr] int64 copies (B, rows, columns)."""
    W, H, sy, sc, py = g["width_mbs"], g["height_mbs"], g["stride_y"], g["stride_c"], g["plane_y"]
    f = np.asarray(frames)
    y = f[:, :sy * H * 16].reshape(-1, H * 16, sy)[:, :, :W * 16].astype(I)
    c = f[:, py:py + sc * H * 8].reshape(-1, H * 8, sc)
    return [y, c[:, :, :W * 8].astype(I), c[:, :, sc // 2:sc // 2 + W * 8].astype(I)]


def store_planes(frames, g, planes):
    W, H, sy, sc, py = g["width_mbs"], g["height_mbs"], g["stride_y"], g["stride_c"], g["plane_y"]
    out = np.array(frames, np.uint8, copy=True)
    out[:, :sy * H * 16].reshape(-1, H * 16, sy)[:, :, :W * 16] = planes[0]
    c = out[:, py:py + sc * H * 8].reshape(-1, H * 8, sc)
    c[:, :, :W * 8] = planes[1]
    c[:, :, sc // 2:sc // 2 + W * 8] = planes[2]
    return out


def deblock_pictures(g, recs, slices, pre):
    """The deblocked pictures of a batch: g the geometry (a mapping with width_mbs, height_mbs, stride_y, stride_c,
    plane_y), recs (B, H*W) REC, slices (B, n) SLICE, pre (B, frame_bytes) uint8 before the filter.  Macroblocks in raster
    order; in each, the vertical edges left to right, then the horizontal edges top to bottom; luma, Cb and Cr
    independently (8.7).  Returns the pictures and d = derive(...) with d["cov"] the coverage counts."""
    W, H = g["width_mbs"], g["height_mbs"]
    recs = np.asarray(recs, REC).reshape(-1, H, W)
    d = derive(recs, np.asarray(slices, SLICE))
    th, cov = d["th"], collections.Counter()
    pl = planes_of(pre, g)
    for mby in range(H):
        for mbx in range(W):
            for dr in range(2):
                for e in range(4):
                    for p in range(3):
                        n = 16 if p == 0 else 8
                        if p and e & 1:
                            continue
                        # chroma line k takes the bS of luma line 2k: chroma edges 0, 1 are luma edges 0, 2
                        seg = d["luma_bs"][:, mby, mbx, dr, e] if p == 0 else d["bs"][:, mby, mbx, dr, e]
                        bs = seg[:, np.arange(n) * (16 // n) >> 2]        # (B, n lines)
                        if not bs.any():
                            continue
                        kind = 0 if e else 1 + dr
                        t = {k: v[:, mby, mbx, p, kind][:, None] for k, v in th.items()}
                        tc0 = _TC0[np.clip(bs, 0, 3), t["index_a"]]
                        m = 4 if p == 0 else 2               # samples on each side
                        pos = e * n // 4                     # the edge's sample coordinate inside the macroblock
                        X, Y = mbx * n, mby * n
                        a = pl[p]
                        if dr == 0:
                            win = a[:, Y:Y + n, X + pos - m:X + pos + m]
                        else:
                            win = np.swapaxes(a[:, Y + pos - m:Y + pos + m, X:X + n], 1, 2)
                        new, br = (filter_luma if p == 0 else filter_chroma)(win, bs, t["alpha"], t["beta"], tc0)
                        changed = (new != win).any(-1)
                        if dr == 0:
                            a[:, Y:Y + n, X + pos - m:X + pos + m] = new
                        else:
                            a[:, Y + pos - m:Y + pos + m, X:X + n] = np.swapaxes(new, 1, 2)
                        for b in (1, 2, 3, 4):
                            cov["changed", PLANES[p], KINDS[kind], b] += int((changed & (bs == b)).sum())
                        for k, v in br.items():
                            if k != "filtered":
                                cov[k] += int(v.sum())
                        cov["lines", PLANES[p]] += int((bs != 0).sum())
                        edge_on = (bs != 0).any(1)
                        for side, raw in (("a", t["raw_a"][:, 0]), ("b", t["raw_b"][:, 0])):
                            cov["index_%s_clip_0" % side] += int((edge_on & (raw < 0)).sum())
                            cov["index_%s_clip_51" % side] += int((edge_on & (raw > 51)).sum())
    cov["idc2_edges_unfiltered"] += int(d["across"].sum())
    cov["t8x8_internal_edges_skipped"] += int(d["t8_skipped"].sum())
    d["cov"] = cov
    return store_planes(pre, g, pl), d


def explain(d, b, g, plane, x, y):
    """The edge lines of picture b of a derive() result that can change sample (x, y) of plane 0..2: one dict per line,
    with the macroblock, direction, edge, line, bS, alpha, beta and t'C0 the statement derived."""
    n = 16 if plane == 0 else 8
    m = 3 if plane == 0 else 1
    out = []
    for dr in range(2):
        along, across = (y, x) if dr == 0 else (x, y)
        for e in range(4 if plane == 0 else 2):
            for mb_across in range(max(0, (across - m) // n), (across + m) // n + 1):
                pos = mb_across * n + e * 4
                if not (pos - m <= across < pos + m):
                    continue
                mbx, mby = (mb_across, along // n) if dr == 0 else (along // n, mb_across)
                if mbx >= g["width_mbs"] or mby >= g["height_mbs"]:
                    continue
                line = along % n
                le = e if plane == 0 else 2 * e
                bs = int((d["luma_bs"] if plane == 0 else d["bs"])[b, mby, mbx, dr, le, (line * (16 // n)) >> 2])
                kind = 0 if le else 1 + dr
                t = {k: int(v[b, mby, mbx, plane, kind]) for k, v in d["th"].items()}
                out.append(dict(mb=(mbx, mby), plane=PLANES[plane], dir="vertical" if dr == 0 else "horizontal", edge=le, line=line, bs=bs,
                                alpha=t["alpha"], beta=t["beta"], tc0=int(_TC0[bs, t["index_a"]]) if 0 < bs < 4 else None,
                                rule=BS_RULES[int(d["rule"][b, mby, mbx, dr, le, (line * (16 // n)) >> 2])]))
    return out
