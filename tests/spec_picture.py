"""Whole-picture reconstruction of ITU-T H.264 (04/2017) for 8-bit 4:2:0 frame pictures before deblocking: how a picture's
records (edge264_b200/csrc/records.h) are composed into the sample processes of tests/spec_pixels.py and
tests/spec_residual.py.  This module adds no sample arithmetic of its own: every sample comes from a function of those two
statements.  What it states is the selection and the positioning, each rule a named step:
  - order (8.3, 8.4): inter macroblocks read reference pictures only (the record contract never names the picture being
    built as a reference), so they come first; intra macroblocks then in raster order, batched by wavefront (x + 2y
    constant: a macroblock's neighbours A, B, C and D all lie on earlier wavefronts) across the pictures of a batch;
  - neighbour samples by position (6.4.12): p[x,-1], p[-1,y] and p[-1,-1] are read at their picture coordinates from the
    samples constructed so far, inter macroblocks included; availability is the record's unavailability bits as given;
  - Intra4x4 / Intra8x8: block n is predicted in luma4x4BlkIdx / 8x8 order and constructed with its residual before
    block n + 1 is predicted (8.3.1, 8.3.2, 8.5.14); Intra16x16 and chroma: one prediction of the macroblock plus the
    residual of mb_residual; I_PCM: the 384 raw bytes of the coefficient run (8.3.5);
  - inter (8.4.2): for each 4x4 block z, list l is used where ref_idx[l][z >> 2] >= 0 and reads frame slot
    ref_pic[l][z >> 2]; luma at (16 mbx + 4 bx + x + (mvx >> 2), ...) with fraction (mvx & 3, mvy & 3); chroma a 2x2 block
    at (8 mbx + 2 bx + x + (mvx >> 3), ...) with fraction (mvx & 7, mvy & 7), the chroma vector being the luma one for
    frames (8.4.1.4); the weighting the slice's wp_mode selects (8.4.2.3);
  - luma-only pictures (E264PicDesc.luma_only): the chroma planes are 128, whatever the records say about chroma.

With ref=True the composition uses, wherever the project reproduces the reference decoder's arithmetic, the named ref_*
functions of the two statements; with ref=False the standard's.  Either way every macroblock is also evaluated the other
way on the same inputs (the neighbours and reference planes as composed), and where the two differ in a plane of a
macroblock, one of DEVIATIONS must be present in that plane of that macroblock (the residual ones in the luma or the chroma
residual, the interpolation one in luma, the weighting and construction ones in the plane they change); a macroblock plane
where they differ without one is returned in d["unexplained"]."""
import collections
import numpy as np
import spec_pixels as px
import spec_residual as rs
from spec_deblock import REC, SLICE, MBK_INTER, planes_of

I = np.int64
MBK_I4x4, MBK_I8x8, MBK_I16x16, MBK_IPCM = 0, 1, 2, 3
KIND_NAMES = ("I4x4", "I8x8", "I16x16", "I_PCM", "inter")
WP_NAMES = ("default", "explicit", "implicit")
# the reproduced behaviours of the reference decoder that can make its result differ from the standard's, by macroblock
DEVIATIONS = ("residual_outside_int16",     # mb_residual's ok: a bounded value of 8.5.10-8.5.13 leaves int16 (non-conforming)
              "residual_8x8_top",           # mb_residual's top: an 8x8 block's m in 32736..32767 (ref_idct8x8_int16)
              "luma_j_inner_int16",         # ref_luma_j_int16's inner sum leaves int16 at f, i, j, k or q
              "explicit_bi_sum_int16",      # ref_wp_bi_int16: an explicit bi-predicted sum leaves int16 at logWD 7
              "pred_plus_r_int16")          # ref_add_int16: pred + r leaves int16
DEV_BIT = {n: 1 << k for k, n in enumerate(DEVIATIONS)}
BLK_X = np.array([rs.blk_xy(z)[0] for z in range(16)])
BLK_Y = np.array([rs.blk_xy(z)[1] for z in range(16)])


def _in16(v):
    return (v >= rs.LO) & (v <= rs.HI)


def coef_run(levels, r):
    """The coefficient run of record r (at most 408 levels: records.h)."""
    off = int(r["coef_off"])
    return levels[off:off + 408]


def _block_index(pb, x0, y0, nh, nw):
    """fancy indices (picture, row, column) of the nh x nw blocks at (x0, y0) of pictures pb"""
    return (pb[:, None, None], np.asarray(y0)[:, None, None] + np.arange(nh)[None, :, None],
            np.asarray(x0)[:, None, None] + np.arange(nw)[None, None, :])


def neighbours(plane, pb, x0, y0, ntop, nleft):
    """6.4.12 for blocks at sample position (x0, y0) of pictures pb: p[-1,-1], p[0..ntop-1,-1], p[-1,0..nleft-1] read from
    plane (B, rows, columns) at their picture coordinates.  Positions outside the picture are clamped to it: the
    prediction functions never read the samples of a neighbour the unavailability bits mark unavailable, and the record
    contract marks every neighbour outside the picture unavailable."""
    rows, cols = plane.shape[1:]
    ty, lx = np.clip(y0 - 1, 0, rows - 1), np.clip(x0 - 1, 0, cols - 1)
    top = plane[pb[:, None], ty[:, None], np.clip(x0[:, None] + np.arange(ntop), 0, cols - 1)]
    left = plane[pb[:, None], np.clip(y0[:, None] + np.arange(nleft), 0, rows - 1), lx[:, None]]
    return plane[pb, ty, lx], top, left


class _Picture:
    """The state of one batch: planes under construction, the residuals, the per-macroblock deviation bits."""

    def __init__(self, g, recs, slices, coefs, luma_only, ref):
        self.W, self.H = int(g["width_mbs"]), int(g["height_mbs"])
        self.geom = {k: int(g[k]) for k in ("width_mbs", "height_mbs", "stride_y", "stride_c", "plane_y")}
        self.B = len(recs)
        self.recs, self.slices, self.coefs = recs, slices, coefs
        self.luma_only, self.ref = np.asarray(luma_only, bool), ref
        self.planes = [np.zeros((self.B, 16 * self.H, 16 * self.W), I)] + [np.zeros((self.B, 8 * self.H, 8 * self.W), I) for _ in range(2)]
        self.dev = np.zeros((self.B, self.H * self.W, 3), I)        # per plane Y, Cb, Cr: DEV_BIT of the deviations present
        self.differs = np.zeros((self.B, self.H * self.W, 3), bool)  # per plane: the standard and the decoder's arithmetic differ
        self.cov = collections.Counter()

    def residuals(self):
        """mb_residual of every macroblock with coded levels, both ways: self.res_dec / self.res_std (K + 1, 384), the
        row of macroblock (b, a) being self.rid[b, a] (the last row, all zero, for the others).  The luma and the chroma
        residual are taken apart (the chroma levels follow the luma ones in the run, records.h), so that a deviation of
        either is attributed to its own planes."""
        B, nmb = self.B, self.H * self.W
        self.rid = np.full((B, nmb), -1, I)
        rows_d, rows_s = [], []
        for b, a in zip(*np.nonzero((self.recs["coded"] != 0) & (self.recs["kind"] != MBK_IPCM))):
            r = self.recs[b, a]
            sl = self.slices[b, r["slice_idx"]]
            kind, t8, coded, run = int(r["kind"]), bool(r["flags"] & 1), int(r["coded"]), coef_run(self.coefs[b], r)
            common = (r["qp"].astype(I), sl["scaling4x4"], sl["scaling8x8"])
            rd, ok, top = rs.mb_residual(kind, t8, coded, common[0], run, *common[1:], luma_only=True, ref=True)
            rstd = rs.mb_residual(kind, t8, coded, common[0], run, *common[1:], luma_only=True, ref=False)[0]
            self.dev[b, a, 0] |= (0 if ok else DEV_BIT["residual_outside_int16"]) | (DEV_BIT["residual_8x8_top"] if top else 0)
            chroma = coded & (0xff << 16 | rs.CODED_CB_DC | rs.CODED_CR_DC)
            if chroma and not self.luma_only[b]:
                n_luma = (16 if coded & rs.CODED_Y_DC else 0) + (64 * sum((coded >> (4 * i)) & 1 for i in range(4)) if t8 else
                                                                  16 * bin(coded & 0xffff).count("1"))
                cd, ok, _ = rs.mb_residual(kind, t8, chroma, common[0], run[n_luma:], *common[1:], ref=True)
                rd, rstd = rd + cd, rstd + rs.mb_residual(kind, t8, chroma, common[0], run[n_luma:], *common[1:], ref=False)[0]
                self.dev[b, a, 1:] |= 0 if ok else DEV_BIT["residual_outside_int16"]
            self.rid[b, a] = len(rows_d)
            rows_d.append(rd)
            rows_s.append(rstd)
            kind = "inter" if r["kind"] == MBK_INTER else "intra"
            if int(r["coded"]) & 0xffff:
                self.cov["transform", "8x8" if r["flags"] & 1 else "4x4", kind] += 1
            if not self.luma_only[b] and int(r["coded"]) & (rs.CODED_CB_DC | rs.CODED_CR_DC):
                self.cov["chroma_dc_only_blocks"] += sum(1 for i in range(8) if not (int(r["coded"]) >> (16 + i)) & 1)
            if r["kind"] == MBK_I16x16 and int(r["coded"]) & rs.CODED_Y_DC:
                self.cov["intra16x16_dc", "with_ac" if int(r["coded"]) & 0xffff else "without_ac"] += 1
        self.res_dec = np.array(rows_d + [np.zeros(384, I)], I)
        self.res_std = np.array(rows_s + [np.zeros(384, I)], I)

    def construct(self, pred, pb, pa, plane, part):
        """8.5.14 for predictions pred (n, ...) of plane 0..2 of macroblocks (pb, pa): the residual `part` (a function of
        the (n, 384) residual rows giving pred's shape), construct / ref_add_int16.  Returns the composed samples."""
        rd, rstd = part(self.res_dec[self.rid[pb, pa]]), part(self.res_std[self.rid[pb, pa]])
        return self.settle(pred, pred, rd, rstd, pb, pa, plane)

    def settle(self, pred_dec, pred_std, rd, rstd, pb, pa, plane):
        """ref_add_int16(pred_dec, rd) and construct(pred_std, rstd) of plane 0..2 of macroblocks (pb, pa, each once): notes
        where the two differ and where pred + r leaves int16; returns the decoder's with ref, else the standard's."""
        dec, std = rs.ref_add_int16(pred_dec, rd), rs.construct(pred_std, rstd)
        wrap = ~_in16(pred_dec + rd)
        axes = tuple(range(1, dec.ndim))
        self.dev[pb, pa, plane] |= np.where(wrap.any(axes), DEV_BIT["pred_plus_r_int16"], 0)
        self.differs[pb, pa, plane] |= (dec != std).any(axes)
        return dec if self.ref else std


def _y_part(bx, by, n):
    """the n x n luma residual block at 4x4-block column bx, row by of each row of (k, 384) residuals"""
    return lambda r: r[:, :256].reshape(-1, 16, 16)[:, 4 * by:4 * by + n, 4 * bx:4 * bx + n]


def _c_part(pl):
    return lambda r: r[:, 256 + 64 * pl:320 + 64 * pl].reshape(-1, 8, 8)


def _groups(keys):
    """indices of each distinct key, keys (n,)"""
    order = np.argsort(keys, kind="stable")
    ks = keys[order]
    cuts = np.nonzero(np.diff(ks))[0] + 1
    return [(int(keys[s[0]]), s) for s in np.split(order, cuts)] if len(keys) else []


# ---- inter (8.4) ----
def _inter(st, refs):
    W, H, B = st.W, st.H, st.B
    pb, pa = np.nonzero(st.recs["kind"] == MBK_INTER)
    M = len(pb)
    if not M:
        return
    r = st.recs[pb, pa]
    sl = st.slices[pb, r["slice_idx"]]
    mbx, mby = pa % W, pa // W
    i8 = np.arange(16) >> 2
    ref_idx = r["ref_idx"][:, :, i8].astype(I).transpose(0, 2, 1)       # (M, 16 blocks, 2 lists)
    slot = r["ref_pic"][:, :, i8].astype(I).transpose(0, 2, 1)
    use = ref_idx >= 0
    mv = r["mv"].astype(I).transpose(0, 2, 1, 3)                         # (M, 16, 2, [x, y])
    colour = ~st.luma_only[pb]
    # the macroblock's 8x8 blocks with different list usage; one slot in both lists
    usage = use[:, ::4, 0] * 1 + use[:, ::4, 1] * 2
    st.cov["mixed_list_usage_8x8"] += int((usage != usage[:, :1]).any(1).sum())
    st.cov["one_slot_both_lists"] += int((use.all(2) & (slot[..., 0] == slot[..., 1])).sum())
    # 8.4.2.2: the samples of each used list, grouped by (picture, slot) so that each group reads one reference picture
    n4 = np.arange(4)
    LX = (16 * mbx)[:, None, None, None, None] + (4 * BLK_X)[None, :, None, None, None] + n4[None, None, None, None, :] + (mv[..., 0] >> 2)[..., None, None]
    LY = (16 * mby)[:, None, None, None, None] + (4 * BLK_Y)[None, :, None, None, None] + n4[None, None, None, :, None] + (mv[..., 1] >> 2)[..., None, None]
    n2 = np.arange(2)
    CX = (8 * mbx)[:, None, None, None, None] + (2 * BLK_X)[None, :, None, None, None] + n2[None, None, None, None, :] + (mv[..., 0] >> 3)[..., None, None]
    CY = (8 * mby)[:, None, None, None, None] + (2 * BLK_Y)[None, :, None, None, None] + n2[None, None, None, :, None] + (mv[..., 1] >> 3)[..., None, None]
    lfx, lfy, cfx, cfy = mv[..., 0] & 3, mv[..., 1] & 3, mv[..., 0] & 7, mv[..., 1] & 7
    pred_dec = [np.zeros((M, 16, 2, 4, 4), I), np.zeros((M, 16, 2, 2, 2), I), np.zeros((M, 16, 2, 2, 2), I)]
    pred_std = [np.zeros((M, 16, 2, 4, 4), I), np.zeros((M, 16, 2, 2, 2), I), np.zeros((M, 16, 2, 2, 2), I)]
    j_out = np.zeros((M, 16, 2), bool)
    flat = np.nonzero(use.ravel())[0]
    keys = (pb[:, None, None] * 64 + np.where(use, slot, 0)).ravel()[flat]
    jfrac = np.zeros((4, 4), bool)
    for fx, fy in px.J_FRACTIONS:
        jfrac[fx, fy] = True
    for key, sel in _groups(keys):
        b, s = divmod(key, 64)
        frame = refs[b].get(s)
        assert frame is not None, f"picture {b} predicts from frame slot {s}, whose content is not known"
        Yp, Cb, Cr = [p[0] for p in planes_of(np.asarray(frame)[None], st.geom)]
        idx = np.unravel_index(flat[sel], use.shape)
        x, y, fx, fy = LX[idx], LY[idx], lfx[idx][:, None, None], lfy[idx][:, None, None]
        pred_dec[0][idx] = px.ref_luma_j_int16(Yp, x, y, fx, fy)
        pred_std[0][idx] = px.luma_sample(Yp, x, y, fx, fy)
        jj = jfrac[lfx[idx], lfy[idx]]
        if jj.any():
            t = px.luma_j_inner(Yp, x[jj], y[jj], fx[jj])
            jo = np.zeros(len(jj), bool)
            jo[jj] = (~_in16(t)).reshape(int(jj.sum()), -1).any(1)
            j_out[idx] = jo
        for c, pl in ((1, Cb), (2, Cr)):
            v = px.chroma_sample(pl, CX[idx], CY[idx], cfx[idx][:, None, None], cfy[idx][:, None, None])
            pred_dec[c][idx] = pred_std[c][idx] = v
        # coverage: fractions and positions clamped past each edge
        col = colour[idx[0]]
        for f in zip(lfx[idx].tolist(), lfy[idx].tolist()):
            st.cov["luma_fraction", f] += 1
        for f in zip(cfx[idx][col].tolist(), cfy[idx][col].tolist()):
            st.cov["chroma_fraction", f] += 1
        for name, (X, Y, w, h), m in (("luma", (x, y, 16 * W, 16 * H), np.ones(len(x), bool)),
                                      ("chroma", (CX[idx], CY[idx], 8 * W, 8 * H), col)):
            for edge, out in (("left", X < 0), ("right", X > w - 1), ("top", Y < 0), ("bottom", Y > h - 1)):
                st.cov["clamped", name, edge] += int((out.reshape(len(x), -1).any(1) & m).sum())
    st.dev[pb, pa, 0] |= np.where(j_out.any((1, 2)), DEV_BIT["luma_j_inner_int16"], 0)
    # 8.4.2.3: the weighting of the slice's wp_mode, per block and component
    wp = sl["wp_mode"].astype(I)[:, None]
    r0, r1 = ref_idx[..., 0] & 15, ref_idx[..., 1] & 15
    bi, only0 = use.all(2), use[..., 0] & ~use[..., 1]
    m_ = np.arange(M)[:, None]
    lw = [np.broadcast_to(sl["luma_log2_wd"].astype(I)[:, None], (M, 16)), np.broadcast_to(sl["chroma_log2_wd"].astype(I)[:, None], (M, 16))]
    w1i = sl["implicit_w1"].astype(I)[m_, r0, r1]
    for name, k in (("default", 0), ("explicit", 1), ("implicit", 2)):
        on = wp == k
        st.cov["wp", name, "L0"] += int((on & only0).sum())
        st.cov["wp", name, "L1"] += int((on & use[..., 1] & ~use[..., 0]).sum())
        st.cov["wp", name, "bi"] += int((on & bi).sum())
    st.cov["implicit_w1", -64] += int(((wp == 2) & bi & (w1i == -64)).sum())
    st.cov["implicit_w1", 128] += int(((wp == 2) & bi & (w1i == 128)).sum())
    for comp, cname in ((0, "luma"), (1, "chroma")):
        for v in (0, 7):
            st.cov["explicit_logwd", cname, v] += int(((wp == 1) & (lw[comp] == v)).sum())
    lum_only = st.luma_only[pb]
    composed = []
    bi_out = np.zeros((M, 3), bool)      # per plane: an explicit bi sum leaves int16 at logWD 7
    for c in range(3):
        logwd = lw[min(c, 1)]
        w = [sl["wp_w"].astype(I)[m_, l, (r0, r1)[l], c] for l in (0, 1)]
        o = [sl["wp_o"].astype(I)[m_, l, (r0, r1)[l], c] for l in (0, 1)]
        e = lambda a: a[:, :, None, None]
        out = []
        for p in (pred_dec[c], pred_std[c]):
            p0, p1 = p[:, :, 0], p[:, :, 1]
            puni = np.where(e(only0), p0, p1)
            wl, ol = np.where(only0, w[0], w[1]), np.where(only0, o[0], o[1])
            if p is pred_dec[c]:
                exp_bi = px.ref_wp_bi_int16(p0, p1, e(w[0]), e(w[1]), e(o[0]), e(o[1]), e(logwd))
                imp_bi = px.ref_wp_bi_int16(p0, p1, e(64 - w1i), e(w1i), 0, 0, 5)
                s = px.bi_sum(p0, p1, e(w[0]), e(w[1]), e(o[0]), e(o[1]), e(logwd))
                bi_out[:, c] |= ((wp == 1) & bi & (logwd == 7) & (~_in16(s)).any((2, 3))).any(1) & ((c == 0) | ~lum_only)
            else:
                exp_bi = px.wp_explicit_bi(p0, p1, e(w[0]), e(w[1]), e(o[0]), e(o[1]), e(logwd))
                imp_bi = px.wp_implicit(p0, p1, e(w1i))
            both = np.select([e(wp == 1), e(wp == 2)], [exp_bi, imp_bi], px.wp_default(p0, p1))
            one = np.where(e(wp == 1), px.wp_explicit_uni(puni, e(wl), e(ol), e(logwd)), puni)
            out.append(np.where(e(bi), both, one))
        composed.append(out)
    st.dev[pb, pa] |= np.where(bi_out, DEV_BIT["explicit_bi_sum_int16"], 0)
    # 8.5.14: the prediction of each plane as a macroblock, plus the residual
    for c in range(3):
        n = 4 if c == 0 else 2
        N = 4 * n
        mb = [np.zeros((M, N, N), I), np.zeros((M, N, N), I)]
        for z in range(16):
            for k in range(2):
                mb[k][:, n * BLK_Y[z]:n * BLK_Y[z] + n, n * BLK_X[z]:n * BLK_X[z] + n] = composed[c][k][:, z]
        part = (lambda r: r[:, :256].reshape(-1, 16, 16)) if c == 0 else _c_part(c - 1)
        keep = np.ones(M, bool) if c == 0 else ~lum_only
        rd, rstd = part(st.res_dec[st.rid[pb, pa]]), part(st.res_std[st.rid[pb, pa]])
        v = st.settle(mb[0][keep], mb[1][keep], rd[keep], rstd[keep], pb[keep], pa[keep], c)
        st.planes[c][_block_index(pb[keep], (N * mbx)[keep], (N * mby)[keep], N, N)] = v


# ---- intra (8.3) ----
def _intra_blocks(st, fn, N, pb, pa, x0, y0, modes, nb_top, nb_left, part, step_note):
    """Predict blocks of size N at (x0, y0) of macroblocks (pb, pa) with mode bytes `modes`, construct them with `part`
    of the residual and write them into the luma plane."""
    plane = st.planes[0]
    for byte, g in _groups(modes):
        mode, un = byte & 15, byte >> 4
        corner, top, left = neighbours(plane, pb[g], x0[g], y0[g], nb_top, nb_left)
        pred = fn(mode, un, corner, top, left)
        st.cov[fn.__name__, mode, un] += len(g)
        step_note(g, un)
        st.planes[0][_block_index(pb[g], x0[g], y0[g], N, N)] = st.construct(pred, pb[g], pa[g], 0, part)


def _intra(st):
    W = st.W
    pb, pa = np.nonzero(st.recs["kind"] != MBK_INTER)
    if not len(pb):
        return
    wave = pa % W + 2 * (pa // W)
    kinds = st.recs["kind"]
    for w, sel in _groups(wave):
        b, a = pb[sel], pa[sel]
        r = st.recs[b, a]
        mbx, mby = a % W, a // W
        k = r["kind"]
        # I_PCM (8.3.5): the raw samples of the coefficient run
        for i in np.nonzero(k == MBK_IPCM)[0]:
            raw = np.asarray(coef_run(st.coefs[b[i]], r[i])[:192]).view(np.uint8).astype(I)
            bi_, x, y = b[i], mbx[i], mby[i]
            st.planes[0][bi_, 16 * y:16 * y + 16, 16 * x:16 * x + 16] = raw[:256].reshape(16, 16)
            for c in (1, 2):
                st.planes[c][bi_, 8 * y:8 * y + 8, 8 * x:8 * x + 8] = raw[256 + 64 * (c - 1):320 + 64 * (c - 1)].reshape(8, 8)
            st.cov["I_PCM"] += 1
        # Intra16x16 (8.3.3)
        s = np.nonzero(k == MBK_I16x16)[0]
        if len(s):
            _intra_blocks(st, px.intra16x16, 16, b[s], a[s], 16 * mbx[s], 16 * mby[s], r["i16_mode"][s].astype(I), 16, 16,
                          lambda rr: rr[:, :256].reshape(-1, 16, 16), lambda g, un: None)
        # Intra4x4 / Intra8x8 (8.3.1, 8.3.2): block by block, each constructed before the next is predicted
        for kind, fn, N, nblk in ((MBK_I4x4, px.intra4x4, 4, 16), (MBK_I8x8, px.intra8x8, 8, 4)):
            s = np.nonzero(k == kind)[0]
            for z in range(nblk if len(s) else 0):
                bx, by = (BLK_X[z], BLK_Y[z]) if N == 4 else (z & 1, z >> 1)
                inside = (z in (3, 7, 11, 13, 15)) if N == 4 else z == 3
                edge_blk = (z == 5) if N == 4 else z == 1

                def note(g, un, s=s, inside=inside, edge_blk=edge_blk):
                    if un & px.C and not un & px.B:
                        st.cov["C_substituted", "inside_mb"] += len(g) if inside else 0
                        st.cov["C_substituted", "right_edge"] += int((mbx[s][g] == W - 1).sum()) if edge_blk else 0
                _intra_blocks(st, fn, N, b[s], a[s], 16 * mbx[s] + N * bx, 16 * mby[s] + N * by, r["modes"][s, z].astype(I),
                              2 * N, N, _y_part(bx * N // 4, by * N // 4, N), note)
        # chroma (8.3.4) of every intra macroblock but I_PCM
        s = np.nonzero(k != MBK_IPCM)[0]
        for byte, g in _groups(r["chroma_mode"][s].astype(I)):
            mode, un = byte & 15, byte >> 4
            gb, ga = b[s][g], a[s][g]
            col = ~st.luma_only[gb]
            st.cov["intra_chroma", mode, un] += int(col.sum())
            for c in (1, 2):
                corner, top, left = neighbours(st.planes[c], gb, 8 * mbx[s][g], 8 * mby[s][g], 8, 8)
                pred = px.intra_chroma(mode, un, corner, top, left)
                v = st.construct(pred[col], gb[col], ga[col], c, _c_part(c - 1))
                st.planes[c][_block_index(gb[col], 8 * mbx[s][g][col], 8 * mby[s][g][col], 8, 8)] = v
        # intra macroblocks predicted from an inter neighbour (A, B or D, available for the macroblock's chroma)
        un = r["chroma_mode"].astype(I) >> 4
        for bit, dx, dy in ((px.A, -1, 0), (px.B, 0, -1), (px.D, -1, -1)):
            ok = (k != MBK_IPCM) & ~(un & bit).astype(bool) & (mbx + dx >= 0) & (mby + dy >= 0)
            na = np.where(ok, a + dy * W + dx, 0)
            st.cov["intra_from_inter_neighbour"] += int((ok & (kinds[b, na] == MBK_INTER)).sum())


def concealment_shaped(recs):
    """Records shaped like the decoder's concealment (decoder.c conceal_missing): Intra16x16 DC and chroma DC with A, B and D
    unavailable and no levels, or a P_Skip-like inter macroblock from list 0 at ref_idx 0 without deblocking."""
    intra = (recs["kind"] == MBK_I16x16) & (recs["i16_mode"] == 0xb2) & (recs["chroma_mode"] == 0xb0) & (recs["coded"] == 0) & ((recs["flags"] & 0x08) == 0)
    inter = ((recs["kind"] == MBK_INTER) & (recs["coded"] == 0) & ((recs["flags"] & 0x18) == 0x10) & (recs["ref_idx"][..., 0, :] == 0).all(-1)
             & (recs["ref_idx"][..., 1, :] < 0).all(-1))
    return intra, inter


def reconstruct_pictures(g, recs, slices, coefs, refs, luma_only, ref=True):
    """The pictures of a batch of one geometry before deblocking.  g: a mapping with width_mbs, height_mbs, stride_y,
    stride_c, plane_y, frame_bytes; recs (B, H*W) REC; slices (B, n) SLICE; coefs: B int16 arrays of levels; refs: B
    mappings frame slot -> the frame it holds (uint8, frame_bytes, in the layout of E264PicDesc); luma_only (B,).
    Returns the planes [Y, Cb, Cr] (B, rows, columns) int64 and d: d["cov"] the coverage counts, d["dev"] the deviation
    counts, d["unexplained"] the (picture, macroblock address, plane) where the other arithmetic differs without a
    deviation of that plane of that macroblock, d["differs"] / d["deviations"] (B, H*W, 3) per macroblock and plane."""
    W, H = int(g["width_mbs"]), int(g["height_mbs"])
    recs = np.asarray(recs, REC).reshape(-1, H * W)
    slices = np.asarray(slices, SLICE).reshape(len(recs), -1)
    st = _Picture(g, recs, slices, coefs, luma_only, ref)
    st.residuals()
    _inter(st, refs)
    _intra(st)
    for c in (1, 2):
        st.planes[c][st.luma_only] = 128
    ci, cn = concealment_shaped(recs)
    st.cov["concealment", "intra"] += int(ci.sum())
    st.cov["concealment", "inter"] += int(cn.sum())
    st.cov["luma_only_pictures"] += int(st.luma_only.sum())
    st.cov["colour_pictures"] += int((~st.luma_only).sum())
    dev = collections.Counter()
    for name, bit in DEV_BIT.items():
        present = (st.dev & bit) != 0
        dev[name, "present"] += int(present.sum())
        dev[name, "differs"] += int((present & st.differs).sum())
        st.cov["deviation_differs", name] += int((present & st.differs).sum())
    dev["macroblocks", "differs"] += int(st.differs.any(2).sum())
    dev["macroblocks", "judged"] += st.B * H * W
    unexplained = list(zip(*np.nonzero(st.differs & (st.dev == 0))))
    return st.planes, dict(cov=st.cov, dev=dev, unexplained=unexplained, differs=st.differs, deviations=st.dev)


def explain(recs, slices, g, plane, x, y):
    """What the composition used for sample (x, y) of plane 0..2 of one picture (records (H*W,), slices (n,)): the
    macroblock, its kind, and the block's mode and unavailability bits, or per list the vector, ref_idx, slot and the
    weights in force."""
    W = int(g["width_mbs"])
    n = 16 if plane == 0 else 8
    mbx, mby = x // n, y // n
    a = mby * W + mbx
    r = recs[a]
    sl = slices[r["slice_idx"]]
    kind = int(r["kind"])
    out = dict(mb=a, mbx=mbx, mby=mby, kind=KIND_NAMES[kind], slice=int(r["slice_idx"]), qp=r["qp"].tolist(), coded=hex(int(r["coded"])))
    u = x % n * 4 // n, y % n * 4 // n            # the 4x4 luma block the sample lies in
    z = int(u[0] & 1 | (u[1] & 1) << 1 | (u[0] & 2) << 1 | (u[1] & 2) << 2)
    if kind == MBK_INTER:
        c = min(plane, 1)
        lists = []
        for l in (0, 1):
            ri = int(r["ref_idx"][l, z >> 2])
            if ri < 0:
                continue
            e = dict(list=l, mv=r["mv"][l, z].tolist(), ref_idx=ri, slot=int(r["ref_pic"][l, z >> 2]))
            if sl["wp_mode"] == 1:
                e.update(w=int(sl["wp_w"][l, ri, plane]), o=int(sl["wp_o"][l, ri, plane]), logwd=int(sl["chroma_log2_wd" if c else "luma_log2_wd"]))
            lists.append(e)
        out.update(block=z, wp=WP_NAMES[int(sl["wp_mode"])], lists=lists)
        if sl["wp_mode"] == 2 and len(lists) == 2:
            out["implicit_w1"] = int(sl["implicit_w1"][lists[0]["ref_idx"] & 15, lists[1]["ref_idx"] & 15])
    elif kind != MBK_IPCM:
        m = {MBK_I4x4: ("block", z, int(r["modes"][z])), MBK_I8x8: ("block8x8", z >> 2, int(r["modes"][z >> 2])),
             MBK_I16x16: ("i16", None, int(r["i16_mode"]))}[kind] if plane == 0 else ("chroma", None, int(r["chroma_mode"]))
        out.update(part=m[0], index=m[1], mode=m[2] & 15, unavailable="".join(ch for bit, ch in ((1, "A"), (2, "B"), (4, "C"), (8, "D")) if m[2] >> 4 & bit))
    return out
